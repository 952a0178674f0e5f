// Instantiations of the decode GEMV for the other vector lengths the reference dispatches
// (csrc/quant_gemv.cu:209-234: 2, 4, 6, 10, 12, 16), one token per pass.
#include "gemv_kernel.cuh"

namespace vptq_b200 {

template <typename T, int V>
static GemvKernelFn pickv(bool main_smem, bool res, bool res_l2) {
  if (res && res_l2) return main_smem ? gemv_kernel_res_l2<T, V, 1, true> : gemv_kernel_res_l2<T, V, 1, false>;
  if (main_smem) return res ? gemv_kernel<T, V, 1, true, true> : gemv_kernel<T, V, 1, true, false>;
  return res ? gemv_kernel<T, V, 1, false, true> : gemv_kernel<T, V, 1, false, false>;
}

template <typename T>
static GemvKernelFn pickv_v(int v, bool main_smem, bool res, bool res_l2) {
  switch (v) {
    case 2: return pickv<T, 2>(main_smem, res, res_l2);
    case 4: return pickv<T, 4>(main_smem, res, res_l2);
    case 6: return pickv<T, 6>(main_smem, res, res_l2);
    case 10: return pickv<T, 10>(main_smem, res, res_l2);
    case 12: return pickv<T, 12>(main_smem, res, res_l2);
    case 16: return pickv<T, 16>(main_smem, res, res_l2);
    default: return nullptr;
  }
}

GemvKernelFn gemv_kernel_vx(int dtype, int v, bool main_smem, bool res, bool res_l2) {
  if (dtype == VPTQ_FP16) return pickv_v<__half>(v, main_smem, res, res_l2);
  if (dtype == VPTQ_BF16) return pickv_v<__nv_bfloat16>(v, main_smem, res, res_l2);
  return nullptr;
}

}  // namespace vptq_b200
