// Instantiations of the decode GEMV for vector_len == 8 (the Llama-3 checkpoints' layout):
// 1, 2 or 4 tokens per pass.
#include "gemv_kernel.cuh"

namespace vptq_b200 {

template <typename T, int NT>
static GemvKernelFn pick8(bool main_smem, bool res, bool res_l2) {
  if (res && res_l2) return main_smem ? gemv_kernel_res_l2<T, 8, NT, true> : gemv_kernel_res_l2<T, 8, NT, false>;
  if (main_smem) return res ? gemv_kernel<T, 8, NT, true, true> : gemv_kernel<T, 8, NT, true, false>;
  return res ? gemv_kernel<T, 8, NT, false, true> : gemv_kernel<T, 8, NT, false, false>;
}

template <typename T>
static GemvKernelFn pick8_nt(int nt, bool main_smem, bool res, bool res_l2) {
  switch (nt) {
    case 1: return pick8<T, 1>(main_smem, res, res_l2);
    case 2: return pick8<T, 2>(main_smem, res, res_l2);
    case 4: return pick8<T, 4>(main_smem, res, res_l2);
    default: return nullptr;
  }
}

GemvKernelFn gemv_kernel_v8(int dtype, int nt, bool main_smem, bool res, bool res_l2) {
  if (dtype == VPTQ_FP16) return pick8_nt<__half>(nt, main_smem, res, res_l2);
  if (dtype == VPTQ_BF16) return pick8_nt<__nv_bfloat16>(nt, main_smem, res, res_l2);
  return nullptr;
}

template <typename T, int NT>
static GemvMultiKernelFn pickm8(bool main_smem, bool res, bool res_l2) {
  if (res && res_l2)
    return main_smem ? gemv_multi_kernel_res_l2<T, 8, NT, true> : gemv_multi_kernel_res_l2<T, 8, NT, false>;
  if (main_smem) return res ? gemv_multi_kernel<T, 8, NT, true, true> : gemv_multi_kernel<T, 8, NT, true, false>;
  return res ? gemv_multi_kernel<T, 8, NT, false, true> : gemv_multi_kernel<T, 8, NT, false, false>;
}

// fused launches exist for the decode case proper (1 or 2 tokens)
GemvMultiKernelFn gemv_multi_kernel_v8(int dtype, int nt, bool main_smem, bool res, bool res_l2) {
  if (dtype == VPTQ_FP16)
    return nt == 1 ? pickm8<__half, 1>(main_smem, res, res_l2) : nt == 2 ? pickm8<__half, 2>(main_smem, res, res_l2) : nullptr;
  if (dtype == VPTQ_BF16)
    return nt == 1   ? pickm8<__nv_bfloat16, 1>(main_smem, res, res_l2)
           : nt == 2 ? pickm8<__nv_bfloat16, 2>(main_smem, res, res_l2)
                     : nullptr;
  return nullptr;
}

}  // namespace vptq_b200
