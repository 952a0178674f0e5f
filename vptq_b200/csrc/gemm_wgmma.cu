// Prefill path: y[T][O] = x[T][I] * W[O][I]^T + bias for many tokens, on the Hopper tensor cores
// (wgmma.mma_async, accumulators in registers, operands staged in shared memory by TMA).
//
// Replaces the reference's tokens >= 3 branch (vptq/ops/quant_gemm.py:231-275: the `dequant` CUDA
// op followed by torch F.linear / cuBLAS).  The algebra is rearranged so that the tensor-core
// operand is the RAW quantised weight (no per-column scale / bias / permutation inside the GEMM):
//
//   y[t][o] = sum_c x'[t][c] * Wq[o][c]  +  rowbias[t]  +  bias[o]
//   x'[t][c]   = x[t][perm[c]] * scale[perm[c]]                 (prep kernel, one pass over x)
//   rowbias[t] = sum_f x[t][f] * wbias[f]                        (same kernel, fp32)
//   Wq[o][c]   = C[idx[o/v][c]][o%v] + R[ridx[o/v][c]][o%v]      (outlier columns from their codebook)
//
// Three kernels on the caller's stream:
//   1. prefill_prep_x     x -> x' (16 bit, quantised column order) and rowbias (fp32)
//   2. dequant (dequant.cu, quantised-order mode)  packed indices -> Wq tile source [O][Ipad]
//   3. gemm_tn_wgmma      persistent, warp-specialised: one TMA producer warp and two consumer
//                         warpgroups; 128x256x64 tiles, 4-stage smem ring (48 KB per stage).  Each
//                         warpgroup owns 64 token rows of the tile and keeps its 64x256 fp32 accumulator
//                         in registers (m64n256k16, 128 registers per thread); its epilogue (adds
//                         rowbias[t] + bias[o], writes 16-bit y) runs while the producer already fills the
//                         ring with the next tile's operands.
//
// The same GEMM computes the layer's input gradient dX = dY . W (VPTQ_FLAG_TRANSPOSE, dgrad_launch below) from a
// TRANSPOSED dequant Wt[I][O] (dequant.cu): A = dY, B = Wt, N = in_features, K = out_features.
#include <cuda.h>

#include <algorithm>
#include <cstdlib>
#include <mutex>
#include <type_traits>

#include "common.cuh"
#include "kernels.h"

namespace vptq_b200 {

// implemented in dequant.cu
int dequant_quant_order_launch(const vptq_linear_desc& d, void* wq_out, int64_t ld, cudaStream_t stream);
namespace {

constexpr int BM = 128, BN = 256, BK = 64;  // CTA tile: tokens x outputs x reduction
constexpr int WGMMA_K = 16;                 // K per wgmma for 16-bit inputs
constexpr int STAGES = 4;
constexpr int TILE_A_BYTES = BM * BK * 2, TILE_B_BYTES = BN * BK * 2;
constexpr int CONSUMERS = 2;                         // warpgroups, 64 of the BM rows each
constexpr int GEMM_THREADS = CONSUMERS * 128 + 32;   // warps 0-7: consumers, warp 8: TMA producer
constexpr int GEMM_SMEM = STAGES * (TILE_A_BYTES + TILE_B_BYTES) + 1024 /*align*/ + 256 /*barriers*/;

// ---------------------------------------------------------------------------------------------
// x' = x[perm] * scale[perm]  and  rowbias = x . wbias
// ---------------------------------------------------------------------------------------------
// One CTA per token: the row of x is staged in shared memory with coalesced 16-byte loads, then
// gathered from there (2-byte shared-memory reads) while perm / scale stream in coalesced, and x' is
// written with 16-byte stores.  `scale_q` is the optional quantised-order copy scale[perm[c]]
// (vptq_linear_desc.weight_scale_q); without it scale is gathered through perm.
template <typename T>
__global__ void __launch_bounds__(256) prefill_prep_x(const T* __restrict__ x, int64_t x_stride,
                                                      const uint16_t* __restrict__ perm,
                                                      const T* __restrict__ scale, const T* __restrict__ scale_q,
                                                      const T* __restrict__ wbias, T* __restrict__ xq,
                                                      int64_t xq_stride, float* __restrict__ rowbias, int I) {
  extern __shared__ __align__(16) uint8_t prep_smem[];
  T* sx = reinterpret_cast<T*>(prep_smem);
  const int t = blockIdx.x, tid = threadIdx.x;
  const T* xr = x + int64_t(t) * x_stride;
  T* out = xq + int64_t(t) * xq_stride;
  float bs = 0.f;
  const bool vec = ((reinterpret_cast<uintptr_t>(xr) & 15u) == 0) && ((I & 7) == 0) &&
                   ((reinterpret_cast<uintptr_t>(wbias) & 15u) == 0);
  if (vec) {
    for (int i = tid * 8; i < I; i += 256 * 8) {
      const uint4 v = *reinterpret_cast<const uint4*>(xr + i);
      *reinterpret_cast<uint4*>(sx + i) = v;
      if (wbias) {
        const uint4 w = *reinterpret_cast<const uint4*>(wbias + i);
        const uint32_t* vp = reinterpret_cast<const uint32_t*>(&v);
        const uint32_t* wp = reinterpret_cast<const uint32_t*>(&w);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 a = DT<T>::unpack2(vp[k]), c = DT<T>::unpack2(wp[k]);
          bs = fmaf(a.x, c.x, fmaf(a.y, c.y, bs));
        }
      }
    }
  } else {
    for (int i = tid; i < I; i += 256) {
      sx[i] = xr[i];
      if (wbias) bs = fmaf(DT<T>::to_float(xr[i]), DT<T>::to_float(wbias[i]), bs);
    }
  }
  __syncthreads();
  const bool vec_out = ((I & 7) == 0) && (!perm || (reinterpret_cast<uintptr_t>(perm) & 15u) == 0) &&
                       (!scale_q || (reinterpret_cast<uintptr_t>(scale_q) & 15u) == 0) && ((xq_stride & 7) == 0);
  if (vec_out) {
    for (int c = tid * 8; c < I; c += 256 * 8) {
      uint32_t pc[8];
      if (perm) {
        const uint4 pv = *reinterpret_cast<const uint4*>(perm + c);
        const uint32_t* pp = reinterpret_cast<const uint32_t*>(&pv);
#pragma unroll
        for (int k = 0; k < 4; ++k) pc[2 * k] = pp[k] & 0xffffu, pc[2 * k + 1] = pp[k] >> 16;
      } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) pc[k] = uint32_t(c + k);
      }
      float sc[8];
      if (scale_q) {
        const uint4 sv = *reinterpret_cast<const uint4*>(scale_q + c);
        const uint32_t* sp = reinterpret_cast<const uint32_t*>(&sv);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 f2 = DT<T>::unpack2(sp[k]);
          sc[2 * k] = f2.x, sc[2 * k + 1] = f2.y;
        }
      } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) sc[k] = scale ? DT<T>::to_float(scale[pc[k]]) : 1.f;
      }
      uint32_t w[4];
#pragma unroll
      for (int k = 0; k < 4; ++k)
        w[k] = DT<T>::pack2(DT<T>::to_float(sx[pc[2 * k]]) * sc[2 * k], DT<T>::to_float(sx[pc[2 * k + 1]]) * sc[2 * k + 1]);
      *reinterpret_cast<uint4*>(out + c) = make_uint4(w[0], w[1], w[2], w[3]);
    }
  } else {
    for (int c = tid; c < I; c += 256) {
      const int f = perm ? int(perm[c]) : c;
      const float sc = scale_q ? DT<T>::to_float(scale_q[c]) : (scale ? DT<T>::to_float(scale[f]) : 1.f);
      out[c] = DT<T>::from_float(DT<T>::to_float(sx[f]) * sc);
    }
  }
  for (int c = I + tid; c < xq_stride; c += 256) out[c] = DT<T>::from_float(0.f);  // K padding
  __shared__ float red[8];
  bs = warp_sum(bs);
  if ((tid & 31) == 0) red[tid >> 5] = bs;
  __syncthreads();
  if (tid == 0) {
    float v = 0.f;
    for (int w = 0; w < 8; ++w) v += red[w];
    rowbias[t] = v;
  }
}

// ---------------------------------------------------------------------------------------------
// wgmma / TMA PTX wrappers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// shared-memory matrix descriptor: K-major tile whose rows are 128 bytes (64 x 16 bit), 128B swizzle
// (8-row x 128-byte atoms, 1024 bytes apart)
__device__ __forceinline__ uint64_t gmma_desc_k_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= uint64_t((saddr & 0x3FFFFu) >> 4);  // bits [0,14)  start address >> 4
  d |= uint64_t(1) << 16;                  // bits [16,30) leading-dim byte offset (unused: K-major, swizzled)
  d |= uint64_t(1024 >> 4) << 32;          // bits [32,46) stride-dim byte offset: next 8-row group
  d |= uint64_t(1) << 62;                  // bits [62,64) layout: SWIZZLE_128B
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across a wgmma fence or wait
__device__ __forceinline__ void fence_acc(float (&d)[128]) {
#pragma unroll
  for (int i = 0; i < 128; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define VPTQ_WGMMA_D128                                                                             \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "                        \
  "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "               \
  "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "               \
  "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "               \
  "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "               \
  "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "               \
  "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "   \
  "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}"
#define VPTQ_WGMMA_D128_OPERANDS(d)                                                                         \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),                 \
      "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),       \
      "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),     \
      "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),     \
      "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),     \
      "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),     \
      "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),     \
      "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),     \
      "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),     \
      "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),     \
      "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),     \
      "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),     \
      "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), \
      "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]),           \
      "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]),           \
      "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]),           \
      "+f"(d[125]), "+f"(d[126]), "+f"(d[127])

// D[64 x 256] (+)= A[64 x 16, smem desc] * B[256 x 16, smem desc]^T for the whole warpgroup; both operands K-major
template <typename T>
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  if constexpr (std::is_same<T, __half>::value) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 " VPTQ_WGMMA_D128 ", %128, %129, p, 1, 1, 0, 0;\n\t}"
        : VPTQ_WGMMA_D128_OPERANDS(d)
        : "l"(a_desc), "l"(b_desc), "r"(accumulate));
  } else {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 " VPTQ_WGMMA_D128 ", %128, %129, p, 1, 1, 0, 0;\n\t}"
        : VPTQ_WGMMA_D128_OPERANDS(d)
        : "l"(a_desc), "l"(b_desc), "r"(accumulate));
  }
}

struct GemmParams {
  const void* bias;       // [O] 16 bit or nullptr
  const float* rowbias;   // [T]
  void* y;
  int64_t y_stride;
  int T, O, K;            // K = padded reduction length (multiple of 8)
  int is_bf16;
};

template <typename T>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tn_wgmma(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
              const __grid_constant__ GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B tiles must start on 1024-byte boundaries
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sa = smem;
  uint8_t* sb = smem + STAGES * TILE_A_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * (TILE_A_BYTES + TILE_B_BYTES));
  uint64_t* empty = full + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nkb = (p.K + BK - 1) / BK;
  // persistent CTAs walk the tile list with stride gridDim.x; tokens (m) vary fastest so that the
  // CTAs running at the same time share the same weight (B) tiles in L2
  const int tiles_m = (p.T + BM - 1) / BM, tiles_n = (p.O + BN - 1) / BN;
  const int ntiles = tiles_m * tiles_n;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) mbar_init(&full[s], 1), mbar_init(&empty[s], CONSUMERS);
    fence_mbar_init();
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b) : "memory");
  }
  __syncthreads();

  if (warp == CONSUMERS * 4) {
    // ===== TMA producer (one lane) =====
    if (lane == 0) {
      int it = 0;  // running k-block counter across tiles: slot = it % STAGES, round = it / STAGES
      for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int m0 = (tile % tiles_m) * BM, n0 = (tile / tiles_m) * BN;
        for (int kb = 0; kb < nkb; ++kb, ++it) {
          const int s = it % STAGES;
          mbar_wait(&empty[s], ((it / STAGES) & 1) ^ 1);  // slot free (passes immediately in round 0)
          mbar_arrive_expect_tx(&full[s], TILE_A_BYTES + TILE_B_BYTES);
          tma_load_2d(sa + s * TILE_A_BYTES, &map_a, kb * BK, m0, &full[s]);
          tma_load_2d(sb + s * TILE_B_BYTES, &map_b, kb * BK, n0, &full[s]);
        }
      }
    }
    return;
  }

  // ===== consumer warpgroup wg: rows [64 wg, 64 wg + 64) of every tile =====
  const int wg = warp >> 2, wt = threadIdx.x & 127;
  const T* bias = reinterpret_cast<const T*>(p.bias);
  const bool pair_ok = (p.y_stride & 1) == 0 && (reinterpret_cast<uintptr_t>(p.y) & 3u) == 0;
  float acc[128];
  int it = 0;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int m0 = (tile % tiles_m) * BM, n0 = (tile / tiles_m) * BN;
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < nkb; ++kb, ++it) {
      const int s = it % STAGES;
      mbar_wait(&full[s], (it / STAGES) & 1);  // TMA bytes have landed
      const uint64_t da = gmma_desc_k_sw128(smem_u32(sa + s * TILE_A_BYTES + wg * 64 * BK * 2));
      const uint64_t db = gmma_desc_k_sw128(smem_u32(sb + s * TILE_B_BYTES));
      fence_acc(acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / WGMMA_K; ++k) {
        // advance 16 elements (32 bytes) along K inside the 128-byte swizzle atom: +2 in 16-byte units
        wgmma_m64n256k16<T>(acc, da + uint64_t(2 * k), db + uint64_t(2 * k), 1u);
      }
      wgmma_commit();
      // the group of the previous k-block has completed: its smem slot goes back to the producer
      wgmma_wait<1>();
      fence_acc(acc);
      if (kb > 0 && wt == 0) mbar_arrive(&empty[(it - 1) % STAGES]);
    }
    wgmma_wait<0>();
    fence_acc(acc);
    if (nkb > 0 && wt == 0) mbar_arrive(&empty[(it - 1) % STAGES]);

    // ===== epilogue: registers -> (+rowbias +bias) -> 16-bit y =====
    // accumulator layout of m64nNk16: thread (warp w, lane l) of the warpgroup holds rows 16w + l/4 and
    // 16w + l/4 + 8, columns 8j + 2(l%4) + {0, 1} for j = 0 .. N/8-1, as acc[4j .. 4j+3]
    const int r0 = m0 + wg * 64 + (wt >> 5) * 16 + (lane >> 2), r1 = r0 + 8;
    const float rb0 = (p.rowbias && r0 < p.T) ? p.rowbias[r0] : 0.f;
    const float rb1 = (p.rowbias && r1 < p.T) ? p.rowbias[r1] : 0.f;
    T* y0 = reinterpret_cast<T*>(p.y) + int64_t(r0) * p.y_stride;
    T* y1 = reinterpret_cast<T*>(p.y) + int64_t(r1) * p.y_stride;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int n = n0 + 8 * j + 2 * (lane & 3);
      if (n < p.O) {
        const bool two = n + 1 < p.O;
        const float b0 = bias ? DT<T>::to_float(bias[n]) : 0.f;
        const float b1 = (bias && two) ? DT<T>::to_float(bias[n + 1]) : 0.f;
        if (two && pair_ok) {
          if (r0 < p.T) *reinterpret_cast<uint32_t*>(y0 + n) = DT<T>::pack2(acc[4 * j] + rb0 + b0, acc[4 * j + 1] + rb0 + b1);
          if (r1 < p.T) *reinterpret_cast<uint32_t*>(y1 + n) = DT<T>::pack2(acc[4 * j + 2] + rb1 + b0, acc[4 * j + 3] + rb1 + b1);
        } else {
          if (r0 < p.T) {
            y0[n] = DT<T>::from_float(acc[4 * j] + rb0 + b0);
            if (two) y0[n + 1] = DT<T>::from_float(acc[4 * j + 1] + rb0 + b1);
          }
          if (r1 < p.T) {
            y1[n] = DT<T>::from_float(acc[4 * j + 2] + rb1 + b0);
            if (two) y1[n + 1] = DT<T>::from_float(acc[4 * j + 3] + rb1 + b1);
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_tiled() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

// row-major [rows][cols] 16-bit matrix, row pitch `ld` elements; box = 64 columns x box_rows rows, 128B swizzle
int make_map(CUtensorMap* m, int is_bf16, const void* base, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
  EncodeTiledFn enc = encode_tiled();
  if (!enc) {
    set_error("quant_gemm: cuTensorMapEncodeTiled not available from the driver");
    return VPTQ_ERR_CUDA;
  }
  cuuint64_t dims[2] = {cuuint64_t(cols), cuuint64_t(rows)};
  cuuint64_t strides[1] = {cuuint64_t(ld) * 2};
  cuuint32_t box[2] = {BK, cuuint32_t(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                   const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("quant_gemm: cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%lld ld=%lld", int(r), (long long)rows,
              (long long)cols, (long long)ld);
    return VPTQ_ERR_CUDA;
  }
  return 0;
}

struct GemmWorkspace {
  size_t off_rowbias, off_xq, off_wq, total;
  int64_t kpad;
};
GemmWorkspace gemm_layout(const vptq_linear_desc& d, int tokens) {
  GemmWorkspace w;
  w.kpad = int64_t(align_up(size_t(d.in_features), 64));  // whole BK blocks: no partially filled swizzle rows
  size_t off = kZeroRegionBytes;                         // the zero-at-rest region stays untouched
  w.off_rowbias = off;
  off += align_up(size_t(tokens) * 4, 1024);
  w.off_xq = off;
  off += align_up(size_t(tokens) * w.kpad * 2, 1024);
  w.off_wq = off;
  off += align_up(size_t(d.out_features) * w.kpad * 2, 1024);
  w.total = off;
  return w;
}

// Input gradient dX[T][I] = dY[T][O] . W: the same GEMM with A = dY, B = Wt[I][ld] (transposed dequant, K = ld
// = O rounded up to whole BK blocks, its columns [O, ld) zero).  dY goes to TMA as it is when its rows are
// 16-byte aligned whole BK blocks; otherwise it is first copied to [T][ld] with zero K padding.
struct DgradWorkspace {
  size_t off_wt, off_dy, total;
  int64_t ld;
};
DgradWorkspace dgrad_layout(const vptq_linear_desc& d, int tokens) {
  DgradWorkspace w;
  w.ld = int64_t(align_up(size_t(d.out_features), 64));
  size_t off = kZeroRegionBytes;                         // the zero-at-rest region stays untouched
  w.off_wt = off;
  off += align_up(size_t(d.in_features) * w.ld * 2, 1024);
  w.off_dy = off;
  off += align_up(size_t(tokens) * w.ld * 2, 1024);
  w.total = off;
  return w;
}

// dy rows -> pitch ld, columns [O, ld) <- 0 (16-bit payload copied as it is)
__global__ void dgrad_stage_dy(const uint16_t* __restrict__ dy, int64_t dy_stride, uint16_t* __restrict__ out,
                               int64_t ld, int O) {
  const uint16_t* src = dy + int64_t(blockIdx.x) * dy_stride;
  uint16_t* dst = out + int64_t(blockIdx.x) * ld;
  for (int64_t c = threadIdx.x; c < ld; c += blockDim.x) dst[c] = c < O ? src[c] : uint16_t(0);
}

}  // namespace

size_t gemm_workspace_bytes(const vptq_linear_desc& d, int tokens) { return gemm_layout(d, tokens).total; }

size_t dgrad_workspace_bytes(const vptq_linear_desc& d, int tokens) { return dgrad_layout(d, tokens).total; }

int dgrad_launch(const vptq_linear_desc& d, const void* dy, int64_t dy_stride, void* dx, int64_t dx_stride, int tokens,
                 void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  const DgradWorkspace w = dgrad_layout(d, tokens);
  if (!workspace || workspace_bytes < w.total) {
    set_error("quant_gemm (transpose): workspace %zu bytes < required %zu", workspace_bytes, w.total);
    return VPTQ_ERR_WORKSPACE;
  }
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  void* wt = ws + w.off_wt;
  const int is_bf16 = d.dtype == VPTQ_BF16;
  if (int rc = dequant_transposed_launch(d, wt, w.ld, stream)) return rc;
  const void* a = dy;
  int64_t a_ld = dy_stride;
  if (int64_t(d.out_features) != w.ld || (reinterpret_cast<uintptr_t>(dy) & 15u) || (dy_stride % 8)) {
    a = ws + w.off_dy, a_ld = w.ld;
    dgrad_stage_dy<<<tokens, 256, 0, stream>>>(reinterpret_cast<const uint16_t*>(dy), dy_stride,
                                                reinterpret_cast<uint16_t*>(ws + w.off_dy), w.ld, d.out_features);
  }
  CUtensorMap map_a, map_b;
  if (int rc = make_map(&map_a, is_bf16, a, tokens, w.ld, a_ld, BM)) return rc;
  if (int rc = make_map(&map_b, is_bf16, wt, d.in_features, w.ld, w.ld, BN)) return rc;
  GemmParams p{};
  p.bias = nullptr, p.rowbias = nullptr, p.y = dx, p.y_stride = dx_stride;
  p.T = tokens, p.O = d.in_features, p.K = int(w.ld), p.is_bf16 = is_bf16;
  const DeviceInfo* dev = device_info();
  if (!dev) return VPTQ_ERR_CUDA;
  const int ntiles = ((d.in_features + BN - 1) / BN) * ((tokens + BM - 1) / BM);
  dim3 grid(unsigned(std::min(ntiles, dev->sm_count)));  // persistent: one CTA per SM
  if (is_bf16) {
    if (int rc = ensure_smem_attr(reinterpret_cast<const void*>(gemm_tn_wgmma<__nv_bfloat16>), GEMM_SMEM)) return rc;
    gemm_tn_wgmma<__nv_bfloat16><<<grid, GEMM_THREADS, GEMM_SMEM, stream>>>(map_a, map_b, p);
  } else {
    if (int rc = ensure_smem_attr(reinterpret_cast<const void*>(gemm_tn_wgmma<__half>), GEMM_SMEM)) return rc;
    gemm_tn_wgmma<__half><<<grid, GEMM_THREADS, GEMM_SMEM, stream>>>(map_a, map_b, p);
  }
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("quant_gemm (transpose) launch: %s", cudaGetErrorString(e));
    return VPTQ_ERR_CUDA;
  }
  return 0;
}

int gemm_launch(const vptq_linear_desc& d, const void* x, int64_t x_stride, void* y, int64_t y_stride, int tokens,
                void* workspace, size_t workspace_bytes, uint32_t /*flags*/, cudaStream_t stream) {
  const GemmWorkspace w = gemm_layout(d, tokens);
  if (!workspace || workspace_bytes < w.total) {
    set_error("quant_gemm: workspace %zu bytes < required %zu", workspace_bytes, w.total);
    return VPTQ_ERR_WORKSPACE;
  }
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  float* rowbias = reinterpret_cast<float*>(ws + w.off_rowbias);
  void* xq = ws + w.off_xq;
  void* wq = ws + w.off_wq;
  const int is_bf16 = d.dtype == VPTQ_BF16;

  // Prep-free path: W in ORIGINAL column order with scale and weight_bias folded in (what the reference's dequant
  // returns, csrc/kernels/dequant.cuh:9-115) through the 8-columns-per-thread dequant, and x handed to TMA as it
  // is -- no x' pass over the tokens, no rowbias.  Needs whole BK blocks (in_features % 64 == 0) and TMA-able x rows.
  const bool direct = std::getenv("VPTQ_B200_GEMM_PREP") == nullptr && int64_t(d.in_features) == w.kpad &&
                      (reinterpret_cast<uintptr_t>(x) & 15u) == 0 && (x_stride % 8) == 0 &&
                      dequant_orig_fast_ok(d, ws + kZeroRegionBytes + align_up(size_t(d.in_features) * 2, 1024), w.kpad);
  if (direct) {
    void* wo = ws + kZeroRegionBytes + align_up(size_t(d.in_features) * 2, 1024);  // behind the inverse permutation
    if (int rc = dequant_launch(d, wo, workspace, workspace_bytes, stream, w.kpad)) return rc;
    CUtensorMap map_a, map_b;
    if (int rc = make_map(&map_a, is_bf16, x, tokens, w.kpad, x_stride, BM)) return rc;
    if (int rc = make_map(&map_b, is_bf16, wo, d.out_features, w.kpad, w.kpad, BN)) return rc;
    GemmParams p{};
    p.bias = d.bias, p.rowbias = nullptr, p.y = y, p.y_stride = y_stride;
    p.T = tokens, p.O = d.out_features, p.K = int(w.kpad), p.is_bf16 = is_bf16;
    const DeviceInfo* dev = device_info();
    if (!dev) return VPTQ_ERR_CUDA;
    const int ntiles = ((d.out_features + BN - 1) / BN) * ((tokens + BM - 1) / BM);
    dim3 grid(unsigned(std::min(ntiles, dev->sm_count)));
    if (is_bf16) {
      if (int rc = ensure_smem_attr(reinterpret_cast<const void*>(gemm_tn_wgmma<__nv_bfloat16>), GEMM_SMEM)) return rc;
      gemm_tn_wgmma<__nv_bfloat16><<<grid, GEMM_THREADS, GEMM_SMEM, stream>>>(map_a, map_b, p);
    } else {
      if (int rc = ensure_smem_attr(reinterpret_cast<const void*>(gemm_tn_wgmma<__half>), GEMM_SMEM)) return rc;
      gemm_tn_wgmma<__half><<<grid, GEMM_THREADS, GEMM_SMEM, stream>>>(map_a, map_b, p);
    }
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
      set_error("quant_gemm launch: %s", cudaGetErrorString(e));
      return VPTQ_ERR_CUDA;
    }
    return 0;
  }

  // 1. x' and rowbias
  const size_t prep_smem = align_up(size_t(d.in_features) * 2, 16);
  {
    if (int rc = ensure_smem_attr(reinterpret_cast<const void*>(prefill_prep_x<__half>), 132 * 1024)) return rc;
    if (int rc = ensure_smem_attr(reinterpret_cast<const void*>(prefill_prep_x<__nv_bfloat16>), 132 * 1024)) return rc;
  }
  if (is_bf16)
    prefill_prep_x<__nv_bfloat16><<<tokens, 256, prep_smem, stream>>>(
        reinterpret_cast<const __nv_bfloat16*>(x), x_stride, d.perm,
        reinterpret_cast<const __nv_bfloat16*>(d.weight_scale), reinterpret_cast<const __nv_bfloat16*>(d.weight_scale_q),
        reinterpret_cast<const __nv_bfloat16*>(d.weight_bias), reinterpret_cast<__nv_bfloat16*>(xq), w.kpad, rowbias,
        d.in_features);
  else
    prefill_prep_x<__half><<<tokens, 256, prep_smem, stream>>>(
        reinterpret_cast<const __half*>(x), x_stride, d.perm, reinterpret_cast<const __half*>(d.weight_scale),
        reinterpret_cast<const __half*>(d.weight_scale_q), reinterpret_cast<const __half*>(d.weight_bias),
        reinterpret_cast<__half*>(xq), w.kpad, rowbias, d.in_features);
  // 2. Wq in quantised column order (no scale / bias / perm)
  if (int rc = dequant_quant_order_launch(d, wq, w.kpad, stream)) return rc;
  // 3. tensor-core GEMM
  CUtensorMap map_a, map_b;
  if (int rc = make_map(&map_a, is_bf16, xq, tokens, w.kpad, w.kpad, BM)) return rc;
  if (int rc = make_map(&map_b, is_bf16, wq, d.out_features, w.kpad, w.kpad, BN)) return rc;
  GemmParams p{};
  p.bias = d.bias, p.rowbias = rowbias, p.y = y, p.y_stride = y_stride;
  p.T = tokens, p.O = d.out_features, p.K = int(w.kpad), p.is_bf16 = is_bf16;
  const DeviceInfo* dev = device_info();
  if (!dev) return VPTQ_ERR_CUDA;
  const int ntiles = ((d.out_features + BN - 1) / BN) * ((tokens + BM - 1) / BM);
  dim3 grid(unsigned(std::min(ntiles, dev->sm_count)));  // persistent: one CTA per SM
  cudaError_t e;
  if (is_bf16) {
    if (int rc = ensure_smem_attr(reinterpret_cast<const void*>(gemm_tn_wgmma<__nv_bfloat16>), GEMM_SMEM)) return rc;
    gemm_tn_wgmma<__nv_bfloat16><<<grid, GEMM_THREADS, GEMM_SMEM, stream>>>(map_a, map_b, p);
  } else {
    if (int rc = ensure_smem_attr(reinterpret_cast<const void*>(gemm_tn_wgmma<__half>), GEMM_SMEM)) return rc;
    gemm_tn_wgmma<__half><<<grid, GEMM_THREADS, GEMM_SMEM, stream>>>(map_a, map_b, p);
  }
  e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("quant_gemm launch: %s", cudaGetErrorString(e));
    return VPTQ_ERR_CUDA;
  }
  return 0;
}

}  // namespace vptq_b200
