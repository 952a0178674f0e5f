// Dequantise a VPTQ layer to a dense [out_features][in_features] 16-bit matrix in ORIGINAL column
// order with weight_scale / weight_bias applied -- the tensor the reference's `dequant` op returns
// (csrc/dequant.cu:227-287, kernel csrc/kernels/dequant.cuh:9-115; python spec
// vptq/ops/quant_gemm.py:43-158).
//
// Thread mapping: a thread owns two adjacent ORIGINAL columns f, f+1 of one index row, so a warp
// stores 128 contiguous bytes per output row (the reference stores one 2-byte element per thread
// and row).  (C + R) * scale + bias is evaluated in fp32 and rounded once.
#include <algorithm>
#include <mutex>

#include "common.cuh"
#include "kernels.h"

namespace vptq_b200 {

namespace {

struct DequantParams {
  const uint32_t* indices;
  int64_t idx_stride_g, idx_stride_r;
  const void* centroids;
  int64_t cb_stride;
  const void* res_centroids;
  int64_t rcb_stride;
  const uint16_t* outlier_idx;
  const void* outlier_cb;
  const uint16_t* inv_perm;  // [I] or nullptr
  const void* scale;
  const void* wbias;
  void* out;
  int64_t ld;       // output row pitch in elements
  int quant_order;  // 1: columns stay in quantised order, no scale / bias (tensor-core operand of the prefill GEMM);
                    //    columns [I, ld) are zero-filled
  int I, O, Ro, G, gs, S, vol;
  int ib, rb;
  // transposed kernels only
  const uint16_t* perm;    // [I] quantised column -> original feature, or nullptr
  const void* scale_q;     // weight_scale / weight_bias in quantised column order, or nullptr
  const void* wbias_q;
};

__global__ void invert_perm_kernel(const uint16_t* __restrict__ perm, uint16_t* __restrict__ inv, int n) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < n) inv[perm[c]] = uint16_t(c);
}

template <typename T, int V>
__global__ void __launch_bounds__(256) dequant_kernel(const __grid_constant__ DequantParams p) {
  const int r = blockIdx.y;
  const int fbase = (blockIdx.x * blockDim.x + threadIdx.x) * 2;
  const int ncols = p.quant_order ? int(p.ld) : p.I;
  if (fbase >= ncols) return;
  const T* scale = reinterpret_cast<const T*>(p.scale);
  const T* wbias = reinterpret_cast<const T*>(p.wbias);
  const int b = p.ib + p.rb;
  const uint32_t fmask = b >= 32 ? 0xffffffffu : ((1u << b) - 1u);
  const uint64_t pol = policy_evict_last();

  float val[2][V];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int f = fbase + h;
    if (f >= p.I) {
#pragma unroll
      for (int e = 0; e < V; ++e) val[h][e] = 0.f;
      continue;
    }
    const int c = (p.inv_perm && !p.quant_order) ? int(p.inv_perm[f]) : f;
    const float sc = (scale && !p.quant_order) ? DT<T>::to_float(scale[f]) : 1.f;
    const float wb = (wbias && !p.quant_order) ? DT<T>::to_float(wbias[f]) : 0.f;
    if (c < p.S) {  // outlier column: its own codebook with vector length `vol`
      const T* ocb = reinterpret_cast<const T*>(p.outlier_cb);
#pragma unroll
      for (int e = 0; e < V; ++e) {
        const int o = r * V + e;
        float w = 0.f;
        if (o < p.O) {
          const int rol = o / p.vol, eo = o - rol * p.vol;
          const int oi = p.outlier_idx[int64_t(rol) * p.S + c];
          w = DT<T>::to_float(ocb[int64_t(oi) * p.vol + eo]);
        }
        val[h][e] = fmaf(w, sc, wb);
      }
    } else {
      const int ci = c - p.S;
      const int g = ci / p.gs, j = ci - g * p.gs;
      const uint32_t* row = p.indices + int64_t(g) * p.idx_stride_g + int64_t(r) * p.idx_stride_r;
      const uint32_t bit = uint32_t(j) * uint32_t(b);
      const uint32_t w0 = bit >> 5, sh = bit & 31u;
      const uint32_t lo = ldg_nc_u32(row + w0);
      const uint32_t hi = (sh + b > 32) ? ldg_nc_u32(row + w0 + 1) : 0u;  // never reads past the row
      const uint32_t field = __funnelshift_r(lo, hi, sh) & fmask;
      const uint32_t mi = field & ((1u << p.ib) - 1u), ri = field >> p.ib;
      uint32_t cw[V / 2];
      ldg_entry<V>(cw, reinterpret_cast<const T*>(p.centroids) + int64_t(g) * p.cb_stride + size_t(mi) * V, pol);
      float w[V];
#pragma unroll
      for (int i = 0; i < V / 2; ++i) {
        const float2 t = DT<T>::unpack2(cw[i]);
        w[2 * i] = t.x, w[2 * i + 1] = t.y;
      }
      if (p.rb) {
        uint32_t rw[V / 2];
        ldg_entry<V>(rw, reinterpret_cast<const T*>(p.res_centroids) + int64_t(g) * p.rcb_stride + size_t(ri) * V, pol);
#pragma unroll
        for (int i = 0; i < V / 2; ++i) {
          const float2 t = DT<T>::unpack2(rw[i]);
          w[2 * i] += t.x, w[2 * i + 1] += t.y;
        }
      }
#pragma unroll
      for (int e = 0; e < V; ++e) val[h][e] = fmaf(w[e], sc, wb);
    }
  }

  T* out = reinterpret_cast<T*>(p.out);
  const bool pair = (fbase + 1 < ncols) && ((p.ld & 1) == 0);
#pragma unroll
  for (int e = 0; e < V; ++e) {
    const int o = r * V + e;
    if (o >= p.O) break;  // padding rows are dropped (vptq/ops/quant_gemm.py:123-124)
    T* dst = out + int64_t(o) * p.ld + fbase;
    if (pair) {
      *reinterpret_cast<uint32_t*>(dst) = DT<T>::pack2(val[0][e], val[1][e]);
    } else {
      dst[0] = DT<T>::from_float(val[0][e]);
      if (fbase + 1 < ncols) dst[1] = DT<T>::from_float(val[1][e]);
    }
  }
}


// ---------------------------------------------------------------------------------------------
// Fast path of the quantised-order dequant (the prefill GEMM's B operand), vector_len 8:
// a thread owns 8 CONSECUTIVE columns of one index row, gathers their 8 codebook entries
// (8 independent 16-byte loads in flight), adds the residual entries from a bank-replicated
// shared-memory table, transposes the 8x8 block in registers (PRMT) and writes one 16-byte
// vector per output row: every warp store covers 512 contiguous bytes.
// ---------------------------------------------------------------------------------------------
constexpr int DQ_ROWS = 8, DQ_COLS = 1024, DQ_THREADS = 256;

template <typename T>
__global__ void __launch_bounds__(DQ_THREADS) dequant_q8_kernel(const __grid_constant__ DequantParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int b = p.ib + p.rb;
  const int chunks_per_group = (p.gs + DQ_COLS - 1) / DQ_COLS;
  const int g = blockIdx.x / chunks_per_group, ch = blockIdx.x % chunks_per_group;
  const int j0 = ch * DQ_COLS;                         // first column of the chunk inside its group
  const int ncols = min(DQ_COLS, p.gs - j0);           // multiple of 8
  const int r0 = blockIdx.y * DQ_ROWS;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t row_words = (uint32_t(DQ_COLS) * b + 31) / 32 + 4;  // per staged row, padded
  uint32_t* s_idx = reinterpret_cast<uint32_t*>(smem);               // [DQ_ROWS][row_words]
  uint8_t* s_res = smem + ((DQ_ROWS * row_words * 4 + 127) & ~127u); // replicated residual table
  __shared__ uint64_t bar;

  const uint32_t* idx_g = p.indices + int64_t(g) * p.idx_stride_g;
  const int nw = (ncols * b + 31) >> 5;
  const int64_t w0 = (int64_t(j0) * b) >> 5;  // j0 is a multiple of 1024: word aligned
  const bool tma_ok = ((reinterpret_cast<uintptr_t>(idx_g) & 15u) == 0) && ((p.idx_stride_r & 3) == 0) && ((nw & 3) == 0);
  if (tid == 0) {
    mbar_init(&bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  const uint64_t pol = policy_evict_first();
  if (tma_ok) {
    if (tid == 0) {
      int rows = min(DQ_ROWS, p.Ro - r0);
      mbar_arrive_expect_tx(&bar, uint32_t(rows) * uint32_t(nw) * 4u);
      for (int i = 0; i < rows; ++i)
        tma_bulk_g2s(s_idx + i * row_words, idx_g + int64_t(r0 + i) * p.idx_stride_r + w0, uint32_t(nw) * 4u, &bar, pol);
    }
  } else {
    for (int i = 0; i < DQ_ROWS && r0 + i < p.Ro; ++i)
      for (int w = tid; w < nw; w += DQ_THREADS) s_idx[i * row_words + w] = ldg_nc_u32(idx_g + int64_t(r0 + i) * p.idx_stride_r + w0 + w);
  }
  // residual table: 8 copies of every 16-byte entry, copy k at slot i*8+k (lane L reads copy L&7)
  const T* rcb = p.rb ? reinterpret_cast<const T*>(p.res_centroids) + int64_t(g) * p.rcb_stride : nullptr;
  const int Kr = p.rb ? (1 << p.rb) : 0;
  for (int e = tid; e < Kr; e += DQ_THREADS) {
    const uint4 v = ldg_nc_v4(reinterpret_cast<const uint8_t*>(rcb) + size_t(e) * 16, policy_evict_last());
#pragma unroll
    for (int c = 0; c < 8; ++c) sts_v4(smem_u32(s_res) + (e * 8 + c) * 16, v);
  }
  __syncthreads();
  if (tma_ok) mbar_wait(&bar, 0);

  const int r = r0 + warp;
  if (r >= p.Ro) return;
  const uint32_t fmask = b >= 32 ? 0xffffffffu : ((1u << b) - 1u), imask = (1u << p.ib) - 1u;
  const uint32_t* sw = s_idx + warp * row_words;
  const uint8_t* cb = reinterpret_cast<const uint8_t*>(reinterpret_cast<const T*>(p.centroids) + int64_t(g) * p.cb_stride);
  const uint32_t res_lane = smem_u32(s_res) + (lane & 7) * 16;
  const uint64_t keep = policy_evict_last();
  T* out = reinterpret_cast<T*>(p.out);
  const int col_base = p.S + g * p.gs + j0;  // quantised column of the chunk's first field

  for (int jc = lane * 8; jc < ncols; jc += 32 * 8) {
    uint32_t fld[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const uint32_t bit = uint32_t(jc + k) * uint32_t(b), w = bit >> 5;
      fld[k] = __funnelshift_r(sw[w], sw[w + 1], bit & 31u) & fmask;
    }
    uint4 cw[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) cw[k] = ldg_nc_v4(cb + size_t(fld[k] & imask) * 16, keep);
    if (p.rb) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const uint4 rw = lds_v4(res_lane + (fld[k] >> p.ib) * 128);
        cw[k].x = DT<T>::add2(cw[k].x, rw.x), cw[k].y = DT<T>::add2(cw[k].y, rw.y);
        cw[k].z = DT<T>::add2(cw[k].z, rw.z), cw[k].w = DT<T>::add2(cw[k].w, rw.w);
      }
    }
    // 8x8 transpose: output row e takes element e of each of the 8 entries
    const uint32_t* cwp = reinterpret_cast<const uint32_t*>(cw);  // cw[k] word i = cwp[4*k + i]
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int o = r * 8 + e;
      if (o < p.O) {
        const uint32_t sel = (e & 1) ? 0x7632u : 0x5410u;
        uint4 v;
        v.x = __byte_perm(cwp[4 * 0 + (e >> 1)], cwp[4 * 1 + (e >> 1)], sel);
        v.y = __byte_perm(cwp[4 * 2 + (e >> 1)], cwp[4 * 3 + (e >> 1)], sel);
        v.z = __byte_perm(cwp[4 * 4 + (e >> 1)], cwp[4 * 5 + (e >> 1)], sel);
        v.w = __byte_perm(cwp[4 * 6 + (e >> 1)], cwp[4 * 7 + (e >> 1)], sel);
        *reinterpret_cast<uint4*>(out + int64_t(o) * p.ld + col_base + jc) = v;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Fast path of the ORIGINAL-order dequant (the reference op, and the B operand of the prep-free prefill
// path), vector_len 8, one codebook group, no outlier columns: one CTA per index row.  The row's packed
// words are staged in shared memory once (TMA), the residual table is bank-replicated there; a thread
// owns 8 CONSECUTIVE ORIGINAL columns f..f+7: it looks up their quantised columns (inverse permutation,
// one 16-byte load), extracts the 8 fields from the staged row (any bit offset), gathers the 8 codebook
// entries (8 independent 16-byte loads in flight; the generic kernel has two), applies
// (C + R) * scale[f] + wbias[f] in fp32, rounds once, transposes the 8x8 block in registers and writes one
// 16-byte vector per output row: every warp store covers 512 contiguous bytes.
// ---------------------------------------------------------------------------------------------
constexpr int DO_THREADS = 256;

template <typename T>
__global__ void __launch_bounds__(DO_THREADS) dequant_o8_kernel(const __grid_constant__ DequantParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int b = p.ib + p.rb;
  const int r = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31;
  const int nw = (p.I * b + 31) >> 5;                    // packed words of one row
  const uint32_t row_bytes = (uint32_t(nw) * 4u + 8u + 127u) & ~127u;  // (+ one readable pad word)
  uint32_t* s_idx = reinterpret_cast<uint32_t*>(smem);
  uint8_t* s_res = smem + row_bytes;
  __shared__ uint64_t bar;
  const uint32_t* row = p.indices + int64_t(r) * p.idx_stride_r;
  const bool tma_ok = ((reinterpret_cast<uintptr_t>(row) & 15u) == 0) && ((nw & 3) == 0);
  if (tid == 0) {
    mbar_init(&bar, 1);
    fence_mbar_init();
    s_idx[nw] = 0u, s_idx[nw + 1] = 0u;
  }
  __syncthreads();
  if (tma_ok) {
    if (tid == 0) {
      mbar_arrive_expect_tx(&bar, uint32_t(nw) * 4u);
      for (uint32_t off = 0; off < uint32_t(nw) * 4u; off += 32768u)
        tma_bulk_g2s(reinterpret_cast<uint8_t*>(s_idx) + off, reinterpret_cast<const uint8_t*>(row) + off,
                     min(32768u, uint32_t(nw) * 4u - off), &bar, policy_evict_first());
    }
  } else {
    for (int w = tid; w < nw; w += DO_THREADS) s_idx[w] = ldg_nc_u32(row + w);
  }
  const T* rcb = reinterpret_cast<const T*>(p.res_centroids);
  const int Kr = p.rb ? (1 << p.rb) : 0;
  for (int slot = tid; slot < Kr * 8; slot += DO_THREADS)   // copy k of entry i at slot i*8+k: conflict-free fill
    sts_v4(smem_u32(s_res) + uint32_t(slot) * 16u,
           ldg_nc_v4(reinterpret_cast<const uint8_t*>(rcb) + size_t(slot >> 3) * 16, policy_evict_last()));
  __syncthreads();
  if (tma_ok) mbar_wait(&bar, 0);

  const uint32_t fmask = b >= 32 ? 0xffffffffu : ((1u << b) - 1u), imask = (1u << p.ib) - 1u;
  const uint8_t* cb = reinterpret_cast<const uint8_t*>(p.centroids);
  const uint32_t res_lane = smem_u32(s_res) + (lane & 7) * 16;
  const uint64_t keep = policy_evict_last();
  const T* scale = reinterpret_cast<const T*>(p.scale);
  const T* wbias = reinterpret_cast<const T*>(p.wbias);
  T* out = reinterpret_cast<T*>(p.out);

  for (int f0 = tid * 8; f0 < p.I; f0 += DO_THREADS * 8) {   // (I % 8 == 0)
    uint32_t col[8];
    if (p.inv_perm) {
      const uint4 q = *reinterpret_cast<const uint4*>(p.inv_perm + f0);
      col[0] = q.x & 0xffffu, col[1] = q.x >> 16, col[2] = q.y & 0xffffu, col[3] = q.y >> 16;
      col[4] = q.z & 0xffffu, col[5] = q.z >> 16, col[6] = q.w & 0xffffu, col[7] = q.w >> 16;
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) col[k] = uint32_t(f0 + k);
    }
    uint32_t fld[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const uint32_t bit = col[k] * uint32_t(b), w = bit >> 5;
      fld[k] = __funnelshift_r(s_idx[w], s_idx[w + 1], bit & 31u) & fmask;
    }
    uint4 cw[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) cw[k] = ldg_nc_v4(cb + size_t(fld[k] & imask) * 16, keep);
    uint4 scv = make_uint4(0u, 0u, 0u, 0u), wbv = scv;
    if (scale) {
      scv = *reinterpret_cast<const uint4*>(scale + f0);
      wbv = *reinterpret_cast<const uint4*>(wbias + f0);
    }
    const uint32_t scw[4] = {scv.x, scv.y, scv.z, scv.w}, wbw[4] = {wbv.x, wbv.y, wbv.z, wbv.w};
    uint32_t hv[8][4];  // column k, outputs (2i, 2i+1) packed -- after scale / bias, rounded once
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      uint4 rw = make_uint4(0u, 0u, 0u, 0u);
      if (p.rb) rw = lds_v4(res_lane + (fld[k] >> p.ib) * 128);
      const float2 s2 = DT<T>::unpack2(scw[k >> 1]), b2 = DT<T>::unpack2(wbw[k >> 1]);
      const float sc = scale ? ((k & 1) ? s2.y : s2.x) : 1.f, wb = scale ? ((k & 1) ? b2.y : b2.x) : 0.f;
      const uint32_t cwk[4] = {cw[k].x, cw[k].y, cw[k].z, cw[k].w}, rwk[4] = {rw.x, rw.y, rw.z, rw.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float2 c2 = DT<T>::unpack2(cwk[i]);
        if (p.rb) {
          const float2 r2 = DT<T>::unpack2(rwk[i]);
          c2.x += r2.x, c2.y += r2.y;
        }
        hv[k][i] = DT<T>::pack2(fmaf(c2.x, sc, wb), fmaf(c2.y, sc, wb));
      }
    }
    // 8x8 transpose: output row e takes element e of each of the 8 columns
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int o = r * 8 + e;
      if (o < p.O) {
        const uint32_t sel = (e & 1) ? 0x7632u : 0x5410u;
        uint4 v;
        v.x = __byte_perm(hv[0][e >> 1], hv[1][e >> 1], sel);
        v.y = __byte_perm(hv[2][e >> 1], hv[3][e >> 1], sel);
        v.z = __byte_perm(hv[4][e >> 1], hv[5][e >> 1], sel);
        v.w = __byte_perm(hv[6][e >> 1], hv[7][e >> 1], sel);
        *reinterpret_cast<uint4*>(out + int64_t(o) * p.ld + f0) = v;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// TRANSPOSED dequant, the B operand of the input-gradient GEMM (dX = dY . W):
//   Wt[f][o] = W[o][f] = weight_scale[f] * (C[idx] + R[ridx])[o % v] + weight_bias[f]
// rows in ORIGINAL feature order, row pitch ld >= O, columns [O, ld) zero (padding rows of the last index row
// and the K tail of the GEMM: zeros, not garbage, because 0 * garbage can be NaN).  Same fp32 arithmetic as
// the original-order kernels, rounded once, so Wt is bit-identical to the transpose of what dequant returns.
// With vector_quant_dim "out" one codebook entry holds v consecutive outputs of one input feature, i.e. v
// consecutive elements of one Wt row: the entry is stored as it is, no register transpose.
// ---------------------------------------------------------------------------------------------

// Fast path: v = 8, one codebook group, no outlier columns.  A CTA owns 32 index rows (one per lane) x 256
// quantised columns: the rows' packed words are staged in shared memory (bulk copies), the residual table is
// bank-replicated there.  A warp takes DT_UNROLL columns at a time; lane L handles index row r0 + L: it
// extracts the field (any b <= 32), gathers C (L2) and R (shared memory), applies scale / weight_bias of
// feature perm[c] and stores one 16-byte vector at Wt[perm[c]][8 (r0 + L)] -- a warp store covers 512
// contiguous bytes.  Index rows past Ro (up to ld / 8) store zeros.
constexpr int DT_ROWS = 32, DT_COLS = 256, DT_THREADS = 256, DT_UNROLL = 4;

template <typename T>
__global__ void __launch_bounds__(DT_THREADS) dequant_t8_kernel(const __grid_constant__ DequantParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int b = p.ib + p.rb;
  const int j0 = blockIdx.x * DT_COLS;                  // first quantised column of the chunk (gs == I)
  const int ncols = min(DT_COLS, p.gs - j0);
  const int r0 = blockIdx.y * DT_ROWS;
  const int rows = max(0, min(DT_ROWS, p.Ro - r0));     // index rows that carry packed words
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t row_words = uint32_t(DT_COLS) * b / 32 + 4;            // per staged row (+ readable pad word)
  uint32_t* s_idx = reinterpret_cast<uint32_t*>(smem);                  // [DT_ROWS][row_words]
  uint8_t* s_res = smem + ((DT_ROWS * row_words * 4 + 127) & ~127u);    // replicated residual table
  __shared__ uint64_t bar;

  const int nw = (ncols * b + 31) >> 5;
  const int64_t w0 = (int64_t(j0) * b) >> 5;            // j0 * b is a multiple of 256: 32-byte aligned
  const bool tma_ok = rows > 0 && ((reinterpret_cast<uintptr_t>(p.indices) & 15u) == 0) &&
                      ((p.idx_stride_r & 3) == 0) && ((nw & 3) == 0);
  if (tid == 0) {
    mbar_init(&bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (tma_ok) {
    if (tid == 0) {
      mbar_arrive_expect_tx(&bar, uint32_t(rows) * uint32_t(nw) * 4u);
      for (int i = 0; i < rows; ++i)
        tma_bulk_g2s(s_idx + i * row_words, p.indices + int64_t(r0 + i) * p.idx_stride_r + w0, uint32_t(nw) * 4u, &bar,
                     policy_evict_first());
    }
  } else {
    for (int i = 0; i < rows; ++i)
      for (int w = tid; w < nw; w += DT_THREADS) s_idx[i * row_words + w] = ldg_nc_u32(p.indices + int64_t(r0 + i) * p.idx_stride_r + w0 + w);
  }
  const int Kr = (p.rb && rows > 0) ? (1 << p.rb) : 0;
  for (int slot = tid; slot < Kr * 8; slot += DT_THREADS)   // copy k of entry i at slot i*8+k: conflict-free fill
    sts_v4(smem_u32(s_res) + uint32_t(slot) * 16u,
           ldg_nc_v4(reinterpret_cast<const uint8_t*>(p.res_centroids) + size_t(slot >> 3) * 16, policy_evict_last()));
  __syncthreads();
  if (tma_ok) mbar_wait(&bar, 0);

  const uint32_t fmask = b >= 32 ? 0xffffffffu : ((1u << b) - 1u), imask = (1u << p.ib) - 1u;
  const uint8_t* cb = reinterpret_cast<const uint8_t*>(p.centroids);
  const uint32_t res_lane = smem_u32(s_res) + (lane & 7) * 16;
  const uint64_t keep = policy_evict_last();
  const T* scale = reinterpret_cast<const T*>(p.scale_q ? p.scale_q : p.scale);
  const T* wbias = reinterpret_cast<const T*>(p.scale_q ? p.wbias_q : p.wbias);
  T* out = reinterpret_cast<T*>(p.out);
  const int o0 = (r0 + lane) * 8;
  const bool live = lane < rows, stored = o0 < p.ld;    // ld % 8 == 0: a vector is wholly inside or outside
  const uint32_t* sw = s_idx + lane * row_words;

  for (int jc = warp * DT_UNROLL; jc < ncols; jc += (DT_THREADS / 32) * DT_UNROLL) {
    uint32_t fld[DT_UNROLL];
#pragma unroll
    for (int k = 0; k < DT_UNROLL; ++k) {
      const uint32_t bit = uint32_t(jc + k) * uint32_t(b), w = bit >> 5;
      fld[k] = (live && jc + k < ncols) ? (__funnelshift_r(sw[w], sw[w + 1], bit & 31u) & fmask) : 0u;
    }
    uint4 cw[DT_UNROLL];
#pragma unroll
    for (int k = 0; k < DT_UNROLL; ++k) cw[k] = live ? ldg_nc_v4(cb + size_t(fld[k] & imask) * 16, keep) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
    for (int k = 0; k < DT_UNROLL; ++k) {
      const int c = j0 + jc + k;
      if (c >= j0 + ncols) break;
      const int f = p.perm ? int(p.perm[c]) : c;
      const int sf = p.scale_q ? c : f;                 // scale_q / wbias_q are indexed by the quantised column
      const float sc = scale ? DT<T>::to_float(scale[sf]) : 1.f, wb = scale ? DT<T>::to_float(wbias[sf]) : 0.f;
      uint4 rw = make_uint4(0u, 0u, 0u, 0u);
      if (p.rb && live) rw = lds_v4(res_lane + (fld[k] >> p.ib) * 128);
      const uint32_t cwk[4] = {cw[k].x, cw[k].y, cw[k].z, cw[k].w}, rwk[4] = {rw.x, rw.y, rw.z, rw.w};
      uint32_t hv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float2 c2 = DT<T>::unpack2(cwk[i]);
        if (p.rb) {
          const float2 r2 = DT<T>::unpack2(rwk[i]);
          c2.x += r2.x, c2.y += r2.y;
        }
        hv[i] = DT<T>::pack2(fmaf(c2.x, sc, wb), fmaf(c2.y, sc, wb));
        const int o = o0 + 2 * i;                       // outputs o, o + 1 past O (or a row past Ro): zeros
        if (!live || o >= p.O) hv[i] = 0u;
        else if (o + 1 >= p.O) hv[i] &= 0xffffu;
      }
      if (stored) *reinterpret_cast<uint4*>(out + int64_t(f) * p.ld + o0) = make_uint4(hv[0], hv[1], hv[2], hv[3]);
    }
  }
}

// Generic transposed path: every other layer (v in {2, 4, ..., 16}, several groups, outlier columns with their
// own codebook and vector length, no perm / no norm).  A thread owns one quantised column c -- the warp's field
// reads are adjacent -- and walks the index rows; it writes v elements of row perm[c] of Wt per index row.
template <typename T, int V>
__global__ void __launch_bounds__(256) dequant_t_kernel(const __grid_constant__ DequantParams p) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= p.I) return;
  const int f = p.perm ? int(p.perm[c]) : c;
  const T* scale = reinterpret_cast<const T*>(p.scale);
  const T* wbias = reinterpret_cast<const T*>(p.wbias);
  const float sc = scale ? DT<T>::to_float(scale[f]) : 1.f;
  const float wb = wbias ? DT<T>::to_float(wbias[f]) : 0.f;
  const int b = p.ib + p.rb;
  const uint32_t fmask = b >= 32 ? 0xffffffffu : ((1u << b) - 1u);
  const uint64_t pol = policy_evict_last();
  const int nrows = int((p.ld + V - 1) / V);            // index rows past Ro only write the zero K tail
  T* dst = reinterpret_cast<T*>(p.out) + int64_t(f) * p.ld;
  for (int r = blockIdx.y; r < nrows; r += gridDim.y) {
    float w[V];
    if (r >= p.Ro) {
#pragma unroll
      for (int e = 0; e < V; ++e) w[e] = 0.f;
    } else if (c < p.S) {  // outlier column: its own codebook with vector length `vol`
      const T* ocb = reinterpret_cast<const T*>(p.outlier_cb);
#pragma unroll
      for (int e = 0; e < V; ++e) {
        const int o = r * V + e;
        w[e] = 0.f;
        if (o < p.O) {
          const int rol = o / p.vol, eo = o - rol * p.vol;
          const int oi = p.outlier_idx[int64_t(rol) * p.S + c];
          w[e] = DT<T>::to_float(ocb[int64_t(oi) * p.vol + eo]);
        }
      }
    } else {
      const int ci = c - p.S;
      const int g = ci / p.gs, j = ci - g * p.gs;
      const uint32_t* row = p.indices + int64_t(g) * p.idx_stride_g + int64_t(r) * p.idx_stride_r;
      const uint32_t bit = uint32_t(j) * uint32_t(b);
      const uint32_t w0 = bit >> 5, sh = bit & 31u;
      const uint32_t lo = ldg_nc_u32(row + w0);
      const uint32_t hi = (sh + b > 32) ? ldg_nc_u32(row + w0 + 1) : 0u;  // never reads past the row
      const uint32_t field = __funnelshift_r(lo, hi, sh) & fmask;
      const uint32_t mi = field & ((1u << p.ib) - 1u), ri = field >> p.ib;
      uint32_t cw[V / 2];
      ldg_entry<V>(cw, reinterpret_cast<const T*>(p.centroids) + int64_t(g) * p.cb_stride + size_t(mi) * V, pol);
#pragma unroll
      for (int i = 0; i < V / 2; ++i) {
        const float2 t = DT<T>::unpack2(cw[i]);
        w[2 * i] = t.x, w[2 * i + 1] = t.y;
      }
      if (p.rb) {
        uint32_t rw[V / 2];
        ldg_entry<V>(rw, reinterpret_cast<const T*>(p.res_centroids) + int64_t(g) * p.rcb_stride + size_t(ri) * V, pol);
#pragma unroll
        for (int i = 0; i < V / 2; ++i) {
          const float2 t = DT<T>::unpack2(rw[i]);
          w[2 * i] += t.x, w[2 * i + 1] += t.y;
        }
      }
    }
#pragma unroll
    for (int e = 0; e < V; ++e) {
      const int o = r * V + e;
      if (o >= p.ld) break;
      dst[o] = DT<T>::from_float(o < p.O ? fmaf(w[e], sc, wb) : 0.f);
    }
  }
}

// columns [I, ld) of every output row <- 0 (K padding of the GEMM operand)
template <typename T>
__global__ void dequant_zero_pad_kernel(T* out, int64_t ld, int I, int O) {
  const int o = blockIdx.x;
  for (int64_t c = I + threadIdx.x; c < ld; c += blockDim.x) out[int64_t(o) * ld + c] = DT<T>::from_float(0.f);
}

template <typename T>
int launch_v(const DequantParams& p, int v, cudaStream_t stream) {
  const int ncols = p.quant_order ? int(p.ld) : p.I;
  dim3 block(256), grid(unsigned((ncols + 511) / 512), unsigned(p.Ro));
  switch (v) {
#define VPTQ_CASE(VV) \
  case VV: dequant_kernel<T, VV><<<grid, block, 0, stream>>>(p); break;
    VPTQ_CASE(2) VPTQ_CASE(4) VPTQ_CASE(6) VPTQ_CASE(8) VPTQ_CASE(10) VPTQ_CASE(12) VPTQ_CASE(16)
#undef VPTQ_CASE
    default: set_error("dequant: vector_len %d not supported", v); return VPTQ_ERR_UNSUPPORTED;
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("dequant launch: %s", cudaGetErrorString(e));
    return VPTQ_ERR_CUDA;
  }
  return 0;
}

}  // namespace

size_t dequant_workspace_bytes(const vptq_linear_desc& d) {
  // the inverse permutation is scratch: it goes behind the zero-at-rest counter region
  return d.perm ? kZeroRegionBytes + align_up(size_t(d.in_features) * 2, 256) : 0;
}

// v = 8, one codebook group, no outlier columns, whole 8-column groups, 16-byte aligned rows, the packed row +
// the replicated residual table fit in shared memory
bool dequant_orig_fast_ok(const vptq_linear_desc& d, const void* w_out, int64_t ld) {
  const bool outl = d.outlier_size > 0 && d.outlier_indices != nullptr;
  if (d.vector_len != 8 || d.num_codebooks != 1 || outl || (d.in_features % 8) || (ld % 8)) return false;
  if ((reinterpret_cast<uintptr_t>(w_out) & 15u) || (reinterpret_cast<uintptr_t>(d.weight_scale) & 15u) ||
      (reinterpret_cast<uintptr_t>(d.weight_bias) & 15u))
    return false;
  const int b = ilog2(d.num_centroids) + (d.num_res_centroids > 0 ? ilog2(d.num_res_centroids) : 0);
  const size_t row = (size_t(d.in_features) * b + 31) / 32 * 4 + 136;
  const size_t res = d.num_res_centroids > 0 ? size_t(d.num_res_centroids) * 128 : 0;
  return d.num_res_centroids <= 512 && row + res <= 190 * 1024;
}

int dequant_launch(const vptq_linear_desc& d, void* w_out, void* workspace, size_t workspace_bytes,
                   cudaStream_t stream, int64_t ld) {
  DequantParams p{};
  p.indices = reinterpret_cast<const uint32_t*>(d.indices);
  p.idx_stride_g = d.index_stride_codebook, p.idx_stride_r = d.index_stride_row;
  p.centroids = d.centroids, p.cb_stride = d.centroid_stride;
  p.res_centroids = d.res_centroids, p.rcb_stride = d.res_centroid_stride;
  p.I = d.in_features, p.O = d.out_features, p.G = d.num_codebooks, p.gs = d.group_size;
  p.Ro = (d.out_features + d.vector_len - 1) / d.vector_len;
  p.ib = ilog2(d.num_centroids);
  p.rb = d.num_res_centroids > 0 ? ilog2(d.num_res_centroids) : 0;
  p.S = (d.outlier_size > 0 && d.outlier_indices) ? d.outlier_size : 0;
  p.vol = p.S ? d.outlier_vector_len : 1;
  p.outlier_idx = p.S ? d.outlier_indices : nullptr;
  p.outlier_cb = p.S ? d.outlier_centroids : nullptr;
  p.scale = d.weight_scale, p.wbias = d.weight_bias;
  p.out = w_out;
  p.ld = ld > 0 ? ld : d.in_features;
  p.quant_order = 0;
  p.inv_perm = nullptr;
  if (d.perm) {
    const size_t need = dequant_workspace_bytes(d);
    if (!workspace || workspace_bytes < need) {
      set_error("dequant: workspace %zu bytes < required %zu (inverse permutation)", workspace_bytes, need);
      return VPTQ_ERR_WORKSPACE;
    }
    uint16_t* inv = reinterpret_cast<uint16_t*>(reinterpret_cast<uint8_t*>(workspace) + kZeroRegionBytes);  // (256-byte aligned)
    invert_perm_kernel<<<(d.in_features + 255) / 256, 256, 0, stream>>>(d.perm, inv, d.in_features);
    p.inv_perm = inv;
  }
  p.ld = ld > 0 ? ld : d.in_features;
  if (dequant_orig_fast_ok(d, w_out, p.ld)) {
    const int b = p.ib + p.rb;
    const size_t nw = (size_t(d.in_features) * b + 31) / 32;
    const size_t smem = ((nw * 4 + 8 + 127) & ~size_t(127)) + (p.rb ? (size_t(1) << p.rb) * 128 : 0);
    dim3 grid(unsigned(p.Ro));
    if (d.dtype == VPTQ_FP16) {
      if (int rc = ensure_smem_attr(reinterpret_cast<const void*>(dequant_o8_kernel<__half>), 200 * 1024)) return rc;
      dequant_o8_kernel<__half><<<grid, DO_THREADS, smem, stream>>>(p);
    } else {
      if (int rc = ensure_smem_attr(reinterpret_cast<const void*>(dequant_o8_kernel<__nv_bfloat16>), 200 * 1024)) return rc;
      dequant_o8_kernel<__nv_bfloat16><<<grid, DO_THREADS, smem, stream>>>(p);
    }
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
      set_error("dequant (original order, fast path) launch: %s", cudaGetErrorString(e));
      return VPTQ_ERR_CUDA;
    }
    return 0;
  }
  const int rc = d.dtype == VPTQ_FP16 ? launch_v<__half>(p, d.vector_len, stream)
                                      : launch_v<__nv_bfloat16>(p, d.vector_len, stream);
  if (rc) return rc;
  return 0;
}

// Wq[o][c] = C[idx] + R[ridx] (outlier columns from their own codebook) in QUANTISED column order,
// row pitch `ld`, columns [I, ld) zero: the B operand of the prefill GEMM (gemm_tcgen05.cu).
int dequant_quant_order_launch(const vptq_linear_desc& d, void* wq_out, int64_t ld, cudaStream_t stream) {
  DequantParams p{};
  p.indices = reinterpret_cast<const uint32_t*>(d.indices);
  p.idx_stride_g = d.index_stride_codebook, p.idx_stride_r = d.index_stride_row;
  p.centroids = d.centroids, p.cb_stride = d.centroid_stride;
  p.res_centroids = d.res_centroids, p.rcb_stride = d.res_centroid_stride;
  p.I = d.in_features, p.O = d.out_features, p.G = d.num_codebooks, p.gs = d.group_size;
  p.Ro = (d.out_features + d.vector_len - 1) / d.vector_len;
  p.ib = ilog2(d.num_centroids);
  p.rb = d.num_res_centroids > 0 ? ilog2(d.num_res_centroids) : 0;
  p.S = (d.outlier_size > 0 && d.outlier_indices) ? d.outlier_size : 0;
  p.vol = p.S ? d.outlier_vector_len : 1;
  p.outlier_idx = p.S ? d.outlier_indices : nullptr;
  p.outlier_cb = p.S ? d.outlier_centroids : nullptr;
  p.out = wq_out, p.ld = ld, p.quant_order = 1;
  const int b = p.ib + p.rb;
  const size_t res_rep_bytes = p.rb ? (size_t(1) << p.rb) * 16 * 8 : 0;
  const bool fast = d.vector_len == 8 && p.S == 0 && (d.group_size % 8) == 0 && (ld % 8) == 0 &&
                    res_rep_bytes <= 64 * 1024 && (reinterpret_cast<uintptr_t>(wq_out) & 15u) == 0;
  if (!fast)
    return d.dtype == VPTQ_FP16 ? launch_v<__half>(p, d.vector_len, stream)
                                : launch_v<__nv_bfloat16>(p, d.vector_len, stream);
  const uint32_t row_words = (uint32_t(DQ_COLS) * b + 31) / 32 + 4;
  const size_t smem = ((size_t(DQ_ROWS) * row_words * 4 + 127) & ~size_t(127)) + res_rep_bytes;
  dim3 grid(unsigned(d.num_codebooks * ((d.group_size + DQ_COLS - 1) / DQ_COLS)), unsigned((p.Ro + DQ_ROWS - 1) / DQ_ROWS));
  if (d.dtype == VPTQ_FP16) {
    if (int rc = ensure_smem_attr(reinterpret_cast<const void*>(dequant_q8_kernel<__half>), 100 * 1024)) return rc;
    dequant_q8_kernel<__half><<<grid, DQ_THREADS, smem, stream>>>(p);
    if (ld > d.in_features)
      dequant_zero_pad_kernel<__half><<<d.out_features, 64, 0, stream>>>(reinterpret_cast<__half*>(wq_out), ld, d.in_features, d.out_features);
  } else {
    if (int rc = ensure_smem_attr(reinterpret_cast<const void*>(dequant_q8_kernel<__nv_bfloat16>), 100 * 1024)) return rc;
    dequant_q8_kernel<__nv_bfloat16><<<grid, DQ_THREADS, smem, stream>>>(p);
    if (ld > d.in_features)
      dequant_zero_pad_kernel<__nv_bfloat16><<<d.out_features, 64, 0, stream>>>(reinterpret_cast<__nv_bfloat16*>(wq_out), ld, d.in_features, d.out_features);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("dequant (quantised order) launch: %s", cudaGetErrorString(e));
    return VPTQ_ERR_CUDA;
  }
  return 0;
}

// Wt[f][o] = W[o][f] (original feature order, scale / bias folded in), row pitch `ld` (a multiple of 8, >= O),
// columns [O, ld) zero: the B operand of the input-gradient GEMM (gemm_wgmma.cu, dgrad_launch).
int dequant_transposed_launch(const vptq_linear_desc& d, void* wt_out, int64_t ld, cudaStream_t stream) {
  DequantParams p{};
  p.indices = reinterpret_cast<const uint32_t*>(d.indices);
  p.idx_stride_g = d.index_stride_codebook, p.idx_stride_r = d.index_stride_row;
  p.centroids = d.centroids, p.cb_stride = d.centroid_stride;
  p.res_centroids = d.res_centroids, p.rcb_stride = d.res_centroid_stride;
  p.I = d.in_features, p.O = d.out_features, p.G = d.num_codebooks, p.gs = d.group_size;
  p.Ro = (d.out_features + d.vector_len - 1) / d.vector_len;
  p.ib = ilog2(d.num_centroids);
  p.rb = d.num_res_centroids > 0 ? ilog2(d.num_res_centroids) : 0;
  p.S = (d.outlier_size > 0 && d.outlier_indices) ? d.outlier_size : 0;
  p.vol = p.S ? d.outlier_vector_len : 1;
  p.outlier_idx = p.S ? d.outlier_indices : nullptr;
  p.outlier_cb = p.S ? d.outlier_centroids : nullptr;
  p.scale = d.weight_scale, p.wbias = d.weight_bias;
  p.perm = d.perm;
  p.scale_q = (d.weight_scale_q && d.weight_bias_q && d.weight_scale) ? d.weight_scale_q : nullptr;
  p.wbias_q = p.scale_q ? d.weight_bias_q : nullptr;
  p.out = wt_out, p.ld = ld;
  const size_t res_rep_bytes = p.rb ? (size_t(1) << p.rb) * 16 * 8 : 0;
  const bool fast = d.vector_len == 8 && d.num_codebooks == 1 && p.S == 0 && (ld % 8) == 0 &&
                    res_rep_bytes <= 64 * 1024 && (reinterpret_cast<uintptr_t>(wt_out) & 15u) == 0;
  cudaError_t e;
  if (fast) {
    const int b = p.ib + p.rb;
    const size_t smem = ((size_t(DT_ROWS) * (size_t(DT_COLS) * b / 32 + 4) * 4 + 127) & ~size_t(127)) + res_rep_bytes;
    dim3 grid(unsigned((d.group_size + DT_COLS - 1) / DT_COLS), unsigned((ld / 8 + DT_ROWS - 1) / DT_ROWS));
    if (d.dtype == VPTQ_FP16) {
      if (int rc = ensure_smem_attr(reinterpret_cast<const void*>(dequant_t8_kernel<__half>), 100 * 1024)) return rc;
      dequant_t8_kernel<__half><<<grid, DT_THREADS, smem, stream>>>(p);
    } else {
      if (int rc = ensure_smem_attr(reinterpret_cast<const void*>(dequant_t8_kernel<__nv_bfloat16>), 100 * 1024)) return rc;
      dequant_t8_kernel<__nv_bfloat16><<<grid, DT_THREADS, smem, stream>>>(p);
    }
    e = cudaGetLastError();
  } else {
    dim3 grid(unsigned((d.in_features + 255) / 256), unsigned(std::min<int64_t>((ld + d.vector_len - 1) / d.vector_len, 65535)));
    switch (d.vector_len) {
#define VPTQ_CASE(VV)                                                                         \
  case VV:                                                                                    \
    if (d.dtype == VPTQ_FP16) dequant_t_kernel<__half, VV><<<grid, 256, 0, stream>>>(p);      \
    else dequant_t_kernel<__nv_bfloat16, VV><<<grid, 256, 0, stream>>>(p);                    \
    break;
      VPTQ_CASE(2) VPTQ_CASE(4) VPTQ_CASE(6) VPTQ_CASE(8) VPTQ_CASE(10) VPTQ_CASE(12) VPTQ_CASE(16)
#undef VPTQ_CASE
      default: set_error("dequant (transposed): vector_len %d not supported", d.vector_len); return VPTQ_ERR_UNSUPPORTED;
    }
    e = cudaGetLastError();
  }
  if (e != cudaSuccess) {
    set_error("dequant (transposed) launch: %s", cudaGetErrorString(e));
    return VPTQ_ERR_CUDA;
  }
  return 0;
}

}  // namespace vptq_b200
