// Decode GEMV for 1..4 tokens of vector-length-16 layers (the v16-k65536 checkpoints: 1.375-1.5 bits per weight)
// from the slice x tile lists of vptq_linear_desc::lists_*, built with index rows of 16 outputs
// (vptq_b200/lists.py: build_lists(vector_len=16), C: vptq_b200_lists16_build_host).  The entry word, geometry, tab
// and dealing pass are those of the v = 8 lists; the kernel is the batched list kernel's (gemv_lists_batch.cu) with
// every per-output quantity widened to 16:
//
//   * instances NTOK = 1, 2, 4 (x fp16/bf16, residual or not).  A call of `tokens` <= NTOK masks the missing tokens;
//   * partition: ONE combo (column tile, codebook slice) per CTA, k_l CTAs per combo of layer l, chosen from the
//     layer shapes and the SM count only (lists16_partition) -- never from the token count: every instance runs
//     the same CTAs, warps and warp runs, so a token's outputs are bit-identical whatever else is in its launch;
//   * shared memory: the combo's 4096-entry slice (128 KiB) as two planes, lo = elements 0..7 and hi = elements
//     8..15 of every entry, [4096][8] 16-bit each, staged with 16-byte cp.async straight from the checkpoint's
//     [K][16] codebook (no derived copy: in-place codebook updates need no refresh).  An entry is two conflict-free
//     LDS.128 whose 16-byte bank group is index & 7 in both planes, as at v = 8, so the dealing pass holds.  The
//     residual table in the same two planes, replicated `res_rep` times (8, 4, 2 or 1: what the budget leaves); the
//     x' tile as [column][NTOK] 16-bit values; a TMA ring of list steps per warp; the CTA's list table;
//   * per entry, per token, the list kernels' arithmetic: x' = x * scale rounded to the layer type, c + r in
//     packed fp16 (fp16) or fp32 (bf16), fp32 FMAs per unit, sum x * wbias of a tile added in fp32 to the tile's
//     slice-0 unit, each unit sum rounded to 2^-30 fixed point and added with red.global.add.u64 into
//     [row][NTOK][16] accumulators, bias after the conversion.  Non-finite and out-of-range unit sums are always kept
//     out of the fixed point (32-bit class record per (row, token)), padding lanes are always masked;
//   * arrival counters of 32-row blocks; the CTA completing a block converts it for every token, writes y and
//     leaves the accumulators, records and counters zeroed.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <type_traits>

#include "gemv_kernel.cuh"

namespace vptq_b200 {

namespace {

constexpr int kV = 16;                           // outputs per index row
constexpr int kSliceEntries = 4096;
constexpr int kPlaneBytes = kSliceEntries * 16;  // 64 KiB: 8 elements of every entry of the slice
constexpr int kLW = 16, kLT = kLW * 32;          // warps, threads per CTA (the same for every NTOK)
constexpr int kStSteps = 8;                      // steps (32 entries, 128 bytes) per ring stage
constexpr int kStageBytes = kStSteps * 128;
constexpr int kRB = 32;     // index rows per arrival counter
constexpr int kMaxTok = 4;  // largest instance (NTOK = 8 does not fit next to the 128 KiB planes at TCW = 4096)
constexpr int kMaxRowTokens = kMaxIndexRows / 2;  // [row][token][16] u64 = 128 bytes each in the 4 MiB accumulator head
constexpr uint32_t kStepMask = (1u << 26) - 1u;
// zero-at-rest head of the workspace: arrival counters in [0, kClassOffset), the 32-bit class records of every
// (index row, token) behind them, the [row][NTOK][16] accumulators from kCounterRegionBytes on
constexpr size_t kClassOffset = 16384;
static_assert(kClassOffset + size_t(kMaxRowTokens) * 4 <= kCounterRegionBytes, "");
static_assert(kCounterRegionBytes + size_t(kMaxRowTokens) * kV * 8 <= kZeroRegionBytes, "");
static_assert(VPTQ_B200_LISTS16_WORKSPACE_BYTES == kZeroRegionBytes, "");

struct L16Layer {
  const uint32_t* stream;  // [T][32] entry words
  const uint32_t* tab;     // [U + 1]
  const void* centroids;   // [K][16]
  const void* res_centroids;
  const void* scale;  // ORIGINAL feature order (or nullptr: no scale / bias)
  const void* wbias;
  const void* bias;
  void* y;
  int64_t y_stride;
  unsigned long long* yacc;  // [Ro][NTOK][16] fixed-point (2^-30) accumulators, zero at rest
  uint32_t* counters;        // [ceil(Ro / kRB)], zero at rest
  uint32_t* cls;             // [Ro][NTOK] class records of unit sums kept out of yacc, zero at rest
  float lim;                 // unit sums with |v| >= lim (or not finite) are not added as integers
  int I, O, Ro, Kr, NS, Q, TCW;
  int k;  // CTAs per combo
};

struct L16Params {
  int n, tokens;                             // fused layers, tokens of this launch (<= NTOK)
  uint32_t grid_begin[kMaxFusedLayers + 1];  // layer l owns blocks [grid_begin[l], grid_begin[l+1])
  const void* x;
  int64_t x_stride;
  int x_vec;  // rows of x are 16-byte aligned: 128-bit loads
  L16Layer layer[kMaxFusedLayers];
  uint32_t off_bars, off_tab, off_red, off_piece, off_done, off_lo, off_hi, off_rlo, off_rhi, off_x, off_ring;
  int stages, res_rep;
};

__device__ __forceinline__ uint32_t lds_u32(uint32_t a) {
  uint32_t r;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(r) : "r"(a));
  return r;
}
__device__ __forceinline__ uint32_t mad_u32(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t r;
  asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
  return r;
}
// one plane's half of an entry (8 elements) into w[o .. o+4): one LDS.128
__device__ __forceinline__ void lds_half(uint32_t (&w)[8], int o, uint32_t a) {
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(w[o]), "=r"(w[o + 1]), "=r"(w[o + 2]), "=r"(w[o + 3]) : "r"(a));
}
// the NTOK 16-bit x' values of one column: one 16-, 32- or 64-bit shared access
constexpr int tok_words(int ntok) { return (ntok + 1) / 2; }
template <int NTOK>
__device__ __forceinline__ void lds_tok(uint32_t (&w)[tok_words(NTOK)], uint32_t a) {
  if constexpr (NTOK == 1) {
    uint16_t h;
    asm volatile("ld.shared.u16 %0, [%1];" : "=h"(h) : "r"(a));
    w[0] = h;
  } else if constexpr (NTOK == 2) {
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w[0]) : "r"(a));
  } else {
    static_assert(NTOK == 4, "");
    asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(w[0]), "=r"(w[1]) : "r"(a));
  }
}
template <int NTOK>
__device__ __forceinline__ void sts_tok(uint32_t a, const uint32_t (&w)[tok_words(NTOK)]) {
  if constexpr (NTOK == 1) {
    asm volatile("st.shared.u16 [%0], %1;" ::"r"(a), "h"(uint16_t(w[0])) : "memory");
  } else if constexpr (NTOK == 2) {
    asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(w[0]) : "memory");
  } else {
    asm volatile("st.shared.v2.u32 [%0], {%1,%2};" ::"r"(a), "r"(w[0]), "r"(w[1]) : "memory");
  }
}

// fp32 -> 2^-30 fixed point: the rounding costs up to 2^-31 per unit, a floor of Q * 2^-31 per output.  Only
// |v| < lim = 2^33 / 2^ceil(log2 Q) is admitted (no sum of Q admitted terms reaches 2^63); anything else leaves its
// class in the (row, token) record and the output becomes +inf, -inf or NaN.
constexpr float kFixScale = 1073741824.f, kFixInv = 1.f / 1073741824.f;
constexpr uint32_t kClsPosInf = 1u, kClsNegInf = 2u, kClsNaN = 3u;  // OR of two classes = class of their sum
template <int NTOK>
__device__ __forceinline__ void add_unit(const L16Layer& L, int row, int tok, int e, float v) {
  const bool in_range = fabsf(v) < L.lim;  // (false for inf and NaN)
  const long long q = __float2ll_rn((in_range ? v : 0.f) * kFixScale);
  const size_t rt = size_t(row) * NTOK + tok;
  asm volatile("red.global.add.u64 [%0], %1;" ::"l"(L.yacc + rt * kV + e), "l"(q) : "memory");
  if (!in_range) {
    const uint32_t c = v == INFINITY ? kClsPosInf : v == -INFINITY ? kClsNegInf : kClsNaN;
    atomicOr(L.cls + rt, c << (2u * uint32_t(e)));
  }
}

// acc[k][e] += x'_k * (c[e] + r[e]) for every token k, e < 16: c + r formed once (fp16: packed fp16, bf16: fp32),
// then per token the list kernels' FMAs
template <typename T, bool RES, int NTOK>
__device__ __forceinline__ void fma_tokens(float (&acc)[NTOK][kV], const uint32_t (&xw)[tok_words(NTOK)],
                                           const uint32_t (&cw)[8], const uint32_t (&rw)[8]) {
  float c[kV];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float2 f;
    if constexpr (std::is_same<T, __half>::value) {
      f = DT<T>::unpack2(RES ? DT<T>::add2(cw[i], rw[i]) : cw[i]);
    } else {
      f = DT<T>::unpack2(cw[i]);
      if constexpr (RES) {
        const float2 r = DT<T>::unpack2(rw[i]);
        f.x += r.x, f.y += r.y;
      }
    }
    c[2 * i] = f.x, c[2 * i + 1] = f.y;
  }
#pragma unroll
  for (int k = 0; k < NTOK; ++k) {
    const float2 xv = DT<T>::unpack2(xw[k / 2]);
    const float xk = (k & 1) ? xv.y : xv.x;
#pragma unroll
    for (int e = 0; e < kV; ++e) acc[k][e] = fmaf(xk, c[e], acc[k][e]);
  }
}

// 8 consecutive 16-bit elements p[f .. f+8); elements at or beyond fend read as `fill`
template <typename T>
__device__ __forceinline__ uint4 load8v(const T* p, int f, int fend, uint16_t fill, bool vec) {
  if (vec && f + 8 <= fend) return *reinterpret_cast<const uint4*>(p + f);
  uint16_t h[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) h[k] = (f + k < fend) ? reinterpret_cast<const uint16_t*>(p)[f + k] : fill;
  return make_uint4(h[0] | uint32_t(h[1]) << 16, h[2] | uint32_t(h[3]) << 16, h[4] | uint32_t(h[5]) << 16,
                    h[6] | uint32_t(h[7]) << 16);
}

// x' = x * scale for 8 features (stored in the layer's 16-bit type) and sum x * wbias (fp32)
template <typename T>
__device__ __forceinline__ uint4 make_xq(const uint4& xr, const uint4& sc, const uint4& wb, bool with_bias, float& bs) {
  const uint32_t xs[4] = {xr.x, xr.y, xr.z, xr.w}, ss[4] = {sc.x, sc.y, sc.z, sc.w}, ws[4] = {wb.x, wb.y, wb.z, wb.w};
  uint32_t o[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 xf = DT<T>::unpack2(xs[i]);
    if constexpr (std::is_same<T, __half>::value) {
      __half2 p = __hmul2(*reinterpret_cast<const __half2*>(&xs[i]), *reinterpret_cast<const __half2*>(&ss[i]));
      o[i] = *reinterpret_cast<uint32_t*>(&p);
    } else {  // (the fp32 product of two bf16 values is exact: one rounding)
      const float2 sf = DT<T>::unpack2(ss[i]);
      o[i] = DT<T>::pack2(xf.x * sf.x, xf.y * sf.y);
    }
    if (with_bias) {
      const float2 wf = DT<T>::unpack2(ws[i]);
      bs = fmaf(xf.x, wf.x, bs);
      bs = fmaf(xf.y, wf.y, bs);
    }
  }
  return make_uint4(o[0], o[1], o[2], o[3]);
}

template <typename T, bool RES, int NTOK>
__global__ void __launch_bounds__(kLT, 1) gemv_lists16_kernel(const __grid_constant__ L16Params mp) {
  // steps whose gathers are in flight together: the accumulators take 16 NTOK registers, an entry 16 (with residual)
  // (the per-lane FMA order is the step order whatever the batch is: results do not depend on it)
  constexpr int kSPS = NTOK == 1 ? 4 : NTOK == 2 ? 2 : 1;
  constexpr int kTW = tok_words(NTOK);
  extern __shared__ __align__(128) uint8_t smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int l = 0;
#pragma unroll
  for (int i = 1; i < kMaxFusedLayers; ++i)
    if (i < mp.n && blockIdx.x >= mp.grid_begin[i]) l = i;
  const L16Layer& L = mp.layer[l];
  const int q = int(blockIdx.x - mp.grid_begin[l]);
  const int combo = q / L.k, jc = q - combo * L.k;
  const int Ro = L.Ro, TCW = L.TCW, I = L.I, ntok = mp.tokens, stages = mp.stages;
  const int r0 = int(int64_t(Ro) * jc / L.k), r1 = int(int64_t(Ro) * (jc + 1) / L.k);
  const int nun = r1 - r0;  // this CTA's units: rows [r0, r1) of one combo
  const int tile = combo / L.NS, slice = combo - tile * L.NS;

  uint64_t* full = reinterpret_cast<uint64_t*>(smem + mp.off_bars) + warp * stages;
  uint32_t* s_tab = reinterpret_cast<uint32_t*>(smem + mp.off_tab);  // [nun + 1]
  float* s_red = reinterpret_cast<float*>(smem + mp.off_red);         // [warps][NTOK] bias partial sums
  float* s_cb = s_red + kLW * kMaxTok;                                // [NTOK] sum x * wbias of the tile
  int* s_ndone = reinterpret_cast<int*>(s_cb + kMaxTok);
  float* s_piece = reinterpret_cast<float*>(smem + mp.off_piece);                  // [warps][2][NTOK][16]
  int* s_pu = reinterpret_cast<int*>(smem + mp.off_piece + kLW * 2 * NTOK * kV * 4);  // [warps][2]
  int* s_done = reinterpret_cast<int*>(smem + mp.off_done);                        // row blocks completed here
  const uint32_t s_lo = smem_u32(smem + mp.off_lo), s_hi = smem_u32(smem + mp.off_hi);
  const uint32_t s_rlo = smem_u32(smem + mp.off_rlo), s_rhi = smem_u32(smem + mp.off_rhi);
  const uint32_t s_x = smem_u32(smem + mp.off_x);  // [TCW][NTOK] 16-bit x'
  uint8_t* ring = smem + mp.off_ring + size_t(warp) * stages * kStageBytes;

  const uint64_t pol_stream = policy_evict_first();
  const uint64_t pol_keep = policy_evict_last();
  if (tid < kLW * stages) {
    mbar_init(reinterpret_cast<uint64_t*>(smem + mp.off_bars) + tid, 1);
    fence_mbar_init();
  }
  if (tid == 0) *s_ndone = 0;
  for (int i = tid; i <= nun; i += kLT) s_tab[i] = L.tab[size_t(combo) * Ro + r0 + i];
  // x-independent column data of the tile: scale, and weight_bias where this CTA owns the bias term (slice 0)
  const T* scale = reinterpret_cast<const T*>(L.scale);
  const T* wbias = reinterpret_cast<const T*>(L.wbias);
  const uint16_t one16 = std::is_same<T, __half>::value ? uint16_t(0x3c00u) : uint16_t(0x3f80u);
  const uint32_t one32 = uint32_t(one16) | uint32_t(one16) << 16;
  const int j0 = tid * 8;  // column of the tile this thread prepares (TCW <= 4096 = 8 * kLT)
  const bool col = j0 < TCW && tile * TCW + j0 < I;
  const int f0 = tile * TCW + j0, fend = min(I, (tile + 1) * TCW);
  const bool with_bias = scale != nullptr && slice == 0;
  uint4 sc = make_uint4(one32, one32, one32, one32), wb = make_uint4(0u, 0u, 0u, 0u);
  if (scale && col) {
    sc = load8v<T>(scale, f0, fend, one16, true);
    if (with_bias) wb = load8v<T>(wbias, f0, fend, 0, true);
  }
  if (lane == 0) s_pu[warp * 2] = -1, s_pu[warp * 2 + 1] = -1;
  __syncthreads();
  pdl_launch_dependents();

  // -------- this warp's run: an equal share of the CTA's contiguous step range (a function of the lists only) --
  const int T0 = int(s_tab[0] & kStepMask), T1 = int(s_tab[nun] & kStepMask), TT = T1 - T0;
  const int t_begin = T0 + int(int64_t(TT) * warp / kLW), t_end = T0 + int(int64_t(TT) * (warp + 1) / kLW);
  const int nstage = (t_end - t_begin + kStSteps - 1) / kStSteps;
  auto issue = [&](int qi, int slot) {
    if (lane == 0) {
      const int t = t_begin + qi * kStSteps, cnt = min(kStSteps, t_end - t);
      mbar_arrive_expect_tx(&full[slot], uint32_t(cnt) * 128u);
      tma_bulk_g2s(ring + size_t(slot) * kStageBytes, L.stream + size_t(t) * 32, uint32_t(cnt) * 128u, &full[slot],
                   pol_stream);
    }
  };
  // x-independent work first: it overlaps the previous kernel's tail under programmatic dependent launch.
  // The slice's planes: 16-byte chunk c of the slice is half c & 1 of entry c >> 1 (consecutive threads read
  // consecutive global bytes); the residual planes likewise, copy j of entry r at (r * res_rep + j) * 16.
  for (int qi = 0; qi < min(stages, nstage); ++qi) issue(qi, qi);
  {
    const uint8_t* cb = reinterpret_cast<const uint8_t*>(L.centroids) + size_t(slice) * kSliceEntries * 32;
#pragma unroll 4
    for (int c = tid; c < 2 * kSliceEntries; c += kLT)
      cp_async_16(((c & 1) ? s_hi : s_lo) + uint32_t(c >> 1) * 16u, cb + size_t(c) * 16, pol_keep);
    if constexpr (RES) {
      const uint8_t* rb = reinterpret_cast<const uint8_t*>(L.res_centroids);
      const int rep = mp.res_rep, nres = L.Kr * rep * 2;
      for (int c = tid; c < nres; c += kLT) {
        const int rc = c >> 1, r = rc / rep;
        cp_async_16(((c & 1) ? s_rhi : s_rlo) + uint32_t(rc) * 16u, rb + size_t(r) * 32 + (c & 1) * 16, pol_keep);
      }
    }
    cp_async_commit();
  }
  pdl_wait_prior_grid();

  // -------- x'[f][k] = x_k[f] * scale[f], interleaved by token; sum_f x_k[f] * wbias[f] ----------------------
  {
    const T* x = reinterpret_cast<const T*>(mp.x);
    uint32_t xq[NTOK][4];
    float bs[NTOK];
#pragma unroll
    for (int k = 0; k < NTOK; ++k) {
      bs[k] = 0.f;
      uint4 o = make_uint4(0u, 0u, 0u, 0u);
      if (col && k < ntok) {
        const uint4 xr = load8v<T>(x + size_t(k) * size_t(mp.x_stride), f0, fend, 0, mp.x_vec != 0);
        o = make_xq<T>(xr, sc, wb, with_bias, bs[k]);
      }
      xq[k][0] = o.x, xq[k][1] = o.y, xq[k][2] = o.z, xq[k][3] = o.w;
    }
    if (col) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        uint32_t w[kTW];
#pragma unroll
        for (int k2 = 0; k2 < kTW; ++k2) {
          const uint32_t lo = (xq[2 * k2][i / 2] >> ((i & 1) * 16)) & 0xffffu;
          const uint32_t hi = 2 * k2 + 1 < NTOK ? (xq[(2 * k2 + 1) % NTOK][i / 2] >> ((i & 1) * 16)) & 0xffffu : 0u;
          w[k2] = lo | hi << 16;
        }
        sts_tok<NTOK>(s_x + uint32_t(j0 + i) * uint32_t(NTOK * 2), w);
      }
    }
    if (with_bias) {  // (CTA-uniform)
#pragma unroll
      for (int k = 0; k < NTOK; ++k) {
        const float v = warp_sum(bs[k]);
        if (lane == 0) s_red[warp * kMaxTok + k] = v;
      }
    }
  }
  cp_async_wait<0>();
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int k = 0; k < NTOK; ++k) {
      const float v = with_bias ? warp_sum(lane < kLW ? s_red[lane * kMaxTok + k] : 0.f) : 0.f;
      if (lane == 0) s_cb[k] = v;
    }
  }
  __syncthreads();

  // -------- main loop ---------------------------------------------------------------------------------
  if (nstage > 0) {
    const uint32_t rstride = uint32_t(mp.res_rep) * 16u;
    const uint32_t rsel = uint32_t(lane & (mp.res_rep - 1)) * 16u;  // lane reads copy lane mod res_rep
    const uint32_t rlo_lane = s_rlo + rsel, rhi_lane = s_rhi + rsel;
    const uint32_t ring_lane = smem_u32(ring) + uint32_t(lane) * 4u;
    int u;  // the unit this run starts in: the last i with first(i) <= t_begin (every unit has >= 1 step)
    {
      int lo = 0, hi = nun - 1;
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (int(s_tab[mid] & kStepMask) <= t_begin) lo = mid;
        else hi = mid - 1;
      }
      u = lo;
    }
    const int uF = u;
    int u_end = int(s_tab[u + 1] & kStepMask);
    uint32_t tail = s_tab[u] >> 26;
    float acc[NTOK][kV];
#pragma unroll
    for (int k = 0; k < NTOK; ++k)
#pragma unroll
      for (int e = 0; e < kV; ++e) acc[k][e] = 0.f;
    // the current unit's sums are final for this run: interior units go to global memory, the first and the last
    // unit of the run may be shared with the neighbouring warps and are parked for the merge below
    auto flush = [&](bool complete) {
      const bool boundary = u == uF || !complete || u_end >= t_end;
      const int kk = warp * 2 + (u == uF ? 0 : 1);
#pragma unroll
      for (int k = 0; k < NTOK; ++k) {
        if (k < ntok) {  // (warp-uniform)
          float a_lo[8], a_hi[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) a_lo[e] = acc[k][e], a_hi[e] = acc[k][8 + e];
          const float m_lo = warp_reduce_to_lane<8>(a_lo, lane), m_hi = warp_reduce_to_lane<8>(a_hi, lane);
          if (lane < 8) {
            if (!boundary) {
              add_unit<NTOK>(L, r0 + u, k, lane, m_lo + s_cb[k]);
              add_unit<NTOK>(L, r0 + u, k, 8 + lane, m_hi + s_cb[k]);
            } else {
              s_piece[(kk * NTOK + k) * kV + lane] = m_lo;
              s_piece[(kk * NTOK + k) * kV + 8 + lane] = m_hi;
            }
          }
        }
#pragma unroll
        for (int e = 0; e < kV; ++e) acc[k][e] = 0.f;
      }
      if (boundary && lane == 0) s_pu[kk] = u;
    };
    auto advance = [&]() {
      ++u;
      if (u < nun) {
        u_end = int(s_tab[u + 1] & kStepMask);
        tail = s_tab[u] >> 26;
      }
    };
    int slot = 0, t = t_begin;
    uint32_t par = 0;
#pragma unroll 1
    for (int qi = 0; qi < nstage; ++qi) {
      mbar_wait(&full[slot], par);
      uint32_t st = ring_lane + uint32_t(slot) * uint32_t(kStageBytes);
      const int se = min(t + kStSteps, t_end);
#pragma unroll 1
      while (t < se) {
        const int cnt = min(kSPS, se - t);
        uint32_t ent[kSPS], cw[kSPS][8], rw[kSPS][8], xw[kSPS][kTW];
#pragma unroll
        for (int j = 0; j < kSPS; ++j)
          if (j < cnt) ent[j] = lds_u32(st + uint32_t(j) * 128u);
#pragma unroll
        for (int j = 0; j < kSPS; ++j) {
          if (j < cnt) {
            // entry = index12 | column12 << 12 | residual8 << 24; both planes at the same offset
            const uint32_t co = (ent[j] & 0xfffu) * 16u;
            lds_half(cw[j], 0, s_lo + co);
            lds_half(cw[j], 4, s_hi + co);
            if constexpr (RES) {
              lds_half(rw[j], 0, mad_u32(ent[j] >> 24, rstride, rlo_lane));
              lds_half(rw[j], 4, mad_u32(ent[j] >> 24, rstride, rhi_lane));
            }
            lds_tok<NTOK>(xw[j], mad_u32((ent[j] >> 12) & 0xfffu, uint32_t(NTOK * 2), s_x));
          }
        }
#pragma unroll
        for (int j = 0; j < kSPS; ++j) {
          if (j < cnt) {
            const bool last = t + 1 == u_end;
            // padding lanes of a unit's last step add nothing (not 0 * entry: an inf or NaN entry 0 would give NaN)
            if (!last || uint32_t(lane) < tail) fma_tokens<T, RES, NTOK>(acc, xw[j], cw[j], rw[j]);
            ++t;
            if (last) {
              flush(true);
              advance();
            }
          }
        }
        st += uint32_t(cnt) * 128u;
      }
      __syncwarp();  // every lane has read its words of the stage: refill it
      if (qi + stages < nstage) issue(qi + stages, slot);
      if (++slot == stages) slot = 0, par ^= 1u;
    }
    // the run ended inside a unit: its sums so far are this warp's piece of that unit
    if (u < nun && int(s_tab[u] & kStepMask) < t_end) flush(false);
  }
  __syncthreads();

  // -------- merge the pieces of units shared between warps (in warp order) ---------------------------------
  for (int it = tid; it < kLW * 2 * NTOK * kV; it += kLT) {
    const int i = it / (NTOK * kV), k = (it / kV) % NTOK, e = it % kV;
    const int un = s_pu[i];
    if (un < 0 || k >= ntok) continue;
    bool leader = true;
    for (int j = i - 1; j >= 0; --j) {
      const int pj = s_pu[j];
      if (pj < 0) continue;
      leader = pj != un;
      break;
    }
    if (!leader) continue;
    float v = s_piece[(i * NTOK + k) * kV + e];
    for (int j = i + 1; j < kLW * 2; ++j) {
      const int pj = s_pu[j];
      if (pj < 0) continue;
      if (pj != un) break;
      v += s_piece[(j * NTOK + k) * kV + e];
    }
    add_unit<NTOK>(L, r0 + un, k, e, v + s_cb[k]);
  }
  __threadfence();
  __syncthreads();

  // -------- arrival: every row block of rows [r0, r1) learns how many of its units are done --------------
  {
    const int nb = (r1 - 1) / kRB - r0 / kRB + 1;
    for (int i = tid; i < nb; i += kLT) {
      const int b = r0 / kRB + i, lo = max(r0, b * kRB), hi = min(r1, (b + 1) * kRB);
      const uint32_t cnt = uint32_t(hi - lo), rows_b = uint32_t(min(kRB, Ro - b * kRB));
      const uint32_t prev = atomicAdd(&L.counters[b], cnt);
      if (prev + cnt == uint32_t(L.Q) * rows_b) s_done[atomicAdd(s_ndone, 1)] = b;
    }
  }
  __syncthreads();
  const int nd = *s_ndone;
  if (nd > 0) {
    // this CTA's arrival completed nd row blocks: every unit of their rows has added its sums.  One thread per
    // (row, token, half): 8 outputs each
    __threadfence();
    const T* bias = reinterpret_cast<const T*>(L.bias);
    const int nrow = nd * kRB;
    for (int i = tid; i < nrow * ntok * 2; i += kLT) {
      const int h = i & 1, i2 = i >> 1;
      const int k = i2 / nrow, ri = i2 - k * nrow;
      const int r = s_done[ri / kRB] * kRB + ri % kRB;
      if (r >= Ro) continue;
      const size_t rt = size_t(r) * NTOK + k;
      unsigned long long* p = L.yacc + rt * kV + h * 8;
      long long qv[8];
      uint32_t cls;
      asm volatile("ld.global.cg.u32 %0, [%1];" : "=r"(cls) : "l"(L.cls + rt) : "memory");
#pragma unroll
      for (int j = 0; j < 4; ++j)
        asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(qv[2 * j]), "=l"(qv[2 * j + 1]) : "l"(p + 2 * j) : "memory");
#pragma unroll
      for (int j = 0; j < 4; ++j) *reinterpret_cast<ulonglong2*>(p + 2 * j) = make_ulonglong2(0ull, 0ull);  // zero at rest
      const int o = r * kV + h * 8;
      float v[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const uint32_t c = (cls >> (2 * (h * 8 + e))) & 3u;
        const float s = c == 0u ? float(qv[e]) * kFixInv : c == kClsPosInf ? INFINITY : c == kClsNegInf ? -INFINITY : NAN;
        v[e] = s + ((bias && o + e < L.O) ? DT<T>::to_float(bias[o + e]) : 0.f);
      }
      T* y = reinterpret_cast<T*>(L.y) + size_t(k) * size_t(L.y_stride);
      if (o + 8 <= L.O && (reinterpret_cast<uintptr_t>(y + o) & 15u) == 0) {
        *reinterpret_cast<uint4*>(y + o) = make_uint4(DT<T>::pack2(v[0], v[1]), DT<T>::pack2(v[2], v[3]),
                                                      DT<T>::pack2(v[4], v[5]), DT<T>::pack2(v[6], v[7]));
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e)
          if (o + e < L.O) y[o + e] = DT<T>::from_float(v[e]);
      }
    }
    __syncthreads();  // (both halves of a record have read it)
    for (int i = tid; i < nrow * ntok; i += kLT) {
      const int k = i / nrow, ri = i - k * nrow;
      const int r = s_done[ri / kRB] * kRB + ri % kRB;
      if (r < Ro) L.cls[size_t(r) * NTOK + k] = 0u;
    }
    if (tid < nd) L.counters[s_done[tid]] = 0u;  // leave the counters zeroed for the next launch
  }
}

using L16KernelFn = void (*)(const L16Params);

template <typename T, int NTOK>
L16KernelFn pick_t(bool res) {
  return res ? gemv_lists16_kernel<T, true, NTOK> : gemv_lists16_kernel<T, false, NTOK>;
}
L16KernelFn pick(int dtype, bool res, int ntok) {
  if (dtype == VPTQ_FP16) {
    if (ntok == 1) return pick_t<__half, 1>(res);
    if (ntok == 2) return pick_t<__half, 2>(res);
    if (ntok == 4) return pick_t<__half, 4>(res);
  } else if (dtype == VPTQ_BF16) {
    if (ntok == 1) return pick_t<__nv_bfloat16, 1>(res);
    if (ntok == 2) return pick_t<__nv_bfloat16, 2>(res);
    if (ntok == 4) return pick_t<__nv_bfloat16, 4>(res);
  }
  return nullptr;
}

// smallest instance that holds `tokens`
int instance(int tokens) { return tokens <= 1 ? 1 : tokens <= 2 ? 2 : 4; }

int lists_tcw16(int I) {
  const int nt = (I + 4095) / 4096;
  return ((I + nt - 1) / nt + 7) / 8 * 8;
}

// What a launch of these layers looks like, for any token count.
struct L16Plan {
  int n, Q, NS, TCW, I;
  int Ro[kMaxFusedLayers], k[kMaxFusedLayers];
  int rows, max_nun, max_kr;
  bool res;
};

// The partition (tokens never enter it): the batched list kernel's (gemv_lists_batch.cu: batch_partition) --
// B = SM count / Q combo copies shared out to the layers in proportion to their rows, at least one each, at most
// one CTA per row; integer comparisons, mirrored in tests/test_lists16_host.py.  0 or a vptq_status, message set.
int lists16_partition(int n, const vptq_linear_desc* const* descs, int sm_count, L16Plan* pl) {
  if (n < 1 || n > kMaxFusedLayers || !descs) {
    set_error("quant_gemv_lists16: 1..%d layers", kMaxFusedLayers);
    return VPTQ_ERR_UNSUPPORTED;
  }
  const vptq_linear_desc& d0 = *descs[0];
  pl->res = d0.num_res_centroids > 0;
  for (int l = 0; l < n; ++l) {
    const vptq_linear_desc& d = *descs[l];
    if (!gemv_lists16_eligible(d) || d.dtype != d0.dtype || d.in_features != d0.in_features ||
        d.num_centroids != d0.num_centroids || (d.num_res_centroids > 0) != pl->res) {
      set_error("quant_gemv_lists16: layer %d carries no vector-length-16 index lists this kernel takes (vector_len 16, "
                "one codebook group, no outliers, K = 4096 * (2..16), Kr <= 256), or does not match layer 0", l);
      return VPTQ_ERR_UNSUPPORTED;
    }
  }
  pl->n = n, pl->I = d0.in_features, pl->TCW = d0.lists_tile_cols;
  pl->NS = d0.num_centroids / kSliceEntries;
  pl->Q = pl->NS * ((pl->I + pl->TCW - 1) / pl->TCW);
  const int Q = pl->Q, B = sm_count / Q;
  if (n > B) {
    set_error("quant_gemv_lists16: %d layers x %d combos exceed %d SMs", n, Q, sm_count);
    return VPTQ_ERR_UNSUPPORTED;
  }
  int64_t rows = 0;
  for (int l = 0; l < n; ++l) pl->Ro[l] = (descs[l]->out_features + kV - 1) / kV, rows += pl->Ro[l];
  if (rows > kMaxRowTokens) {
    set_error("quant_gemv_lists16: %lld index rows exceed %d", (long long)rows, kMaxRowTokens);
    return VPTQ_ERR_UNSUPPORTED;
  }
  pl->rows = int(rows);
  int* k = pl->k;
  const int* Ro = pl->Ro;
  int used = 0;
  for (int l = 0; l < n; ++l) {
    k[l] = std::max(1, int(int64_t(B) * Ro[l] / rows));
    k[l] = std::min(k[l], Ro[l]);
    used += k[l];
  }
  while (used > B) {  // take from the layer with the most CTAs per row
    int v = -1;
    for (int l = 0; l < n; ++l)
      if (k[l] > 1 && (v < 0 || int64_t(k[l]) * Ro[v] > int64_t(k[v]) * Ro[l])) v = l;
    --k[v], --used;  // (n <= B: some layer has k > 1)
  }
  while (used < B) {  // give to the layer with the most rows per CTA
    int v = -1;
    for (int l = 0; l < n; ++l)
      if (k[l] < Ro[l] && (v < 0 || int64_t(Ro[l]) * k[v] > int64_t(Ro[v]) * k[l])) v = l;
    if (v < 0) break;
    ++k[v], ++used;
  }
  pl->max_nun = 0, pl->max_kr = 0;
  for (int l = 0; l < n; ++l) {
    pl->max_nun = std::max(pl->max_nun, (Ro[l] + k[l] - 1) / k[l]);
    pl->max_kr = std::max(pl->max_kr, descs[l]->num_res_centroids > 0 ? descs[l]->num_res_centroids : 0);
  }
  size_t nblk = 0;
  for (int l = 0; l < n; ++l) nblk += size_t((Ro[l] + kRB - 1) / kRB);
  if (nblk * 4 > kClassOffset) {
    set_error("quant_gemv_lists16: %zu row blocks exceed the counter region", nblk);
    return VPTQ_ERR_UNSUPPORTED;
  }
  return 0;
}

// shared-memory carve-up of instance NTOK; returns the bytes (0: nothing fits).  The residual replication comes
// first (every step gathers from it), then the ring depth.
size_t lists16_carve(const L16Plan& pl, int ntok, size_t limit, L16Params* mp) {
  for (int rep = 8; rep >= 1; rep >>= 1) {
    for (int stages = 3; stages >= 2; --stages) {
      size_t off = 0;
      mp->off_bars = uint32_t(off), off += align_up(size_t(kLW * stages) * 8, 128);
      mp->off_tab = uint32_t(off), off += align_up(size_t(pl.max_nun + 1) * 4, 128);
      mp->off_red = uint32_t(off), off += align_up(size_t(kLW + 1) * kMaxTok * 4 + 16, 128);
      mp->off_piece = uint32_t(off), off += align_up(size_t(kLW) * 2 * ntok * kV * 4 + size_t(kLW) * 2 * 4, 128);
      mp->off_done = uint32_t(off), off += align_up(size_t(pl.max_nun / kRB + 2) * 4, 128);
      mp->off_lo = uint32_t(off), off += size_t(kPlaneBytes);
      mp->off_hi = uint32_t(off), off += size_t(kPlaneBytes);
      const size_t rplane = align_up(size_t(pl.max_kr) * 16 * rep, 128);
      mp->off_rlo = uint32_t(off), off += rplane;
      mp->off_rhi = uint32_t(off), off += rplane;
      mp->off_x = uint32_t(off), off += align_up(size_t(pl.TCW) * ntok * 2, 128);
      mp->off_ring = uint32_t(off), off += size_t(kLW) * stages * kStageBytes;
      mp->stages = stages, mp->res_rep = rep;
      if (off <= limit) return off;
    }
  }
  return 0;
}

// largest instance that fits these layers' rows and shared memory (0: none, message set)
int lists16_max(const L16Plan& pl, int smem_optin) {
  for (int ntok = kMaxTok; ntok >= 1; ntok >>= 1) {
    if (int64_t(pl.rows) * ntok > kMaxRowTokens) continue;
    L16Params mp{};
    if (lists16_carve(pl, ntok, size_t(smem_optin), &mp)) return ntok;
  }
  set_error("quant_gemv_lists16: no shared-memory layout fits");
  return 0;
}

}  // namespace

bool gemv_lists16_eligible(const vptq_linear_desc& d) {
  if (!d.lists_stream || !d.lists_tab) return false;
  const bool outl = d.outlier_size > 0 && d.outlier_indices != nullptr;
  if (d.vector_len != kV || d.num_codebooks != 1 || outl) return false;
  if (d.num_centroids < 2 * kSliceEntries || d.num_centroids % kSliceEntries) return false;
  if (d.num_centroids / kSliceEntries > 16) return false;
  if (d.num_res_centroids > 256) return false;
  if (d.in_features < 8 || d.lists_tile_cols != lists_tcw16(d.in_features)) return false;
  if ((reinterpret_cast<uintptr_t>(d.lists_stream) & 15u) || (reinterpret_cast<uintptr_t>(d.lists_tab) & 3u)) return false;
  if ((reinterpret_cast<uintptr_t>(d.weight_scale) & 15u) || (reinterpret_cast<uintptr_t>(d.weight_bias) & 15u)) return false;
  return true;
}

int gemv_lists16_max_tokens(int n, const vptq_linear_desc* const* descs) {
  const DeviceInfo* dev = device_info();
  if (!dev) return 0;
  L16Plan pl;
  if (lists16_partition(n, descs, dev->sm_count, &pl)) return 0;
  return lists16_max(pl, dev->smem_optin);
}

int gemv_lists16_launch(int n, const vptq_linear_desc* const* descs, const void* x, int64_t x_stride, void* const* ys,
                        const int64_t* y_strides, int tokens, uint32_t flags, cudaStream_t stream, void* workspace,
                        size_t workspace_bytes) {
  const DeviceInfo* dev = device_info();
  if (!dev) return VPTQ_ERR_CUDA;
  L16Plan pl;
  if (int rc = lists16_partition(n, descs, dev->sm_count, &pl)) return rc;
  const int max_tokens = lists16_max(pl, dev->smem_optin);
  if (max_tokens == 0) return VPTQ_ERR_UNSUPPORTED;
  if (tokens < 1 || tokens > max_tokens) {
    set_error("quant_gemv_lists16: %d tokens; these layers take 1..%d", tokens, max_tokens);
    return VPTQ_ERR_UNSUPPORTED;
  }
  if (reinterpret_cast<uintptr_t>(x) & 15u) {
    set_error("quant_gemv_lists16: x must be 16-byte aligned");
    return VPTQ_ERR_UNSUPPORTED;
  }
  if (!workspace || workspace_bytes < kZeroRegionBytes) {
    set_error("quant_gemv_lists16: workspace %zu bytes < required %zu", workspace_bytes, kZeroRegionBytes);
    return VPTQ_ERR_WORKSPACE;
  }
  const int ntok = instance(tokens);
  L16KernelFn fn = pick(descs[0]->dtype, pl.res, ntok);
  if (!fn) return VPTQ_ERR_UNSUPPORTED;
  L16Params mp{};
  const size_t need = lists16_carve(pl, ntok, size_t(dev->smem_optin), &mp);
  if (!need) {
    set_error("quant_gemv_lists16: no shared-memory layout fits");
    return VPTQ_ERR_UNSUPPORTED;
  }
  if (int rc = ensure_smem_attr(reinterpret_cast<const void*>(fn), dev->smem_optin)) return rc;

  mp.n = n, mp.tokens = tokens, mp.x = x, mp.x_stride = x_stride, mp.x_vec = (x_stride % 8) == 0;
  int lg_q = 0;
  while ((1 << lg_q) < pl.Q) ++lg_q;
  uint8_t* wsb = reinterpret_cast<uint8_t*>(workspace);
  size_t acc_off = kCounterRegionBytes, ctr_off = 0, cls_off = kClassOffset;
  uint32_t begin = 0;
  for (int l = 0; l < n; ++l) {
    const vptq_linear_desc& d = *descs[l];
    L16Layer& L = mp.layer[l];
    L.stream = reinterpret_cast<const uint32_t*>(d.lists_stream), L.tab = d.lists_tab;
    L.centroids = d.centroids, L.res_centroids = d.res_centroids;
    L.scale = d.weight_scale, L.wbias = d.weight_scale ? d.weight_bias : nullptr;
    L.bias = d.bias, L.y = ys[l], L.y_stride = y_strides[l];
    L.I = pl.I, L.O = d.out_features, L.Ro = pl.Ro[l], L.Kr = d.num_res_centroids > 0 ? d.num_res_centroids : 0;
    L.NS = pl.NS, L.Q = pl.Q, L.TCW = pl.TCW, L.k = pl.k[l];
    L.yacc = reinterpret_cast<unsigned long long*>(wsb + acc_off);
    L.counters = reinterpret_cast<uint32_t*>(wsb + ctr_off);
    L.cls = reinterpret_cast<uint32_t*>(wsb + cls_off);
    L.lim = std::ldexp(1.f, 33 - lg_q);
    acc_off += size_t(pl.Ro[l]) * ntok * kV * 8;
    ctr_off += size_t((pl.Ro[l] + kRB - 1) / kRB) * 4;
    cls_off += size_t(pl.Ro[l]) * ntok * 4;
    mp.grid_begin[l] = begin;
    begin += uint32_t(pl.k[l] * pl.Q);
  }
  for (int l = n; l <= kMaxFusedLayers; ++l) mp.grid_begin[l] = begin;

  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(begin);
  cfg.blockDim = dim3(unsigned(kLT));
  cfg.dynamicSmemBytes = need;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  int nattr = 0;
  if (flags & VPTQ_FLAG_PDL) {
    attr[nattr].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[nattr].val.programmaticStreamSerializationAllowed = 1;
    ++nattr;
  }
  cfg.attrs = attr, cfg.numAttrs = unsigned(nattr);
  const cudaError_t e = cudaLaunchKernelEx(&cfg, fn, mp);
  if (e != cudaSuccess) {
    set_error("quant_gemv_lists16 launch (grid=%u smem=%zu): %s", begin, need, cudaGetErrorString(e));
    return VPTQ_ERR_CUDA;
  }
  return 0;
}

}  // namespace vptq_b200
