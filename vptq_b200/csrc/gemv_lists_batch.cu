// Decode GEMV for 1..8 tokens (beams, batched sequences, speculative verification) from the slice x tile lists
// of vptq_linear_desc::lists_* -- the lists, builders and dealing pass of the single-token kernel
// (gemv_lists.cu), read without materialising the weight.  Every entry, codebook slice and residual row a
// lane gathers serves all tokens of the launch: only the x' gather and the FMAs grow with the token count.
//
//   * instances NTOK = 2, 4, 8 (x fp16/bf16, residual or not).  A call of `tokens` <= NTOK masks the missing
//     tokens: their x' is 0 and their sums are never added, converted or stored;
//   * partition: ONE combo (column tile, codebook slice) per CTA.  Combo c of layer l is worked by k_l CTAs;
//     CTA j takes index rows [Ro j / k_l, Ro (j + 1) / k_l).  k_l is chosen from the layer shapes and the SM
//     count only (batch_partition), never from the token count: every instance runs the same CTAs, the same
//     16 warps and the same warp runs, so each token's fp32 unit sums see the same entries in the same order.
//     A token's outputs are bit-identical whatever else is in its batch;
//   * shared memory: one 64 KiB slice, the 8x bank-replicated residual table, the x' tile as [column][NTOK]
//     16-bit values (a lane gets every token's x' of its entry with one LDS.32 / .64 / .128), a TMA ring per
//     warp and the CTA's list table;
//   * per entry, per token, the single-token kernel's arithmetic: x' = x * scale rounded to the layer type,
//     c + r in packed fp16 (fp16) or fp32 (bf16), fp32 FMAs per unit, sum x * wbias of a tile added in fp32 to
//     the tile's slice-0 unit, each unit sum rounded to 2^-30 fixed point and added with red.global.add.u64
//     into [row][NTOK][8] accumulators, bias after the conversion.  Non-finite and out-of-range unit sums are
//     always kept out of the fixed point (per (row, token) class record), padding lanes are always masked;
//   * arrival counters of 32-row blocks count units as in the single-token kernel; the CTA completing a
//     block converts it for every token, writes y and leaves the accumulators, records and counters zeroed.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <type_traits>

#include "gemv_kernel.cuh"

namespace vptq_b200 {

namespace {

constexpr int kSliceEntries = 4096;
constexpr int kSliceBytes = kSliceEntries * 16;  // 64 KiB
constexpr int kLW = 16, kLT = kLW * 32;          // warps, threads per CTA (the same for every NTOK)
constexpr int kStSteps = 8;                      // steps (32 entries, 128 bytes) per ring stage
constexpr int kStageBytes = kStSteps * 128;
constexpr int kRB = 32;      // index rows per arrival counter
constexpr int kResRep = 8;   // bank-group replication of the residual table
constexpr int kMaxTok = 8;   // largest instance
constexpr uint32_t kStepMask = (1u << 26) - 1u;
// zero-at-rest head of the workspace: arrival counters in [0, kClassOffset), the 16-bit class records of every
// (index row, token) behind them, the [row][NTOK][8] accumulators from kCounterRegionBytes on
constexpr size_t kClassOffset = 16384;
static_assert(kClassOffset + (size_t(kMaxIndexRows) + 2 * kMaxFusedLayers) * 2 <= kCounterRegionBytes, "");
static_assert(kCounterRegionBytes + size_t(kMaxIndexRows) * 64 <= kZeroRegionBytes, "");

struct BatchLayer {
  const uint32_t* stream;  // [T][32] entry words
  const uint32_t* tab;     // [U + 1]
  const void* centroids;
  const void* res_centroids;
  const void* scale;  // ORIGINAL feature order (or nullptr: no scale / bias)
  const void* wbias;
  const void* bias;
  void* y;
  int64_t y_stride;
  unsigned long long* yacc;  // [Ro][NTOK][8] fixed-point (2^-30) accumulators, zero at rest
  uint32_t* counters;        // [ceil(Ro / kRB)], zero at rest
  uint16_t* cls;             // [Ro][NTOK] class records of unit sums kept out of yacc, zero at rest
  float lim;                 // unit sums with |v| >= lim (or not finite) are not added as integers
  int I, O, Ro, Kr, NS, Q, TCW;
  int k;  // CTAs per combo
};

struct BatchParams {
  int n, tokens;                             // fused layers, tokens of this launch (<= NTOK)
  uint32_t grid_begin[kMaxFusedLayers + 1];  // layer l owns blocks [grid_begin[l], grid_begin[l+1])
  const void* x;
  int64_t x_stride;
  int x_vec;  // rows of x are 16-byte aligned: 128-bit loads
  BatchLayer layer[kMaxFusedLayers];
  uint32_t off_bars, off_tab, off_red, off_piece, off_done, off_slice, off_res, off_x, off_ring;
  int stages;
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
// the NTOK 16-bit x' values of one column: one 32-, 64- or 128-bit shared access
template <int NTOK>
__device__ __forceinline__ void lds_tok(uint32_t (&w)[NTOK / 2], uint32_t a) {
  if constexpr (NTOK == 2) {
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w[0]) : "r"(a));
  } else if constexpr (NTOK == 4) {
    asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(w[0]), "=r"(w[1]) : "r"(a));
  } else {
    static_assert(NTOK == 8, "");
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]) : "r"(a));
  }
}
template <int NTOK>
__device__ __forceinline__ void sts_tok(uint32_t a, const uint32_t (&w)[NTOK / 2]) {
  if constexpr (NTOK == 2) {
    asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(w[0]) : "memory");
  } else if constexpr (NTOK == 4) {
    asm volatile("st.shared.v2.u32 [%0], {%1,%2};" ::"r"(a), "r"(w[0]), "r"(w[1]) : "memory");
  } else {
    asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(a), "r"(w[0]), "r"(w[1]), "r"(w[2]), "r"(w[3]) : "memory");
  }
}

// fp32 -> 2^-30 fixed point: the rounding costs up to 2^-31 per unit, a floor of Q * 2^-31 per output.  Only
// |v| < lim = 2^33 / 2^ceil(log2 Q) is admitted (no sum of Q admitted terms reaches 2^63); anything else leaves its
// class in the (row, token) record and the output becomes +inf, -inf or NaN.
constexpr float kFixScale = 1073741824.f, kFixInv = 1.f / 1073741824.f;
constexpr uint32_t kClsPosInf = 1u, kClsNegInf = 2u, kClsNaN = 3u;  // OR of two classes = class of their sum
__device__ __forceinline__ void record_class(uint16_t* rec, int e, float v) {
  const uint32_t c = v == INFINITY ? kClsPosInf : v == -INFINITY ? kClsNegInf : kClsNaN;
  const uintptr_t a = reinterpret_cast<uintptr_t>(rec);  // 16-bit record inside a 32-bit word
  atomicOr(reinterpret_cast<unsigned int*>(a & ~uintptr_t(3)), c << (uint32_t(a & 2u) * 8u + 2u * uint32_t(e)));
}
template <int NTOK>
__device__ __forceinline__ void add_unit(const BatchLayer& L, int row, int tok, int e, float v) {
  const bool in_range = fabsf(v) < L.lim;  // (false for inf and NaN)
  const long long q = __float2ll_rn((in_range ? v : 0.f) * kFixScale);
  const size_t rt = size_t(row) * NTOK + tok;
  asm volatile("red.global.add.u64 [%0], %1;" ::"l"(L.yacc + rt * 8 + e), "l"(q) : "memory");
  if (!in_range) record_class(L.cls + rt, e, v);
}

// acc[k][e] += x'_k * (c[e] + r[e]) for every token k: c + r formed once (fp16: packed fp16, bf16: fp32), then
// per token exactly the single-token kernel's FMAs
template <typename T, bool RES, int NTOK>
__device__ __forceinline__ void fma_tokens(float (&acc)[NTOK][8], const uint32_t (&xw)[NTOK / 2], const uint32_t (&cw)[4],
                                           const uint32_t (&rw)[4]) {
  float c[8];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
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
    for (int e = 0; e < 8; ++e) acc[k][e] = fmaf(xk, c[e], acc[k][e]);
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
__global__ void __launch_bounds__(kLT, 1) gemv_lists_batch_kernel(const __grid_constant__ BatchParams mp) {
  // steps whose gathers are in flight together: fewer at NTOK = 8, where the accumulators take 64 registers
  // (the per-lane FMA order is the step order whatever the batch is: results do not depend on it)
  constexpr int kSPS = NTOK >= 8 ? 2 : 4;
  extern __shared__ __align__(128) uint8_t smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int l = 0;
#pragma unroll
  for (int i = 1; i < kMaxFusedLayers; ++i)
    if (i < mp.n && blockIdx.x >= mp.grid_begin[i]) l = i;
  const BatchLayer& L = mp.layer[l];
  const int q = int(blockIdx.x - mp.grid_begin[l]);
  const int combo = q / L.k, jc = q - combo * L.k;
  const int Ro = L.Ro, TCW = L.TCW, I = L.I, ntok = mp.tokens, stages = mp.stages;
  const int r0 = int(int64_t(Ro) * jc / L.k), r1 = int(int64_t(Ro) * (jc + 1) / L.k);
  const int nun = r1 - r0;  // this CTA's units: rows [r0, r1) of one combo
  const int tile = combo / L.NS, slice = combo - tile * L.NS;

  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + mp.off_bars);
  uint32_t* s_tab = reinterpret_cast<uint32_t*>(smem + mp.off_tab);  // [nun + 1]
  float* s_red = reinterpret_cast<float*>(smem + mp.off_red);         // [warps][NTOK] bias partial sums
  float* s_cb = s_red + kLW * kMaxTok;                                // [NTOK] sum x * wbias of the tile
  int* s_ndone = reinterpret_cast<int*>(s_cb + kMaxTok);
  float* s_piece = reinterpret_cast<float*>(smem + mp.off_piece);                      // [warps][2][NTOK][8]
  int* s_pu = reinterpret_cast<int*>(smem + mp.off_piece + kLW * 2 * NTOK * 32);        // [warps][2]
  int* s_done = reinterpret_cast<int*>(smem + mp.off_done);                            // row blocks completed here
  uint8_t* s_slice = smem + mp.off_slice;
  uint8_t* s_res = smem + mp.off_res;
  const uint32_t s_x = smem_u32(smem + mp.off_x);  // [TCW][NTOK] 16-bit x'
  uint8_t* ring = smem + mp.off_ring + size_t(warp) * stages * kStageBytes;
  uint64_t* full = &bars[1 + warp * stages];

  const uint64_t pol_stream = policy_evict_first();
  const uint64_t pol_keep = policy_evict_last();
  if (tid == 0) {
    mbar_init(&bars[0], 1);
    fence_mbar_init();
    fence_proxy_async_smem();
    const uint8_t* cb = reinterpret_cast<const uint8_t*>(L.centroids);
    mbar_arrive_expect_tx(&bars[0], uint32_t(kSliceBytes));
    for (uint32_t off = 0; off < uint32_t(kSliceBytes); off += 32768u)
      tma_bulk_g2s(s_slice + off, cb + size_t(slice) * kSliceBytes + off, 32768u, &bars[0], pol_keep);
    *s_ndone = 0;
  } else if (tid < 1 + kLW * stages) {
    mbar_init(&bars[tid], 1);
    fence_mbar_init();
  }
  // residual codebook (<= 256 entries), stored 8 times: lane L reads copy L mod 8 (conflict-free quarter-warps)
  constexpr int kResFill = (256 * kResRep + kLT - 1) / kLT;
  uint4 res_entry[kResFill];
  if constexpr (RES) {
#pragma unroll
    for (int j = 0; j < kResFill; ++j) {
      const int slot = tid + j * kLT;
      res_entry[j] = make_uint4(0u, 0u, 0u, 0u);
      if (slot < L.Kr * kResRep)
        res_entry[j] = ldg_nc_v4(reinterpret_cast<const uint8_t*>(L.res_centroids) + (slot / kResRep) * 16, pol_keep);
    }
  }
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
  // x-independent work first: it overlaps the previous kernel's tail under programmatic dependent launch
  for (int qi = 0; qi < min(stages, nstage); ++qi) issue(qi, qi);
  if constexpr (RES) {
#pragma unroll
    for (int j = 0; j < kResFill; ++j) {
      const int slot = tid + j * kLT;
      if (slot < L.Kr * kResRep) sts_v4(smem_u32(s_res) + uint32_t(slot) * 16u, res_entry[j]);
    }
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
        uint32_t w[NTOK / 2];
#pragma unroll
        for (int k2 = 0; k2 < NTOK / 2; ++k2) {
          const uint32_t lo = (xq[2 * k2][i / 2] >> ((i & 1) * 16)) & 0xffffu;
          const uint32_t hi = (xq[2 * k2 + 1][i / 2] >> ((i & 1) * 16)) & 0xffffu;
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
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int k = 0; k < NTOK; ++k) {
      const float v = with_bias ? warp_sum(lane < kLW ? s_red[lane * kMaxTok + k] : 0.f) : 0.f;
      if (lane == 0) s_cb[k] = v;
    }
  }
  __syncthreads();
  mbar_wait(&bars[0], 0);

  // -------- main loop ---------------------------------------------------------------------------------
  if (nstage > 0) {
    const uint32_t res_lane = smem_u32(s_res) + uint32_t(lane & (kResRep - 1)) * 16u;
    const uint32_t ring_lane = smem_u32(ring) + uint32_t(lane) * 4u;
    const uint32_t slice_base = smem_u32(s_slice);
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
    float acc[NTOK][8];
#pragma unroll
    for (int k = 0; k < NTOK; ++k)
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[k][e] = 0.f;
    // the current unit's sums are final for this run: interior units go to global memory, the first and the last
    // unit of the run may be shared with the neighbouring warps and are parked for the merge below
    auto flush = [&](bool complete) {
      const bool boundary = u == uF || !complete || u_end >= t_end;
      const int kk = warp * 2 + (u == uF ? 0 : 1);
#pragma unroll
      for (int k = 0; k < NTOK; ++k) {
        if (k < ntok) {  // (warp-uniform)
          const float mine = warp_reduce_to_lane<8>(acc[k], lane);
          if (lane < 8) {
            if (!boundary) add_unit<NTOK>(L, r0 + u, k, lane, mine + s_cb[k]);
            else s_piece[(kk * NTOK + k) * 8 + lane] = mine;
          }
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[k][e] = 0.f;
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
        uint32_t ent[kSPS], cw[kSPS][4], rw[kSPS][4], xw[kSPS][NTOK / 2];
#pragma unroll
        for (int j = 0; j < kSPS; ++j)
          if (j < cnt) ent[j] = lds_u32(st + uint32_t(j) * 128u);
#pragma unroll
        for (int j = 0; j < kSPS; ++j) {
          if (j < cnt) {
            // entry = index12 | column12 << 12 | residual8 << 24
            lds_entry<8>(cw[j], mad_u32(ent[j] & 0xfffu, 16u, slice_base));
            if constexpr (RES) lds_entry<8>(rw[j], mad_u32(ent[j] >> 24, 128u, res_lane));
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
  for (int it = tid; it < kLW * 2 * NTOK * 8; it += kLT) {
    const int i = it / (NTOK * 8), k = (it >> 3) % NTOK, e = it & 7;
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
    float v = s_piece[(i * NTOK + k) * 8 + e];
    for (int j = i + 1; j < kLW * 2; ++j) {
      const int pj = s_pu[j];
      if (pj < 0) continue;
      if (pj != un) break;
      v += s_piece[(j * NTOK + k) * 8 + e];
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
    // this CTA's arrival completed nd row blocks: every unit of their rows has added its sums
    __threadfence();
    const T* bias = reinterpret_cast<const T*>(L.bias);
    const int nrow = nd * kRB;
    for (int i = tid; i < nrow * ntok; i += kLT) {
      const int k = i / nrow, ri = i - k * nrow;
      const int r = s_done[ri / kRB] * kRB + ri % kRB;
      if (r >= Ro) continue;
      const size_t rt = size_t(r) * NTOK + k;
      unsigned long long* p = L.yacc + rt * 8;
      long long qv[8];
      uint16_t cls;
      asm volatile("ld.global.cg.u16 %0, [%1];" : "=h"(cls) : "l"(L.cls + rt) : "memory");
#pragma unroll
      for (int h = 0; h < 4; ++h)
        asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(qv[2 * h]), "=l"(qv[2 * h + 1]) : "l"(p + 2 * h) : "memory");
#pragma unroll
      for (int h = 0; h < 4; ++h) *reinterpret_cast<ulonglong2*>(p + 2 * h) = make_ulonglong2(0ull, 0ull);  // zero at rest
      if (cls) L.cls[rt] = 0;
      const int o = r * 8;
      float v[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const uint32_t c = (uint32_t(cls) >> (2 * e)) & 3u;
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
    if (tid < nd) L.counters[s_done[tid]] = 0u;  // leave the counters zeroed for the next launch
  }
}

using BatchKernelFn = void (*)(const BatchParams);

template <typename T, int NTOK>
BatchKernelFn pick_batch_t(bool res) {
  return res ? gemv_lists_batch_kernel<T, true, NTOK> : gemv_lists_batch_kernel<T, false, NTOK>;
}
BatchKernelFn pick_batch(int dtype, bool res, int ntok) {
  if (dtype == VPTQ_FP16) {
    if (ntok == 2) return pick_batch_t<__half, 2>(res);
    if (ntok == 4) return pick_batch_t<__half, 4>(res);
    if (ntok == 8) return pick_batch_t<__half, 8>(res);
  } else if (dtype == VPTQ_BF16) {
    if (ntok == 2) return pick_batch_t<__nv_bfloat16, 2>(res);
    if (ntok == 4) return pick_batch_t<__nv_bfloat16, 4>(res);
    if (ntok == 8) return pick_batch_t<__nv_bfloat16, 8>(res);
  }
  return nullptr;
}

// smallest instance that holds `tokens`
int batch_instance(int tokens) { return tokens <= 2 ? 2 : tokens <= 4 ? 4 : 8; }

// What a launch of these layers looks like, for any token count.
struct BatchPlan {
  int n, Q, NS, TCW, I;
  int Ro[kMaxFusedLayers], k[kMaxFusedLayers];
  int rows, max_nun, max_kr, ctas;
  bool res;
};

// The partition (tokens never enter it): B = SM count / Q combo copies are shared out to the layers in proportion
// to their rows (at least one each, at most one CTA per row); integer comparisons, mirrored in
// tests/test_batch_decode_host.py.  0 or a vptq_status with the message set.
int batch_partition(int n, const vptq_linear_desc* const* descs, int sm_count, BatchPlan* pl) {
  if (n < 1 || n > kMaxFusedLayers || !descs) {
    set_error("quant_gemv_batch: 1..%d layers", kMaxFusedLayers);
    return VPTQ_ERR_UNSUPPORTED;
  }
  const vptq_linear_desc& d0 = *descs[0];
  pl->res = d0.num_res_centroids > 0;
  for (int l = 0; l < n; ++l) {
    const vptq_linear_desc& d = *descs[l];
    if (!gemv_lists_eligible(d) || d.dtype != d0.dtype || d.in_features != d0.in_features ||
        d.num_centroids != d0.num_centroids || (d.num_res_centroids > 0) != pl->res) {
      set_error("quant_gemv_batch: layer %d has no index lists the list kernels take, or does not match layer 0", l);
      return VPTQ_ERR_UNSUPPORTED;
    }
  }
  pl->n = n, pl->I = d0.in_features, pl->TCW = d0.lists_tile_cols;
  pl->NS = d0.num_centroids / kSliceEntries;
  pl->Q = pl->NS * ((pl->I + pl->TCW - 1) / pl->TCW);
  const int Q = pl->Q, B = sm_count / Q;
  if (n > B) {
    set_error("quant_gemv_batch: %d layers x %d combos exceed %d SMs", n, Q, sm_count);
    return VPTQ_ERR_UNSUPPORTED;
  }
  int64_t rows = 0;
  for (int l = 0; l < n; ++l) pl->Ro[l] = (descs[l]->out_features + 7) / 8, rows += pl->Ro[l];
  if (rows * kMaxTok > kMaxIndexRows) {
    set_error("quant_gemv_batch: %lld index rows x %d tokens exceed %d", (long long)rows, kMaxTok, kMaxIndexRows);
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
  pl->ctas = used * Q;
  pl->max_nun = 0, pl->max_kr = 0;
  for (int l = 0; l < n; ++l) {
    pl->max_nun = std::max(pl->max_nun, (Ro[l] + k[l] - 1) / k[l]);
    pl->max_kr = std::max(pl->max_kr, descs[l]->num_res_centroids > 0 ? descs[l]->num_res_centroids : 0);
  }
  size_t nblk = 0;
  for (int l = 0; l < n; ++l) nblk += size_t((Ro[l] + kRB - 1) / kRB);
  if (nblk * 4 > kClassOffset) {
    set_error("quant_gemv_batch: %zu row blocks exceed the counter region", nblk);
    return VPTQ_ERR_UNSUPPORTED;
  }
  return 0;
}

// shared-memory carve-up of instance NTOK; returns the bytes (0: nothing fits)
size_t batch_carve(const BatchPlan& pl, int ntok, size_t limit, BatchParams* mp) {
  for (int stages = 3; stages >= 2; --stages) {
    size_t off = 0;
    mp->off_bars = uint32_t(off), off += align_up(size_t(1 + kLW * stages) * 8, 128);
    mp->off_tab = uint32_t(off), off += align_up(size_t(pl.max_nun + 1) * 4, 128);
    mp->off_red = uint32_t(off), off += align_up(size_t(kLW + 1) * kMaxTok * 4 + 16, 128);
    mp->off_piece = uint32_t(off), off += align_up(size_t(kLW) * 2 * ntok * 32 + size_t(kLW) * 2 * 4, 128);
    mp->off_done = uint32_t(off), off += align_up(size_t(pl.max_nun / kRB + 2) * 4, 128);
    mp->off_slice = uint32_t(off), off += size_t(kSliceBytes);
    mp->off_res = uint32_t(off), off += align_up(size_t(pl.max_kr) * 16 * kResRep, 128);
    mp->off_x = uint32_t(off), off += align_up(size_t(pl.TCW) * ntok * 2, 128);
    mp->off_ring = uint32_t(off), off += size_t(kLW) * stages * kStageBytes;
    mp->stages = stages;
    if (off <= limit) return off;
  }
  return 0;
}

}  // namespace

int gemv_lists_batch_max_tokens(int n, const vptq_linear_desc* const* descs) {
  const DeviceInfo* dev = device_info();
  if (!dev) return 0;
  BatchPlan pl;
  if (batch_partition(n, descs, dev->sm_count, &pl)) return 0;
  BatchParams mp{};
  if (!batch_carve(pl, kMaxTok, size_t(dev->smem_optin), &mp)) {
    set_error("quant_gemv_batch: no shared-memory layout fits");
    return 0;
  }
  return kMaxTok;
}

int gemv_lists_batch_launch(int n, const vptq_linear_desc* const* descs, const void* x, int64_t x_stride,
                            void* const* ys, const int64_t* y_strides, int tokens, uint32_t flags, cudaStream_t stream,
                            void* workspace, size_t workspace_bytes) {
  const DeviceInfo* dev = device_info();
  if (!dev) return VPTQ_ERR_CUDA;
  BatchPlan pl;
  if (int rc = batch_partition(n, descs, dev->sm_count, &pl)) return rc;
  if (tokens < 1 || tokens > kMaxTok) {
    set_error("quant_gemv_batch: %d tokens (1..%d)", tokens, kMaxTok);
    return VPTQ_ERR_UNSUPPORTED;
  }
  if (reinterpret_cast<uintptr_t>(x) & 15u) {
    set_error("quant_gemv_batch: x must be 16-byte aligned");
    return VPTQ_ERR_UNSUPPORTED;
  }
  if (!workspace || workspace_bytes < kZeroRegionBytes) {
    set_error("quant_gemv_batch: workspace %zu bytes < required %zu", workspace_bytes, kZeroRegionBytes);
    return VPTQ_ERR_WORKSPACE;
  }
  const int ntok = batch_instance(tokens);
  BatchKernelFn fn = pick_batch(descs[0]->dtype, pl.res, ntok);
  if (!fn) return VPTQ_ERR_UNSUPPORTED;
  BatchParams mp{};
  const size_t need = batch_carve(pl, ntok, size_t(dev->smem_optin), &mp);
  if (!need) {
    set_error("quant_gemv_batch: no shared-memory layout fits");
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
    BatchLayer& L = mp.layer[l];
    L.stream = reinterpret_cast<const uint32_t*>(d.lists_stream), L.tab = d.lists_tab;
    L.centroids = d.centroids, L.res_centroids = d.res_centroids;
    L.scale = d.weight_scale, L.wbias = d.weight_scale ? d.weight_bias : nullptr;
    L.bias = d.bias, L.y = ys[l], L.y_stride = y_strides[l];
    L.I = pl.I, L.O = d.out_features, L.Ro = pl.Ro[l], L.Kr = d.num_res_centroids > 0 ? d.num_res_centroids : 0;
    L.NS = pl.NS, L.Q = pl.Q, L.TCW = pl.TCW, L.k = pl.k[l];
    L.yacc = reinterpret_cast<unsigned long long*>(wsb + acc_off);
    L.counters = reinterpret_cast<uint32_t*>(wsb + ctr_off);
    L.cls = reinterpret_cast<uint16_t*>(wsb + cls_off);
    L.lim = std::ldexp(1.f, 33 - lg_q);
    acc_off += size_t(pl.Ro[l]) * ntok * 64;
    ctr_off += size_t((pl.Ro[l] + kRB - 1) / kRB) * 4;
    cls_off += size_t(pl.Ro[l]) * ntok * 2;  // (ntok even: whole 32-bit words per layer)
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
    set_error("quant_gemv_batch launch (grid=%u smem=%zu): %s", begin, need, cudaGetErrorString(e));
    return VPTQ_ERR_CUDA;
  }
  return 0;
}

}  // namespace vptq_b200
