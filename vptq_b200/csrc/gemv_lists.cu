// Decode GEMV (one token) for layers with a large main codebook (K = NS * 4096 entries, NS = 2..16: up to the
// 1 MiB codebook of K = 65536), reading the slice x tile lists of vptq_linear_desc::lists_* (built at load
// time by vptq_b200/lists.py or vptq_b200_lists_build_host).
//
// The generic kernel (gemv_kernel.cuh) gathers such a codebook through L1/L2 and is bound by the L1TEX tag
// stage, far below the HBM roofline.
// Here every gather is a shared-memory access, and there is no cluster (every SM works), no perm / dependent
// gather in the prologue, a 4-byte entry, and the
// x' tile is bounded by 4096 columns, so any in_features fits:
//   * work item = unit u = (tile t, slice s, index row r): the fields of row r whose main index lies in slice
//     s (64 KiB of the codebook) and whose ORIGINAL input feature lies in column tile t (<= 4096 features).
//     combo = t * NS + s; units are numbered combo-major and their lists are contiguous in that order;
//   * a launch spreads the U units of a layer evenly over its CTAs (one per SM).  A CTA's range is contiguous
//     and touches at most two combos ("segments" A and B): it stages one or two codebook slices (TMA bulk
//     copies), the 8x bank-replicated residual table and one or two x' tiles (x[f] * scale[f], a coalesced
//     128-bit load per thread -- perm was folded into the entries at load time);
//   * the CTA cuts its step range (32 entries per step) into 16 equal runs, one per warp, whatever the unit
//     boundaries are.  A warp streams its run through a private TMA ring (8 steps = 1 KiB per stage) and works in
//     batches of 4 steps (12 gathers in flight per lane; where a unit ends inside a batch the flush sits at a
//     compile-time position: five straight-line batch variants, no per-step test); per
//     entry a lane does LDS.32 (entry), LDS.128 (main), LDS.128 (residual), LDS.U16 (x'), then c + r in
//     packed 16-bit arithmetic (exactly the reference's ADD2, csrc/kernels/quant_gemv.cuh:124-127) and 8
//     FMAs into fp32 accumulators;
//   * a unit that lies inside one warp's run is reduced with 9 shuffles; the (at most two) units a run shares
//     with its neighbours are parked in shared memory and merged in warp order;
//   * reduction over the Q = NS * NT combos of a row: every unit adds its 8 sums, converted to 2^-30 fixed
//     point, into a 64-bit accumulator row in the workspace with red.global.add.u64.  Integer addition is
//     associative, so the result does not depend on the arrival order: bit-identical from run to run, like
//     an ordered sum, without a partial-sum table (a last-arriver that adds Q partials per output was
//     measured at 4-8 us of tail per launch).  Row blocks of 32 index rows carry an arrival counter (units,
//     not CTAs); the CTA whose arrival completes a block converts its rows back, adds bias, writes y and
//     zeroes the accumulators and the counter again.  No second kernel (the reference launches `sum(-1)`,
//     csrc/quant_gemv.cu:235), no spinning on other CTAs;
//   * tensor parallelism (vptq_tp_exchange): the thread that completes an index row also stores it into every
//     peer's buffer over NVLink -- as tagged 8-byte words {2 values, tag} that the consumer launch re-reads
//     until the tag is current (no fence, no flag, no NCCL call), or plain + epoch flags.
// Measured variants that lost (more warps with smaller batches, entry prefetch, returning atomics, a scan of
// the touched rows instead of counters) are listed in DESIGN.md section 3.
// Mathematics and reference citations: gemv_kernel.cuh (the reference's kernel is
// csrc/kernels/quant_gemv.cuh:11-186; nothing of its structure is used here).
#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <type_traits>

#include "gemv_kernel.cuh"

namespace vptq_b200 {

namespace {

constexpr int kSliceEntries = 4096;
constexpr int kSliceBytes = kSliceEntries * 16;  // 64 KiB
constexpr int kTileMax = 4096;
#ifndef VPTQ_LISTS_WARPS
#define VPTQ_LISTS_WARPS 16
#endif
#ifndef VPTQ_LISTS_BATCH
#define VPTQ_LISTS_BATCH 4
#endif
constexpr int kLW = VPTQ_LISTS_WARPS, kLT = kLW * 32;  // warps, threads per CTA
constexpr int kSPS = VPTQ_LISTS_BATCH;   // steps (32 entries, 128 bytes each) per batch: loads of kSPS steps in flight
static_assert(kSPS >= 2 && kSPS <= 4 && kLW <= 32, "batch variants are written out for 2..4 steps");
constexpr int kEnd3 = kSPS >= 3 ? 3 : 2;  // (switch label 3 is unreachable for 2-step batches)
constexpr int kBPS = 2;                  // batches per ring stage (one TMA copy / one barrier wait per 8 steps)
constexpr int kStSteps = kSPS * kBPS;
constexpr int kStageBytes = kStSteps * 128;
constexpr int kMaxWindow = 3072;  // units of one CTA (bounds the tab window in shared memory)
constexpr int kRB = 32;           // index rows per arrival counter
constexpr int kResRep = 8;        // bank-group replication of the residual table
constexpr uint32_t kStepMask = (1u << 26) - 1u;

struct ListsLayer {
  const uint32_t* stream;  // [T][32] entry words
  const uint32_t* tab;     // [U + 1]
  const void* centroids;
  const void* res_centroids;
  const void* scale;  // ORIGINAL feature order (or nullptr: no scale / bias)
  const void* wbias;
  const void* bias;
  void* y;
  unsigned long long* yacc;  // [Ro][8] fixed-point (2^-30) accumulators, zero at rest
  uint32_t* counters;        // [ceil(Ro / kRB)], zero at rest
  int I, O, Ro, Kr, NS, Q, TCW, U;
  int ncta;  // CTAs working on this layer
};

struct ListsParams {
  int n;                                     // fused layers
  uint32_t grid_begin[kMaxFusedLayers + 1];  // layer l owns blocks [grid_begin[l], grid_begin[l+1])
  const void* x;
  ListsLayer layer[kMaxFusedLayers];
  // shared-memory carve-up (bytes)
  uint32_t off_bars, off_tab, off_red, off_piece, off_done, off_slice, off_res, off_x, off_ring;
  int stages;
  unsigned long long* prof;  // developer aid: %globaltimer stamps of the first / last CTA (or nullptr)
  // tensor-parallel exchange over peer memory (tp_world <= 1: off), same protocol as the generic kernel
  // (gemv_kernel.cuh): every output row is stored locally and into all peers' buffers, the last CTA of the
  // launch publishes the launch's epoch in every peer's flag array, a launch with tp_wait_slot >= 0 polls the
  // flags of the launch that produced its x before reading it
  int tp_world, tp_rank, tp_slot, tp_wait_slot;
  void* tp_peer_y[kMaxFusedLayers][8];  // [layer][rank]: start of THIS rank's slice in rank r's y
  uint32_t* tp_peer_flags[8];           // rank r's flag array [slots][world]
  uint32_t* tp_epoch;                   // local: completed runs per launch slot
  uint32_t* tp_done;                    // local: CTA arrival counters per launch slot (zero at rest)
  uint32_t* tp_error;                   // local: set when a flag wait timed out
  int tp_format, tp_nslots;             // VPTQ_TP_PLAIN / VPTQ_TP_TAGGED; launches per token (tag arithmetic)
};

__device__ __forceinline__ uint32_t lds_u32(uint32_t a) {
  uint32_t r;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(r) : "r"(a));
  return r;
}
__device__ __forceinline__ uint16_t lds_u16(uint32_t a) {
  uint16_t r;
  asm volatile("ld.shared.u16 %0, [%1];" : "=h"(r) : "r"(a));
  return r;
}
// a * b + c in one integer instruction (IMAD), so that mask -> scale -> add-base is two instructions, not three
__device__ __forceinline__ uint32_t mad_u32(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t r;
  asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
  return r;
}
// fp32 -> 2^-30 fixed point (saturating) and back; |v| < 2^33 is far beyond any 16-bit activation
constexpr float kFixScale = 1073741824.f, kFixInv = 1.f / 1073741824.f;
__device__ __forceinline__ void red_add_fixed(unsigned long long* p, float v) {
  const long long q = __float2ll_rn(v * kFixScale);
  asm volatile("red.global.add.u64 [%0], %1;" ::"l"(p), "l"(q) : "memory");
}
// acc[e] += x' * (c[e] + r[e]).  fp16: c + r in packed fp16 (the reference's ADD2), fp32 accumulation: the
// fp16 x fp16 product is exact in fp32, so widening both factors and one fp32 FMA round exactly once.
// bf16: c + r and the product in fp32 (x' is kept as fp16 in shared memory for both dtypes).
template <typename T, bool RES>
__device__ __forceinline__ void fma_entry(float (&acc)[8], uint16_t xh, const uint32_t (&cw)[4], const uint32_t (&rw)[4]) {
  if constexpr (std::is_same<T, __half>::value) {
    const float xv = __half2float(__ushort_as_half(xh));
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 c = DT<T>::unpack2(RES ? DT<T>::add2(cw[i], rw[i]) : cw[i]);
      acc[2 * i] = fmaf(xv, c.x, acc[2 * i]);
      acc[2 * i + 1] = fmaf(xv, c.y, acc[2 * i + 1]);
    }
  } else {
    const float xv = __half2float(__ushort_as_half(xh));
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float2 c = DT<T>::unpack2(cw[i]);
      if constexpr (RES) {
        const float2 r = DT<T>::unpack2(rw[i]);
        c.x += r.x, c.y += r.y;
      }
      acc[2 * i] = fmaf(xv, c.x, acc[2 * i]);
      acc[2 * i + 1] = fmaf(xv, c.y, acc[2 * i + 1]);
    }
  }
}

// 8 consecutive 16-bit elements p[f .. f+8) as one 128-bit load; elements at or beyond fend read as `fill`
template <typename T>
__device__ __forceinline__ uint4 load8(const T* p, int f, int fend, uint16_t fill) {
  if (f + 8 <= fend) return *reinterpret_cast<const uint4*>(p + f);
  uint16_t h[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) h[k] = (f + k < fend) ? reinterpret_cast<const uint16_t*>(p)[f + k] : fill;
  return make_uint4(h[0] | uint32_t(h[1]) << 16, h[2] | uint32_t(h[3]) << 16, h[4] | uint32_t(h[5]) << 16,
                    h[6] | uint32_t(h[7]) << 16);
}

// VPTQ_TP_TAGGED: 8 consecutive activations = four 8-byte words {2 values, tag}, written by any rank with aligned
// 16-byte stores (each 8-byte half lands atomically).  Re-read until all four tags are the expected one.
__device__ __forceinline__ uint4 load8_tagged(const void* xl, int f, uint32_t tag, uint32_t* error) {
  const uint8_t* p = reinterpret_cast<const uint8_t*>(xl) + size_t(f) * 4;
  uint4 a, b;
  const long long t0 = clock64();
  for (;;) {
    asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w) : "l"(p) : "memory");
    asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(b.x), "=r"(b.y), "=r"(b.z), "=r"(b.w)
                 : "l"(p + 16)
                 : "memory");
    if (a.y == tag && a.w == tag && b.y == tag && b.w == tag) break;
    if (ld_volatile_u32(error) != 0u) break;
    if (clock64() - t0 > (1ll << 32)) {  // ~2 s: give up loudly instead of hanging the GPU
      *error = 1u;
      break;
    }
  }
  return make_uint4(a.x, a.z, b.x, b.z);
}

// x' = x * scale for 8 features (stored as fp16) and sum x * wbias (fp32)
template <typename T>
__device__ __forceinline__ uint4 make_xq(const uint4& xr, const uint4& sc, const uint4& wb, bool with_bias, float& bs) {
  const uint32_t xs[4] = {xr.x, xr.y, xr.z, xr.w}, ss[4] = {sc.x, sc.y, sc.z, sc.w}, ws[4] = {wb.x, wb.y, wb.z, wb.w};
  uint32_t o[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 xf = DT<T>::unpack2(xs[i]);
    if constexpr (std::is_same<T, __half>::value) {
      // the product rounded to fp16, as the reference forms input_v (csrc/kernels/quant_gemv.cuh:56)
      __half2 p = __hmul2(*reinterpret_cast<const __half2*>(&xs[i]), *reinterpret_cast<const __half2*>(&ss[i]));
      o[i] = *reinterpret_cast<uint32_t*>(&p);
    } else {
      const float2 sf = DT<T>::unpack2(ss[i]);
      __half2 p = __floats2half2_rn(xf.x * sf.x, xf.y * sf.y);
      o[i] = *reinterpret_cast<uint32_t*>(&p);
    }
    if (with_bias) {
      const float2 wf = DT<T>::unpack2(ws[i]);
      bs = fmaf(xf.x, wf.x, bs);
      bs = fmaf(xf.y, wf.y, bs);
    }
  }
  return make_uint4(o[0], o[1], o[2], o[3]);
}

template <typename T, bool RES>
__global__ void __launch_bounds__(kLT, 1) gemv_lists_kernel(const __grid_constant__ ListsParams mp) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int l = 0;
#pragma unroll
  for (int i = 1; i < kMaxFusedLayers; ++i)
    if (i < mp.n && blockIdx.x >= mp.grid_begin[i]) l = i;
  const ListsLayer& L = mp.layer[l];
  const int q = int(blockIdx.x - mp.grid_begin[l]);
  const int Ro = L.Ro, NS = L.NS, TCW = L.TCW, I = L.I, stages = mp.stages;
  // this CTA's units [u0, u1): at most two combos (host: ncta >= Q, so u1 - u0 <= Ro)
  const int u0 = int(int64_t(L.U) * q / L.ncta), u1 = int(int64_t(L.U) * (q + 1) / L.ncta);
  const int nun = u1 - u0;
  const int cA = u0 / Ro, cB = (u1 - 1) / Ro;
  const bool two = cB != cA;
  const int nA = two ? cB * Ro - u0 : nun;  // units of segment A
  const int rA0 = u0 - cA * Ro;             // its first index row (segment B starts at row 0)
  const int tA = cA / NS, sA = cA - tA * NS, tB = cB / NS, sB = cB - tB * NS;
  const bool xB_own = two && tB != tA;  // segment B reads another x' tile (then sB == 0)

  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + mp.off_bars);
  uint32_t* s_tab = reinterpret_cast<uint32_t*>(smem + mp.off_tab);      // [nun + 1]
  float* s_red = reinterpret_cast<float*>(smem + mp.off_red);             // [32] bias partial sums
  int* s_ndone = reinterpret_cast<int*>(smem + mp.off_red + 128);
  float* s_piece = reinterpret_cast<float*>(smem + mp.off_piece);         // [warps][2][8]
  int* s_pu = reinterpret_cast<int*>(smem + mp.off_piece + kLW * 2 * 32);  // [warps][2] unit of each piece
  int* s_done = reinterpret_cast<int*>(smem + mp.off_done);               // row blocks this CTA completes
  uint8_t* s_slice = smem + mp.off_slice;                                 // two slices
  uint8_t* s_res = smem + mp.off_res;
  // two x' tiles (fp16, 8 KiB apart), the first on an 8 KiB boundary of the shared window
  const uint32_t s_x = (smem_u32(smem + mp.off_x) + 8191u) & ~8191u;
  uint8_t* ring = smem + mp.off_ring + size_t(warp) * stages * kStageBytes;
  uint64_t* full = &bars[2 + warp * stages];

  auto stamp = [&](int slot) {
#ifdef VPTQ_B200_PROF_WARPS
    if (mp.prof && tid == 0 && blockIdx.x == 0) {
#else
    if (mp.prof && tid == 0 && (blockIdx.x == 0 || blockIdx.x == gridDim.x - 1)) {
#endif
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      mp.prof[(blockIdx.x == 0 ? 0 : 16) + slot] = t;
    }
  };
  stamp(0);
  const uint64_t pol_stream = policy_evict_first();
  const uint64_t pol_keep = policy_evict_last();

  // -------- barriers; the slice copies leave at once (their issuer initialised their barriers) ----------
  if (tid == 0) {
    mbar_init(&bars[0], 1);
    mbar_init(&bars[1], 1);
    fence_mbar_init();
    fence_proxy_async_smem();
    const uint8_t* cb = reinterpret_cast<const uint8_t*>(L.centroids);
    mbar_arrive_expect_tx(&bars[0], uint32_t(kSliceBytes));
    for (uint32_t off = 0; off < uint32_t(kSliceBytes); off += 32768u)
      tma_bulk_g2s(s_slice + off, cb + size_t(sA) * kSliceBytes + off, 32768u, &bars[0], pol_keep);
    if (two) {
      mbar_arrive_expect_tx(&bars[1], uint32_t(kSliceBytes));
      for (uint32_t off = 0; off < uint32_t(kSliceBytes); off += 32768u)
        tma_bulk_g2s(s_slice + kSliceBytes + off, cb + size_t(sB) * kSliceBytes + off, 32768u, &bars[1], pol_keep);
    }
    *s_ndone = 0;
  } else if (tid >= 2 && tid < 2 + kLW * stages) {
    mbar_init(&bars[tid], 1);
    fence_mbar_init();
  }
  // residual codebook (<= 256 entries of 16 bytes), stored 8 times: copy k of entry i sits at 16-byte slot
  // i*8 + k and lane L reads copy L mod 8, so the 8 lanes of a quarter-warp always hit 8 different bank groups.
  // Thread t fills slots t, t + 512, ...: consecutive lanes write consecutive slots (conflict-free stores).
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
  // list table of this CTA's units
  for (int i = tid; i <= nun; i += kLT) s_tab[i] = L.tab[u0 + i];
  // x-independent column data: scale (and weight_bias where this CTA owns the bias term) of the tile(s)
  const T* scale = reinterpret_cast<const T*>(L.scale);
  const T* wbias = reinterpret_cast<const T*>(L.wbias);
  const uint16_t one16 = std::is_same<T, __half>::value ? uint16_t(0x3c00u) : uint16_t(0x3f80u);
  const uint32_t one32 = uint32_t(one16) | uint32_t(one16) << 16;
  const int j0 = tid * 8;  // column of the tile this thread prepares
  const bool colA = j0 < TCW && tA * TCW + j0 < I;
  const bool colB = xB_own && j0 < TCW && tB * TCW + j0 < I;
  const int fA = tA * TCW + j0, fAend = min(I, (tA + 1) * TCW);
  const int fB = tB * TCW + j0, fBend = min(I, (tB + 1) * TCW);
  const bool biasA = scale != nullptr && sA == 0, biasB = scale != nullptr && xB_own;
  uint4 scA = make_uint4(one32, one32, one32, one32), scB = scA;
  uint4 wbA = make_uint4(0u, 0u, 0u, 0u), wbB = wbA;
  if (scale) {
    if (colA) scA = load8<T>(scale, fA, fAend, one16);
    if (colB) scB = load8<T>(scale, fB, fBend, one16);
    if (colA && biasA) wbA = load8<T>(wbias, fA, fAend, 0);
    if (colB && biasB) wbB = load8<T>(wbias, fB, fBend, 0);
  }
  if (lane == 0) s_pu[warp * 2] = -1, s_pu[warp * 2 + 1] = -1;
  __syncthreads();
  stamp(1);
  pdl_launch_dependents();

  // -------- this warp's run of steps: an equal share of the CTA's contiguous step range ----------------
  const int T0 = int(s_tab[0] & kStepMask), T1 = int(s_tab[nun] & kStepMask), TT = T1 - T0;
  const int t_begin = T0 + int(int64_t(TT) * warp / kLW), t_end = T0 + int(int64_t(TT) * (warp + 1) / kLW);
  const int TB = two ? int(s_tab[nA] & kStepMask) : T1;  // first step of segment B
  // the run as a sequence of ring stages; a stage never straddles the segment boundary
  const int e1 = min(t_end, TB), b2 = max(t_begin, TB);
  const int n1 = (max(e1 - t_begin, 0) + kStSteps - 1) / kStSteps, n2 = (max(t_end - b2, 0) + kStSteps - 1) / kStSteps;
  const int nstage = n1 + n2;
  auto stage_at = [&](int qi, int& t, int& cnt) {
    if (qi < n1) t = t_begin + qi * kStSteps, cnt = min(kStSteps, e1 - t);
    else t = b2 + (qi - n1) * kStSteps, cnt = min(kStSteps, t_end - t);
  };
  // warp-collective: start the copy of stage qi of the run into ring slot `slot` (= qi mod stages)
  auto issue = [&](int qi, int slot) {
    if (lane == 0) {  // (the slot was only READ through the generic proxy before)
      int t, cnt;
      stage_at(qi, t, cnt);
      mbar_arrive_expect_tx(&full[slot], uint32_t(cnt) * 128u);
      tma_bulk_g2s(ring + size_t(slot) * kStageBytes, L.stream + size_t(t) * 32, uint32_t(cnt) * 128u, &full[slot],
                   pol_stream);
    }
  };
  // -------- everything that does not depend on x is queued first: the ring copies of this warp's first stages and
  // the replicated residual table -- a CTA usually starts a few microseconds before the previous kernel has
  // finished, so this is hidden behind griddepcontrol.wait -----------------------------------------------------
  for (int qi = 0; qi < min(stages, nstage); ++qi) issue(qi, qi);

  if constexpr (RES) {
#pragma unroll
    for (int j = 0; j < kResFill; ++j) {
      const int slot = tid + j * kLT;
      if (slot < L.Kr * kResRep) sts_v4(smem_u32(s_res) + uint32_t(slot) * 16u, res_entry[j]);
    }
  }
  // -------- x arrives from the previous kernel: one coalesced 128-bit load per thread ---------------------------
  pdl_wait_prior_grid();
  const bool tagged = mp.tp_world > 1 && mp.tp_format == VPTQ_TP_TAGGED;
  // tag of the words this launch writes / expects in its x: run number * launches per token + slot + 1
  const uint32_t run = mp.tp_world > 1 ? ld_volatile_u32(mp.tp_epoch + mp.tp_slot) : 0u;
  const uint32_t tag_out = run * uint32_t(mp.tp_nslots) + uint32_t(mp.tp_slot) + 1u;
  const uint32_t tag_in = run * uint32_t(mp.tp_nslots) + uint32_t(mp.tp_wait_slot) + 1u;
  if (mp.tp_world > 1 && mp.tp_wait_slot >= 0 && !tagged) {
    // x is assembled from every rank's slice: wait until all peers have published the epoch of the launch
    // that produces it (= this launch's own run number: both run once per token).  A wait that times out
    // (~2 s) sets the error word, which the host checks; once it is set nobody waits any more.
    if (tid < mp.tp_world && tid != mp.tp_rank) {
      const uint32_t want = run + 1u;
      const uint32_t* flag = mp.tp_peer_flags[mp.tp_rank] + mp.tp_wait_slot * mp.tp_world + tid;
      const long long t0 = clock64();
      while (ld_acquire_sys_u32(flag) < want) {
        if (ld_volatile_u32(mp.tp_error) != 0u) break;
        if (clock64() - t0 > (1ll << 32)) {
          *mp.tp_error = 1u;
          break;
        }
      }
    }
    __syncthreads();
  }
  stamp(2);
  const T* x = reinterpret_cast<const T*>(mp.x);
  uint4 xa = make_uint4(0u, 0u, 0u, 0u), xb = xa;
  if (tagged && mp.tp_wait_slot >= 0) {
    // (in_features % 8 == 0 is checked on the host: whole 8-feature groups only)
    if (colA) xa = load8_tagged(mp.x, fA, tag_in, mp.tp_error);
    if (colB) xb = load8_tagged(mp.x, fB, tag_in, mp.tp_error);
  } else {
    if (colA) xa = load8<T>(x, fA, fAend, 0);
    if (colB) xb = load8<T>(x, fB, fBend, 0);
  }
  stamp(3);
  // -------- x'[f] = x[f] * scale[f] -------------------------------------------------------------------------
  {
    float bsA = 0.f, bsB = 0.f;
    if (colA) sts_v4(s_x + uint32_t(j0) * 2u, make_xq<T>(xa, scA, wbA, biasA, bsA));
    if (colB) sts_v4(s_x + 8192u + uint32_t(j0) * 2u, make_xq<T>(xb, scB, wbB, biasB, bsB));
    if (biasA) {  // (CTA-uniform conditions)
      const float v = warp_sum(bsA);
      if (lane == 0) s_red[warp] = v;
    }
    if (biasB) {
      const float v = warp_sum(bsB);
      if (lane == 0) s_red[kLW + warp] = v;
    }
  }
  __syncthreads();
  // sum_f x[f] * wbias[f] over the tile: added once per index row, by the slice-0 combo of the tile
  float cbiasA = 0.f, cbiasB = 0.f;
  if (biasA) cbiasA = warp_sum(lane < kLW ? s_red[lane] : 0.f);
  if (biasB) cbiasB = warp_sum(lane < kLW ? s_red[kLW + lane] : 0.f);
  stamp(4);
  mbar_wait(&bars[0], 0);
  if (two) mbar_wait(&bars[1], 0);
  stamp(5);

  // -------- main loop ---------------------------------------------------------------------------------
  if (nstage > 0) {
    const uint32_t res_lane = smem_u32(s_res) + uint32_t(lane & (kResRep - 1)) * 16u;
    const uint32_t ring_lane = smem_u32(ring) + uint32_t(lane) * 4u;
    // the unit this run starts in: the last i with first(i) <= t_begin (every unit has >= 1 step)
    int u;
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
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
    float cb = 0.f;
    // the current unit's sums are final for this run: interior units go to global memory, the first and the
    // last unit of the run may be shared with the neighbouring warps and are parked for the merge below
    auto flush = [&](bool complete) {
      const float mine = warp_reduce_to_lane<8>(acc, lane);
      const bool boundary = u == uF || !complete || u_end >= t_end;
      if (!boundary) {
        if (lane < 8) red_add_fixed(L.yacc + size_t(u < nA ? rA0 + u : u - nA) * 8 + lane, mine + cb);
      } else {
        const int k = warp * 2 + (u == uF ? 0 : 1);
        if (lane < 8) s_piece[k * 8 + lane] = mine;
        if (lane == 0) s_pu[k] = u;
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] = 0.f;
    };
    auto advance = [&]() {
      ++u;
      if (u < nun) {
        u_end = int(s_tab[u + 1] & kStepMask);
        tail = s_tab[u] >> 26;
      }
    };
    int slot = 0, qi = 0, t = 0;
    uint32_t par = 0;
    uint32_t slice_base = 0, x_base = 0;
    // One batch = up to kSPS steps of a ring stage: all entry words, then all gathers, then the arithmetic.
    //   KEND = 0: no unit ends inside the batch (straight-line FMAs)
    //   KEND = k in 1..kSPS (full batches only): the current unit ends with the batch's k-th step and the next
    //             one does not end inside the batch -- the flush sits at a fixed place, no per-step test
    //   KEND < 0: generic (partial batches at the end of a run / segment, units shorter than a batch)
    auto batch = [&](auto kend_tag, int cnt, uint32_t st) {
      constexpr int KEND = decltype(kend_tag)::value;
      constexpr bool FULL = KEND >= 0;
      uint32_t ent[kSPS];
      uint32_t cw[kSPS][4], rw[kSPS][4];
      uint16_t xh[kSPS];
#pragma unroll
      for (int j = 0; j < kSPS; ++j)
        if (FULL || j < cnt) ent[j] = lds_u32(st + uint32_t(j) * 128u);
#pragma unroll
      for (int j = 0; j < kSPS; ++j) {
        if (FULL || j < cnt) {
          // entry = index12 | column12 << 12 | residual8 << 24; x_base is 8 KiB aligned, so `|` adds
          lds_entry<8>(cw[j], mad_u32(ent[j] & 0xfffu, 16u, slice_base));
          if constexpr (RES) lds_entry<8>(rw[j], mad_u32(ent[j] >> 24, 128u, res_lane));
          xh[j] = lds_u16(x_base | ((ent[j] >> 11) & 0x1ffeu));
        }
      }
      if constexpr (KEND == 0) {
#pragma unroll
        for (int j = 0; j < kSPS; ++j) fma_entry<T, RES>(acc, xh[j], cw[j], rw[j]);
        t += kSPS;
      } else if constexpr (KEND > 0) {
#pragma unroll
        for (int j = 0; j < kSPS; ++j) {
          uint16_t xv = xh[j];
          if (j == KEND - 1 && uint32_t(lane) >= tail) xv = 0;  // last step of the unit: mask the padding entries
          fma_entry<T, RES>(acc, xv, cw[j], rw[j]);
          if (j == KEND - 1) {
            flush(true);
            advance();
          }
        }
        t += kSPS;
      } else {
#pragma unroll
        for (int j = 0; j < kSPS; ++j) {
          if (j < cnt) {
            const bool last = t + 1 == u_end;
            uint16_t xv = xh[j];
            if (last && uint32_t(lane) >= tail) xv = 0;
            fma_entry<T, RES>(acc, xv, cw[j], rw[j]);
            ++t;
            if (last) {
              flush(true);
              advance();
            }
          }
        }
      }
    };
#pragma unroll 1
    for (int part = 0; part < 2; ++part) {
      // part 0 = this run's steps in segment A, part 1 = its steps in segment B (a stage never straddles both)
      const int np = part ? n2 : n1;
      if (np == 0) continue;
      t = part ? b2 : t_begin;
      const int pe = part ? t_end : e1;
      slice_base = smem_u32(s_slice) + (part ? uint32_t(kSliceBytes) : 0u);
      x_base = s_x + ((part && xB_own) ? 8192u : 0u);
      cb = part ? cbiasB : cbiasA;
#pragma unroll 1
      for (int si = 0; si < np; ++si, ++qi) {
        mbar_wait(&full[slot], par);
        uint32_t st = ring_lane + uint32_t(slot) * uint32_t(kStageBytes);
#pragma unroll 1
        for (int bi = 0; bi < kBPS && t < pe; ++bi, st += uint32_t(kSPS) * 128u) {
          const int cnt = min(kSPS, pe - t);
          const int k = u_end - t;  // steps left in the current unit (>= 1)
          if (cnt == kSPS && k > kSPS) {
            batch(std::integral_constant<int, 0>{}, cnt, st);
          } else if (cnt == kSPS && !(u + 1 < nun && int(s_tab[u + 2] & kStepMask) - t <= kSPS)) {
            switch (k) {
              case 1: batch(std::integral_constant<int, 1>{}, cnt, st); break;
              case 2: batch(std::integral_constant<int, 2>{}, cnt, st); break;
              case 3: batch(std::integral_constant<int, kEnd3>{}, cnt, st); break;
              default: batch(std::integral_constant<int, kSPS>{}, cnt, st); break;
            }
          } else {
            batch(std::integral_constant<int, -1>{}, cnt, st);
          }
        }
        __syncwarp();  // every lane has read its words of the stage: refill it
        if (qi + stages < nstage) issue(qi + stages, slot);
        if (++slot == stages) slot = 0, par ^= 1u;
      }
    }
    // the run ended inside a unit: its sums so far are this warp's piece of that unit
    if (u < nun && int(s_tab[u] & kStepMask) < t_end) flush(false);
  }
  stamp(6);  // warp 0 finished its run
#ifdef VPTQ_B200_PROF_WARPS  // developer build: when did every warp of the first CTA finish its run?
  if (mp.prof && lane == 0 && blockIdx.x == 0) {
    unsigned long long tw;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(tw));
    mp.prof[16 + warp] = tw;
  }
#endif
  __syncthreads();
  stamp(7);

  // -------- merge the pieces of units shared between warps (in warp order) ---------------------------------
  if (tid < kLW * 2 * 8) {
    const int i = tid >> 3, e = tid & 7;
    const int un = s_pu[i];
    if (un >= 0) {
      bool leader = true;
      for (int j = i - 1; j >= 0; --j) {
        const int pj = s_pu[j];
        if (pj < 0) continue;
        leader = pj != un;
        break;
      }
      if (leader) {
        float v = s_piece[i * 8 + e];
        for (int j = i + 1; j < kLW * 2; ++j) {
          const int pj = s_pu[j];
          if (pj < 0) continue;
          if (pj != un) break;
          v += s_piece[j * 8 + e];
        }
        red_add_fixed(L.yacc + size_t(un < nA ? rA0 + un : un - nA) * 8 + e, v + (un >= nA ? cbiasB : cbiasA));
      }
    }
  }
  __threadfence();
  __syncthreads();

  // -------- arrival: every row block this CTA's units belong to learns how many of them are done -----------
  {
    const int rA1 = rA0 + nA, nB = nun - nA;
    const int nbA = (rA1 - 1) / kRB - rA0 / kRB + 1;
    const int nbB = two ? (nB - 1) / kRB + 1 : 0;
    if (tid < nbA + nbB) {
      int b, lo, hi;
      if (tid < nbA) b = rA0 / kRB + tid, lo = max(rA0, b * kRB), hi = min(rA1, (b + 1) * kRB);
      else b = tid - nbA, lo = b * kRB, hi = min(nB, (b + 1) * kRB);
      const uint32_t cnt = uint32_t(hi - lo), rows_b = uint32_t(min(kRB, Ro - b * kRB));
      const uint32_t prev = atomicAdd(&L.counters[b], cnt);
      if (prev + cnt == uint32_t(L.Q) * rows_b) s_done[atomicAdd(s_ndone, 1)] = b;
    }
  }
  __syncthreads();
  stamp(8);
  const int nd = *s_ndone;
  bool stored_to_peers = false;
  if (nd > 0) {
    // this CTA's arrival completed nd row blocks: every unit of their rows has added its sums
    __threadfence();
    const T* bias = reinterpret_cast<const T*>(L.bias);
    T* y = reinterpret_cast<T*>(L.y);
    // one thread per index row: 8 accumulators (64 bytes) in, one 16-byte vector of outputs out -- to this
    // rank's y and, tensor-parallel, to the same place in every peer's buffer over NVLink
    for (int i = tid; i < nd * kRB; i += kLT) {
      const int r = s_done[i / kRB] * kRB + i % kRB;
      if (r < Ro) {
        unsigned long long* p = L.yacc + size_t(r) * 8;
        long long q[8];
#pragma unroll
        for (int k = 0; k < 4; ++k)
          asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(q[2 * k]), "=l"(q[2 * k + 1]) : "l"(p + 2 * k) : "memory");
#pragma unroll
        for (int k = 0; k < 4; ++k) *reinterpret_cast<ulonglong2*>(p + 2 * k) = make_ulonglong2(0ull, 0ull);  // zero at rest
        const int o = r * 8;
        float v[8];
#pragma unroll
        for (int e = 0; e < 8; ++e)
          v[e] = float(q[e]) * kFixInv + ((bias && o + e < L.O) ? DT<T>::to_float(bias[o + e]) : 0.f);
        if (o + 8 <= L.O && (reinterpret_cast<uintptr_t>(y) & 15u) == 0) {
          const uint4 pk = make_uint4(DT<T>::pack2(v[0], v[1]), DT<T>::pack2(v[2], v[3]), DT<T>::pack2(v[4], v[5]),
                                      DT<T>::pack2(v[6], v[7]));
          *reinterpret_cast<uint4*>(y + o) = pk;
          if (tagged) {
            // two 16-byte stores of {pair, tag, pair, tag} into every rank's tagged buffer (the local one too)
            for (int rk = 0; rk < mp.tp_world; ++rk) {
              uint8_t* dst = reinterpret_cast<uint8_t*>(mp.tp_peer_y[l][rk]) + size_t(o) * 4;
              asm volatile("st.volatile.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(dst), "r"(pk.x), "r"(tag_out), "r"(pk.y),
                           "r"(tag_out)
                           : "memory");
              asm volatile("st.volatile.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(dst + 16), "r"(pk.z), "r"(tag_out),
                           "r"(pk.w), "r"(tag_out)
                           : "memory");
            }
          } else if (mp.tp_world > 1) {
            for (int rk = 0; rk < mp.tp_world; ++rk)
              if (rk != mp.tp_rank) *reinterpret_cast<uint4*>(reinterpret_cast<T*>(mp.tp_peer_y[l][rk]) + o) = pk;
            stored_to_peers = true;
          }
        } else {
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            if (o + e < L.O) {
              const T hv = DT<T>::from_float(v[e]);
              y[o + e] = hv;
              if (mp.tp_world > 1 && !tagged) {
                for (int rk = 0; rk < mp.tp_world; ++rk)
                  if (rk != mp.tp_rank) reinterpret_cast<T*>(mp.tp_peer_y[l][rk])[o + e] = hv;
                stored_to_peers = true;
              }
            }
          }
        }
      }
    }
    if (tid < nd) L.counters[s_done[tid]] = 0u;  // leave the counters zeroed for the next launch
  }
  // -------- tensor-parallel hand-off: the last CTA of the launch publishes its epoch on every peer ----------
  if (mp.tp_world > 1) {
    if (stored_to_peers) __threadfence_system();  // this thread's peer stores are visible system-wide
    __syncthreads();
    if (tid == 0) {
      const uint32_t prev = atomicAdd(mp.tp_done + mp.tp_slot, 1u);
      if (prev == gridDim.x - 1u) {  // the whole launch (all fused layers) has stored its outputs
        mp.tp_done[mp.tp_slot] = 0u;
        mp.tp_epoch[mp.tp_slot] = run + 1u;  // (every CTA read `run` at its start)
        if (!tagged) {
          __threadfence_system();
          for (int r = 0; r < mp.tp_world; ++r)
            if (r != mp.tp_rank) st_release_sys_u32(mp.tp_peer_flags[r] + mp.tp_slot * mp.tp_world + mp.tp_rank, run + 1u);
        }
      }
    }
  }
  stamp(9);
}

// Tagged-word buffer -> plain 16-bit values, waiting for every word of the producing launch's LAST run (its
// epoch counter has already been advanced locally when this kernel runs behind it on the same stream).
__global__ void tp_untag_kernel(const void* tagged, uint4* y, int n8, const uint32_t* epoch, int slot, int nslots,
                                uint32_t* error) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  const uint32_t tag = (ld_volatile_u32(epoch + slot) - 1u) * uint32_t(nslots) + uint32_t(slot) + 1u;
  y[i] = load8_tagged(tagged, i * 8, tag, error);
}

using ListsKernelFn = void (*)(const ListsParams);

template <typename T>
ListsKernelFn pick_lists_t(bool res) {
  return res ? gemv_lists_kernel<T, true> : gemv_lists_kernel<T, false>;
}
ListsKernelFn pick_lists(int dtype, bool res) {
  if (dtype == VPTQ_FP16) return pick_lists_t<__half>(res);
  if (dtype == VPTQ_BF16) return pick_lists_t<__nv_bfloat16>(res);
  return nullptr;
}

int lists_tcw(int I) {
  const int nt = (I + kTileMax - 1) / kTileMax;
  return ((I + nt - 1) / nt + 7) / 8 * 8;
}

}  // namespace

int tp_untag_launch(const void* tagged, void* y, int n, const vptq_tp_exchange& tp, cudaStream_t stream) {
  const int n8 = n / 8;
  tp_untag_kernel<<<(n8 + 255) / 256, 256, 0, stream>>>(tagged, reinterpret_cast<uint4*>(y), n8, tp.epoch, tp.slot,
                                                         tp.num_slots, tp.error);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("tp_untag launch: %s", cudaGetErrorString(e));
    return VPTQ_ERR_CUDA;
  }
  return 0;
}

bool gemv_lists_eligible(const vptq_linear_desc& d) {
  if (!d.lists_stream || !d.lists_tab) return false;
  const bool outl = d.outlier_size > 0 && d.outlier_indices != nullptr;
  if (d.vector_len != 8 || d.num_codebooks != 1 || outl) return false;
  if (d.num_centroids < 2 * kSliceEntries || d.num_centroids % kSliceEntries) return false;
  if (d.num_centroids / kSliceEntries > 16) return false;
  if (d.num_res_centroids > 256) return false;
  if (d.in_features < 8 || d.lists_tile_cols != lists_tcw(d.in_features)) return false;
  if ((reinterpret_cast<uintptr_t>(d.lists_stream) & 15u) || (reinterpret_cast<uintptr_t>(d.lists_tab) & 3u)) return false;
  if ((reinterpret_cast<uintptr_t>(d.weight_scale) & 15u) || (reinterpret_cast<uintptr_t>(d.weight_bias) & 15u)) return false;
  return true;
}

size_t gemv_lists_workspace_bytes(const vptq_linear_desc& d) {
  // counters and accumulators both live in the fixed zero-at-rest head of the workspace
  return gemv_lists_eligible(d) ? kZeroRegionBytes : 0;
}

int gemv_lists_launch(int n, const vptq_linear_desc* const* descs, const void* x, void* const* ys, uint32_t flags,
                      cudaStream_t stream, void* workspace, size_t workspace_bytes, const vptq_tp_exchange* tp) {
  const DeviceInfo* dev = device_info();
  if (!dev) return VPTQ_ERR_CUDA;
  if (n < 1 || n > kMaxFusedLayers) {
    set_error("gemv_lists: 1..%d layers", kMaxFusedLayers);
    return VPTQ_ERR_UNSUPPORTED;
  }
  const vptq_linear_desc& d0 = *descs[0];
  const bool res = d0.num_res_centroids > 0;
  for (int l = 0; l < n; ++l) {
    const vptq_linear_desc& d = *descs[l];
    if (!gemv_lists_eligible(d) || d.dtype != d0.dtype || d.in_features != d0.in_features ||
        d.num_centroids != d0.num_centroids || (d.num_res_centroids > 0) != res) {
      set_error("gemv_lists: layer %d is not eligible / does not match layer 0", l);
      return VPTQ_ERR_UNSUPPORTED;
    }
  }
  if (reinterpret_cast<uintptr_t>(x) & 15u) {
    set_error("gemv_lists: x must be 16-byte aligned");
    return VPTQ_ERR_UNSUPPORTED;
  }
  ListsKernelFn fn = pick_lists(d0.dtype, res);
  if (!fn) return VPTQ_ERR_UNSUPPORTED;
  if (int rc = ensure_smem_attr(reinterpret_cast<const void*>(fn), dev->smem_optin)) return rc;

  const int I = d0.in_features, TCW = d0.lists_tile_cols;
  const int NS = d0.num_centroids / kSliceEntries, NT = (I + TCW - 1) / TCW, Q = NS * NT;
  // ---- CTAs (one per SM) shared out to the layers in proportion to their rows; every layer needs at
  // least Q of them (a CTA's range must not exceed one combo's worth of units) -----------------------------
  int Ro[kMaxFusedLayers], share[kMaxFusedLayers];
  int64_t rows = 0;
  for (int l = 0; l < n; ++l) Ro[l] = (descs[l]->out_features + 7) / 8, rows += Ro[l];
  const int P = dev->sm_count;
  if (int64_t(n) * Q > P) {
    set_error("gemv_lists: %d layers x %d combos exceed %d SMs", n, Q, P);
    return VPTQ_ERR_UNSUPPORTED;
  }
  {
    int used = 0, big = 0;
    for (int l = 0; l < n; ++l) {
      share[l] = std::max(Q, int(int64_t(P) * Ro[l] / rows));
      share[l] = int(std::min<int64_t>(share[l], int64_t(Q) * Ro[l]));  // never more CTAs than units
      used += share[l];
      if (Ro[l] > Ro[big]) big = l;
    }
    // take the excess from / hand the remainder to whichever layer has the most / fewest CTAs per row
    while (used > P) {
      int v = -1;
      double best = 0;
      for (int l = 0; l < n; ++l) {
        const double per_row = double(share[l]) / Ro[l];
        if (share[l] > Q && per_row > best) v = l, best = per_row;
      }
      if (v < 0) {
        set_error("gemv_lists: the layers do not fit %d CTAs", P);
        return VPTQ_ERR_UNSUPPORTED;
      }
      --share[v], --used;
    }
    while (used < P) {
      int v = -1;
      double worst = 0;
      for (int l = 0; l < n; ++l) {
        const double rows_per = double(Ro[l]) / share[l];
        if (int64_t(share[l]) < int64_t(Q) * Ro[l] && rows_per > worst) v = l, worst = rows_per;
      }
      if (v < 0) break;
      ++share[v], ++used;
    }
  }
  int max_nun = 0, max_kr = 0;
  size_t ws_need = kZeroRegionBytes;
  size_t rows_total = 0;
  size_t nblk = 0;
  for (int l = 0; l < n; ++l) {
    const int64_t U = int64_t(Q) * Ro[l];
    max_nun = std::max<int>(max_nun, int((U + share[l] - 1) / share[l]));
    max_kr = std::max(max_kr, descs[l]->num_res_centroids > 0 ? descs[l]->num_res_centroids : 0);
    rows_total += size_t(Ro[l]);
    nblk += size_t((Ro[l] + kRB - 1) / kRB);
  }
  if (max_nun > kMaxWindow) {
    set_error("gemv_lists: %d units per CTA exceed %d", max_nun, kMaxWindow);
    return VPTQ_ERR_UNSUPPORTED;
  }
  if (rows_total > size_t(kMaxIndexRows)) {
    set_error("gemv_lists: %zu index rows exceed %d", rows_total, kMaxIndexRows);
    return VPTQ_ERR_UNSUPPORTED;
  }
  if (!workspace || workspace_bytes < ws_need || nblk * 4 > kCounterRegionBytes) {
    set_error("gemv_lists: workspace %zu bytes < required %zu", workspace_bytes, ws_need);
    return VPTQ_ERR_WORKSPACE;
  }

  // ---- shared-memory carve-up --------------------------------------------------------------------
  ListsParams mp{};
  const size_t limit = size_t(dev->smem_optin);
  auto carve = [&](int stages) -> size_t {
    size_t off = 0;
    mp.off_bars = uint32_t(off), off += align_up(size_t(2 + kLW * stages) * 8, 128);
    mp.off_tab = uint32_t(off), off += align_up(size_t(max_nun + 1) * 4, 128);
    mp.off_red = uint32_t(off), off += 256;
    mp.off_piece = uint32_t(off), off += size_t(kLW) * 2 * 32 + 128;
    mp.off_done = uint32_t(off), off += align_up(size_t(kMaxWindow / kRB + 8) * 4, 128);
    mp.off_slice = uint32_t(off), off += 2 * size_t(kSliceBytes);
    mp.off_res = uint32_t(off), off += align_up(size_t(max_kr) * 16 * kResRep, 128);
    mp.off_x = uint32_t(off), off += 3 * 8192;  // two tiles + slack for the 8 KiB alignment
    mp.off_ring = uint32_t(off), off += size_t(kLW) * stages * kStageBytes;
    mp.stages = stages;
    return off;
  };
  size_t need = 0;
  bool placed = false;
  for (int stages = 3; stages >= 2; --stages) {
    need = carve(stages);
    if (need <= limit) {
      placed = true;
      break;
    }
  }
  if (!placed) {
    set_error("gemv_lists: no shared-memory layout fits (%zu bytes needed)", need);
    return VPTQ_ERR_UNSUPPORTED;
  }

  mp.n = n, mp.x = x, mp.prof = gemv_profile_buffer();
  if (mp.prof) {
    // developer aid: VPTQ_B200_PROF_SLOTS=N gives every launch its own 32-stamp record (round robin over N)
    static const int slots = [] {
      const char* e = std::getenv("VPTQ_B200_PROF_SLOTS");
      return e ? std::max(1, std::atoi(e)) : 1;
    }();
    static std::atomic<unsigned> counter{0};
    if (slots > 1) mp.prof += 32u * (counter.fetch_add(1) % unsigned(slots));
  }
  uint32_t begin = 0;
  uint8_t* wsb = reinterpret_cast<uint8_t*>(workspace);
  size_t part_off = kCounterRegionBytes, ctr_off = 0;
  for (int l = 0; l < n; ++l) {
    const vptq_linear_desc& d = *descs[l];
    ListsLayer& L = mp.layer[l];
    L.stream = reinterpret_cast<const uint32_t*>(d.lists_stream), L.tab = d.lists_tab;
    L.centroids = d.centroids, L.res_centroids = d.res_centroids;
    L.scale = d.weight_scale, L.wbias = d.weight_scale ? d.weight_bias : nullptr;
    L.bias = d.bias, L.y = ys[l];
    L.I = I, L.O = d.out_features, L.Ro = Ro[l], L.Kr = d.num_res_centroids > 0 ? d.num_res_centroids : 0;
    L.NS = NS, L.Q = Q, L.TCW = TCW, L.U = Q * Ro[l];
    L.ncta = share[l];
    L.yacc = reinterpret_cast<unsigned long long*>(wsb + part_off);
    L.counters = reinterpret_cast<uint32_t*>(wsb + ctr_off);
    part_off += size_t(Ro[l]) * 64;
    ctr_off += size_t((Ro[l] + kRB - 1) / kRB) * 4;
    mp.grid_begin[l] = begin;
    begin += uint32_t(share[l]);
  }
  for (int l = n; l <= kMaxFusedLayers; ++l) mp.grid_begin[l] = begin;
  if (tp && tp->world > 1) {
    mp.tp_world = tp->world, mp.tp_rank = tp->rank, mp.tp_slot = tp->slot, mp.tp_wait_slot = tp->wait_slot;
    for (int l = 0; l < n; ++l)
      for (int r = 0; r < tp->world; ++r) mp.tp_peer_y[l][r] = tp->peer_y[l][r];
    for (int r = 0; r < tp->world; ++r) mp.tp_peer_flags[r] = tp->peer_flags[r];
    mp.tp_epoch = tp->epoch, mp.tp_done = tp->done, mp.tp_error = tp->error;
    mp.tp_format = tp->format, mp.tp_nslots = tp->num_slots;
    if (tp->format == VPTQ_TP_TAGGED) {
      bool ok = tp->num_slots > tp->slot && (I % 8) == 0;
      for (int l = 0; l < n; ++l) ok = ok && (descs[l]->out_features % 8) == 0 && tp->peer_y[l][tp->rank] != nullptr;
      if (!ok) {
        set_error("gemv_lists: VPTQ_TP_TAGGED needs in/out_features %% 8 == 0, num_slots > slot and a local tagged buffer");
        return VPTQ_ERR_INVALID;
      }
    }
  }

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
    set_error("gemv_lists launch (grid=%u smem=%zu): %s", begin, need, cudaGetErrorString(e));
    return VPTQ_ERR_CUDA;
  }
  return 0;
}

}  // namespace vptq_b200
