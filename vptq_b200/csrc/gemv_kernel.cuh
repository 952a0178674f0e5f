// Fused decode GEMV for VPTQ-quantized linear layers on sm_100a.
//
//   y[t][o] = sum_c x'[t][c] * Wq[o][c]  +  sum_f x[t][f] * wbias[f]  +  bias[o]
//   x'[t][c] = x[t][perm[c]] * scale[perm[c]],   Wq[r*v+e][c] = C[idx[r][c]][e] + R[ridx[r][c]][e]
//
// (same mathematics as the reference's WqA16WithOutliers_PackIndice,
// csrc/kernels/quant_gemv.cuh:11-186, with the three hoists it does not make: x' is formed once
// per CTA instead of per (row, column); the weight_bias term is a per-token scalar added in the
// epilogue; accumulation is fp32.)  Nothing here is derived from the reference's kernel
// structure:
//   * a CTA owns one column chunk (its x' slice and codebooks are staged once) and a strided set
//     of index rows; every warp owns whole rows and keeps the v partial sums in registers;
//   * the packed index words of a row arrive through a per-warp ring of 1-D TMA bulk copies
//     (cp.async.bulk + mbarrier, L2 evict_first);
//   * codebooks that fit are staged in shared memory by TMA (small ones bank-group replicated so
//     that 128-bit gathers are conflict-free).  A 65536-entry codebook (1 MiB) cannot be: its
//     16-byte entries are gathered through L1/L2 (evict_last), 8 independent gathers in flight
//     per lane.  The measured bound of that tier is ~1.1 gathers per clock per SM (L1TEX tag
//     stage, tools/gather_microbench.cu); a cp.async/LDGSTS gather ring was tried and measured
//     slower (double index decode + shared-memory round trip), see DESIGN.md;
//   * the split-K reduction over column chunks runs inside a thread-block cluster: every CTA
//     pushes its per-row partial sums into the leader's shared memory with st.async, completion
//     counted on an mbarrier there; the leader sums the chunks in order and writes y.  No second
//     kernel (the reference launches `sum(-1)`, csrc/quant_gemv.cu:235), no global atomics or
//     fences.  Layers cut into more than 8 chunks use a global-memory variant of the same scheme.
#pragma once

#include "common.cuh"
#include "kernels.h"

namespace vptq_b200 {

struct GemvParams {
  // layer
  const uint32_t* indices;
  int64_t idx_stride_g, idx_stride_r;  // 32-bit words
  const void* centroids;
  int64_t cb_stride;  // elements
  const void* res_centroids;
  int64_t rcb_stride;
  const uint16_t* outlier_idx;
  const void* outlier_cb;
  const uint16_t* perm;
  const void* scale;
  const void* wbias;
  const void* scale_q;  // optional load-time copies in quantised column order: scale[perm[c]], wbias[perm[c]]
  const void* wbias_q;
  const void* bias;
  // activations
  const void* x;
  void* y;
  int64_t x_stride, y_stride;  // elements per token
  // global split-K workspace (only when the plan does not use a cluster)
  float* partials;
  uint32_t* counters;
  // shapes
  int I, O, Ro, G, gs, S, vol, Kol, Rol;
  int K, Kr, ib, rb;
  int idx_tma_ok;  // rows are 16-byte aligned -> bulk copies legal
  // tensor-parallel exchange over peer memory (tp_world == 0: off; world 1 still publishes epochs).  The kernel stores
  // every output value into the same slot of every rank's full-width y (NVLink stores), the last CTA to finish
  // publishes a per-launch epoch flag on every peer, and the consumer launch polls those flags
  // before it reads x: no memset, no NCCL call, no extra kernel between two layers.
  int tp_world, tp_rank, tp_slot, tp_wait_slot;
  void* tp_peer_y[8];             // y slice start in rank r's buffer (entry [tp_rank] unused)
  uint32_t* tp_peer_flags[8];     // rank r's flag array [slots][world]; [tp_rank] = the local one
  uint32_t* tp_epoch;             // local: completed runs per launch slot
  uint32_t* tp_done;              // local: CTA arrival counters per launch slot (zero at rest)
  uint32_t* tp_error;             // local: set when a flag wait timed out
  unsigned long long* prof;  // developer aid: per-phase %globaltimer stamps of CTA 0 / last CTA (or nullptr)
  GemvPlan plan;
};

// acc[e] += xv * (c[e] + r[e]) for one gathered (main, residual) entry pair, fp32 arithmetic
template <typename T, int V, bool RES>
__device__ __forceinline__ void fma_entry(float (&acc)[V], float xv, const uint32_t (&cw)[V / 2],
                                          const uint32_t (&rw)[V / 2]) {
#pragma unroll
  for (int i = 0; i < V / 2; ++i) {
    float2 c = DT<T>::unpack2(cw[i]);
    if constexpr (RES) {
      const float2 r = DT<T>::unpack2(rw[i]);
      c.x += r.x;
      c.y += r.y;
    }
    acc[2 * i] = fmaf(xv, c.x, acc[2 * i]);
    acc[2 * i + 1] = fmaf(xv, c.y, acc[2 * i + 1]);
  }
}

// Sum acc[0..V) over the 32 lanes.  Returns, in lane e (e < V), the total of acc[e].
// V == 8: recursive halving -- 4+2+1 exchanges that each halve the live values, then two plain
// butterfly steps: 9 shuffles instead of 40.
template <int V>
__device__ __forceinline__ float warp_reduce_to_lane(float (&acc)[V], int lane) {
  if constexpr (V == 8) {
    float a4[4], a2[2];
    const bool h16 = lane & 16, h8 = lane & 8, h4 = lane & 4;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float keep = h16 ? acc[i + 4] : acc[i], send = h16 ? acc[i] : acc[i + 4];
      a4[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const float keep = h8 ? a4[i + 2] : a4[i], send = h8 ? a4[i] : a4[i + 2];
      a2[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
    }
    const float keep = h4 ? a2[1] : a2[0], send = h4 ? a2[0] : a2[1];
    float v = keep + __shfl_xor_sync(0xffffffffu, send, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    // lanes with bits (16,8,4) = (b2,b1,b0) now hold output e = 4*b2 + 2*b1 + b0; move it to lane e
    return __shfl_sync(0xffffffffu, v, ((lane & 4) << 2) | ((lane & 2) << 2) | ((lane & 1) << 2));
  } else {
    float mine = 0.f;
#pragma unroll
    for (int e = 0; e < V; ++e) {
      const float v = warp_sum(acc[e]);
      if (lane == e) mine = v;
    }
    return mine;
  }
}

// One CTA's share of one layer.  `bidx` / `gdim`: this CTA's index within, and the size of, the
// layer's own grid (a fused launch concatenates the grids of several layers, see gemv_multi_kernel).
// RES_L2: the residual codebook does not fit in shared memory (256 KiB and up): its entries are gathered
// through L1/L2 next to the main entry of the same field, like an L2-gather main codebook.
template <typename T, int V, int NT, bool MAIN_SMEM, bool RES, bool RES_L2 = false>
__device__ __forceinline__ void gemv_body(const GemvParams& p, uint8_t* smem, const uint32_t bidx, const uint32_t gdim,
                                          const uint32_t gdim_total) {
  static_assert(RES || !RES_L2, "RES_L2 needs a residual codebook");
  constexpr bool RES_SMEM = RES && !RES_L2;
  constexpr int U = (NT == 1 && V <= 8) ? 8 : 4;  // independent codebook gathers in flight per lane
  constexpr int EB = 2 * V;                       // bytes per codebook entry
  const GemvPlan& pl = p.plan;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  // phase stamps (ns) of thread 0 of the first and of the last CTA: tools/profile_gemv.py --phases
  auto stamp = [&](int slot) {
    if (p.prof && tid == 0 && (bidx == 0 || bidx == gdim - 1)) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      p.prof[(bidx == 0 ? 0 : 16) + slot] = t;
    }
  };
  stamp(0);
  const int chunk = bidx % pl.nch;  // == %cluster_ctarank when launched as a cluster
  const int cta_in_chunk = bidx / pl.nch;
  const int g = chunk / pl.cpg, cig = chunk % pl.cpg;
  const int f0 = cig * pl.chunk_cols;
  const int f1 = min(p.gs, f0 + pl.chunk_cols);
  const int ncols = f1 - f0;
  const bool owns_outliers = (chunk == 0) && (p.S > 0);
  const int n_all = ncols + (owns_outliers ? p.S : 0);
  const int b = p.ib + p.rb;

  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + pl.off_bars);
  float* s_cbias = reinterpret_cast<float*>(smem + pl.off_cbias);
  uint16_t* s_pcol = reinterpret_cast<uint16_t*>(smem + pl.off_pcol);
  float* s_wb = reinterpret_cast<float*>(smem + pl.off_wb);
  float* sx = reinterpret_cast<float*>(smem + pl.off_sx);
  float* s_part = reinterpret_cast<float*>(smem + pl.off_part);
  float* s_wsum = reinterpret_cast<float*>(smem + pl.off_wsum);       // [rows][wsplit][NT][V] (wsplit > 1)
  uint32_t* s_wcnt = reinterpret_cast<uint32_t*>(smem + pl.off_wcnt);  // [rows] arrival counters
  uint8_t* s_res = smem + pl.off_res;
  uint8_t* s_main = smem + pl.off_main;
  uint8_t* s_raw = smem + pl.off_raw;  // TMA landing zone of tables that are then replicated
  uint8_t* ring = smem + pl.off_ring + warp * pl.stages * pl.stage_bytes;
  uint64_t* cb_bar = &bars[0];
  uint64_t* part_bar = &bars[1];
  uint64_t* full = &bars[2 + warp * pl.stages];

  const T* cent_g = reinterpret_cast<const T*>(p.centroids) + int64_t(g) * p.cb_stride;
  const T* res_g = RES ? reinterpret_cast<const T*>(p.res_centroids) + int64_t(g) * p.rcb_stride : nullptr;

  const int nrows_cta = cta_in_chunk < p.Ro ? (p.Ro - cta_in_chunk + pl.cpc - 1) / pl.cpc : 0;

  // -------- first thing: get the x-independent column metadata of this thread's first 4 columns on
  // their way (perm, scale, wbias come from DRAM once per token: ~1 us that overlaps the setup below)
  const T* scale = reinterpret_cast<const T*>(p.scale);
  const T* wbias = reinterpret_cast<const T*>(p.wbias);
  const T* scale_q = reinterpret_cast<const T*>(p.scale_q);
  const T* wbias_q = reinterpret_cast<const T*>(p.wbias_q);
  // loads only (raw 16-bit values, no conversions: nothing here waits for the data)
  auto load_cols = [&](int i0, int (&pc)[4], T (&sc)[4], T (&wb)[4], bool early) {
    int cc[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int i = i0 + k * int(blockDim.x);
      const int c = i < ncols ? p.S + g * p.gs + f0 + i : i - ncols;
      cc[k] = i < n_all ? c : 0;
      pc[k] = i < n_all ? (p.perm ? int(p.perm[c]) : c) : 0;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      // quantised-order copies (built once at load time) cut the perm -> scale dependent-load chain;
      // without them the dependent gathers are left for phase A (`early` must not wait for perm)
      if (scale_q) sc[k] = scale_q[cc[k]], wb[k] = wbias_q[cc[k]];
      else if (!early) sc[k] = scale ? scale[pc[k]] : DT<T>::from_float(1.f), wb[k] = wbias ? wbias[pc[k]] : DT<T>::from_float(0.f);
    }
  };
  int pc0[4];
  T sc0[4], wb0[4];
  load_cols(tid, pc0, sc0, wb0, true);

  // -------- barrier init -----------------------------------------------------------------
  {
    const int nbar = 2 + nwarps * pl.stages;  // one thread per barrier: a serial loop costs ~0.5 us
    if (tid < nbar) {
      mbar_init(&bars[tid], 1);
      fence_mbar_init();
      // leader: every chunk (this one included) delivers NT*V floats per row with st.async
      if (tid == 1 && pl.cluster && chunk == 0)
        mbar_arrive_expect_tx(part_bar, uint32_t(pl.nch * nrows_cta * NT * V) * 4u);
    }
  }
  if (pl.wsplit > 1)
    for (int i = tid; i < nrows_cta; i += blockDim.x) s_wcnt[i] = 0u;
  __syncthreads();
  stamp(1);
  // "this CTA runs and its barriers exist" (made cluster-visible by fence.mbarrier_init); relaxed: a
  // releasing arrive costs a GPU-scope MEMBAR (~1 us).  Waited before the first st.async.
  if (pl.cluster) cluster_arrive_relaxed();
  pdl_launch_dependents();           // the next kernel may start its own weight-only prologue now

  const uint64_t pol_stream = policy_evict_first();
  const uint64_t pol_keep = policy_evict_last();

  // -------- work list of this warp -------------------------------------------------------
  // `wsplit` warps share one row of the chunk: warp w works on column sub-range `wsub` of the rows
  // of row slot `wslot`; their partial sums meet in shared memory (finish_row).
  const int wsplit = pl.wsplit, wsub = warp % wsplit, wslot = warp / wsplit, nslots = nwarps / wsplit;
  const int sf0 = min(ncols, wsub * pl.sub_cols), sf1 = min(ncols, sf0 + pl.sub_cols);  // relative to the chunk
  const int wcols = sf1 - sf0;
  const int nunits = wslot < nrows_cta ? (nrows_cta - wslot + nslots - 1) / nslots : 0;
  const int nseg = (wcols + pl.seg_fields - 1) / pl.seg_fields;
  const int total = nunits * nseg;
  const uint32_t* idx_g = p.indices + int64_t(g) * p.idx_stride_g;

  // warp-collective: start the copy of segment q of this warp's work list into its ring stage
  auto issue = [&](int q) {
    const int u = q / nseg, s = q - u * nseg;
    const int r = cta_in_chunk + pl.cpc * (wslot + nslots * u);
    const int fs = f0 + sf0 + s * pl.seg_fields;
    const int nf = min(pl.seg_fields, f0 + sf1 - fs);
    const uint32_t* src = idx_g + int64_t(r) * p.idx_stride_r + ((int64_t(fs) * b) >> 5);
    const int nw = (nf * b + 31) >> 5;
    const int st = q % pl.stages;
    uint8_t* dst = ring + st * pl.stage_bytes;
    if (p.idx_tma_ok && (nw & 3) == 0) {
      if (lane == 0) {  // (the stage was only READ through the generic proxy before: no proxy fence needed)
        mbar_arrive_expect_tx(&full[st], uint32_t(nw) * 4u);
        tma_bulk_g2s(dst, src, uint32_t(nw) * 4u, &full[st], pol_stream);
      }
    } else {  // ragged / unaligned rows: plain word copy by the whole warp
      uint32_t* d32 = reinterpret_cast<uint32_t*>(dst);
      for (int i = lane; i < nw; i += 32) d32[i] = ldg_nc_u32(src + i);
      fence_proxy_async_smem();  // a later TMA refill of this stage must be ordered after these generic writes
      __syncwarp();
      if (lane == 0) mbar_arrive(&full[st]);
    }
  };

  // index stream: fill the ring before anything else so HBM latency overlaps the prologue
  const int npre = min(total, pl.stages);
  for (int q = 0; q < npre; ++q) issue(q);

  // -------- codebooks -> shared memory (weights only: legal before the PDL wait) -----------
  // rep == 1: TMA bulk copy straight to its place.  rep == 8 (16-byte entries only): TMA into a
  // landing zone, then entry i is stored 8 times, copy k at 16-byte slot i*8+k; lane L reads slot
  // i*8 + (L & 7), so the 8 lanes of a quarter-warp always hit 8 different 16-byte bank groups
  // and 128-bit gathers are conflict-free.
  uint32_t cb_tx = 0, raw_off = 0;
  uint32_t raw_res = 0, raw_main = 0;  // landing-zone offsets (valid when the table is replicated)
  bool tma_res = false, tma_main = false;
  auto stage_table = [&](uint8_t* dst, const T* src, int entries, int rep, uint32_t& raw_at, bool& by_tma) {
    const uint32_t bytes = uint32_t(entries) * EB;
    by_tma = (bytes & 15u) == 0 && (reinterpret_cast<uintptr_t>(src) & 15u) == 0 && (rep == 1 || V == 8);
    if (by_tma) {
      uint8_t* land = rep == 1 ? dst : s_raw + raw_off;
      raw_at = raw_off;
      if (rep > 1) raw_off += bytes;
      if (tid == 0) {
        for (uint32_t off = 0; off < bytes; off += 32768u) {
          const uint32_t n = min(32768u, bytes - off);
          tma_bulk_g2s(land + off, reinterpret_cast<const uint8_t*>(src) + off, n, cb_bar, pol_keep);
        }
      }
      cb_tx += bytes;
    } else {  // odd sizes / alignments: plain loads
      const uint32_t* s32 = reinterpret_cast<const uint32_t*>(src);
      uint32_t* d32 = reinterpret_cast<uint32_t*>(dst);
      constexpr int WPE = V / 2;  // words per entry
      for (int i = tid; i < entries * WPE; i += blockDim.x) {
        const uint32_t w = ldg_nc_u32(s32 + i);
        const int e = i / WPE, k = i - e * WPE;
        for (int c = 0; c < rep; ++c) d32[(e * rep + c) * WPE + k] = w;
      }
    }
  };
  if constexpr (RES_SMEM) stage_table(s_res, res_g, p.Kr, pl.res_rep, raw_res, tma_res);
  if constexpr (MAIN_SMEM) stage_table(s_main, cent_g, p.K, pl.main_rep, raw_main, tma_main);
  if (tid == 0) {
    if (cb_tx) mbar_arrive_expect_tx(cb_bar, cb_tx);
    else mbar_arrive(cb_bar);
  }

  stamp(2);
  // -------- x' prologue, phase A: everything that does not depend on x --------------------
  // four columns per thread and step, loads grouped by dependence level (perm -> scale, wbias)
  // the 1 MiB codebook of an L2-gather layer is cold (2.6 GB of other layers went through the L2
  // since its last use): pull this CTA's slice of it towards L2 while the prologue runs
  if constexpr (!MAIN_SMEM) {
    if (tid == 32) {
      const uint32_t total_b = uint32_t(p.K) * EB;
      const uint32_t slice = ((total_b + gdim - 1) / gdim + 15u) & ~15u;
      const uint32_t off = bidx * slice;
      if (off < total_b) l2_prefetch_bulk(reinterpret_cast<const uint8_t*>(cent_g) + off, min(slice, total_b - off));
    }
  }
  if constexpr (RES_L2) {
    if (tid == 64) {
      const uint32_t total_b = uint32_t(p.Kr) * EB;
      const uint32_t slice = ((total_b + gdim - 1) / gdim + 15u) & ~15u;
      const uint32_t off = bidx * slice;
      if (off < total_b) l2_prefetch_bulk(reinterpret_cast<const uint8_t*>(res_g) + off, min(slice, total_b - off));
    }
  }
  for (int i0 = tid; i0 < n_all; i0 += 4 * blockDim.x) {
    int pc[4];
    T sc[4], wb[4];
    if (i0 == tid) {  // the batch whose loads were issued at kernel entry
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        pc[k] = pc0[k];
        if (scale_q) sc[k] = sc0[k], wb[k] = wb0[k];
        else sc[k] = scale ? scale[pc[k]] : DT<T>::from_float(1.f), wb[k] = wbias ? wbias[pc[k]] : DT<T>::from_float(0.f);
      }
    } else {
      load_cols(i0, pc, sc, wb, false);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int i = i0 + k * blockDim.x;
      if (i < n_all) s_pcol[i] = uint16_t(pc[k]), sx[i] = DT<T>::to_float(sc[k]), s_wb[i] = DT<T>::to_float(wb[k]);
    }
  }

  stamp(3);
  // replicate TMA-landed tables (smem -> smem) once they have arrived
  if constexpr (RES_SMEM || MAIN_SMEM) mbar_wait(cb_bar, 0);
  if constexpr (V == 8) {
    auto replicate = [&](uint8_t* dst, uint32_t raw_at, int entries) {
      const uint32_t src = smem_u32(s_raw + raw_at), d = smem_u32(dst);
      for (int e = tid; e < entries; e += blockDim.x) {
        const uint4 v = lds_v4(src + e * 16);
#pragma unroll
        for (int c = 0; c < 8; ++c) sts_v4(d + (e * 8 + c) * 16, v);
      }
    };
    if (RES_SMEM && tma_res && pl.res_rep > 1) replicate(s_res, raw_res, p.Kr);
    if (MAIN_SMEM && tma_main && pl.main_rep > 1) replicate(s_main, raw_main, p.K);
  }

  stamp(4);
  // -------- phase B: x arrives from the previous kernel ------------------------------------
  pdl_wait_prior_grid();
  if (p.tp_world > 0 && p.tp_wait_slot >= 0) {
    // x is assembled from every rank's slice: wait until all peers have published the epoch of the
    // launch that produces it (this launch's own run number: both run once per token)
    if (tid == 0) {
      const uint32_t want = ld_volatile_u32(p.tp_epoch + p.tp_slot) + 1u;
      const uint32_t* mine = p.tp_peer_flags[p.tp_rank] + p.tp_wait_slot * p.tp_world;
      const long long t0 = clock64();
      for (int r = 0; r < p.tp_world; ++r) {
        if (r == p.tp_rank) continue;
        // (serial-number compare: correct across the wrap of the 32-bit epoch)
        while (int32_t(ld_acquire_sys_u32(mine + r) - want) < 0) {
          if (ld_volatile_u32(p.tp_error) != 0u) break;  // an earlier wait timed out: the token is lost anyway
          if (clock64() - t0 > (1ll << 32)) {  // ~2 s: give up loudly instead of hanging the GPU
            *p.tp_error = 1u;
            break;
          }
        }
      }
      __threadfence_system();
    }
    __syncthreads();
  }
  stamp(5);
  {
    const T* x = reinterpret_cast<const T*>(p.x);
    float bs[NT];
#pragma unroll
    for (int t = 0; t < NT; ++t) bs[t] = 0.f;
    for (int i0 = tid; i0 < n_all; i0 += 4 * blockDim.x) {
      float xv[4][NT];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int i = i0 + k * int(blockDim.x);
        const int pc = i < n_all ? int(s_pcol[i]) : 0;  // own slots only: no barrier since phase A
#pragma unroll
        for (int t = 0; t < NT; ++t) xv[k][t] = DT<T>::to_float(x[int64_t(t) * p.x_stride + pc]);
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int i = i0 + k * blockDim.x;
        if (i < n_all) {
          const float sc = sx[i], wb = s_wb[i];
#pragma unroll
          for (int t = NT - 1; t >= 0; --t) {
            sx[t * pl.sx_stride + i] = xv[k][t] * sc;
            bs[t] = fmaf(xv[k][t], wb, bs[t]);
          }
        }
      }
    }
    // block-reduce the weight_bias term of this chunk: s_cbias[t] = sum_{c in chunk} x[perm c]*wbias[perm c]
    float* red = s_cbias + NT;  // [NT][nwarps] scratch
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      const float v = warp_sum(bs[t]);
      if (lane == 0) red[t * nwarps + warp] = v;
    }
    __syncthreads();
    if (tid < NT) {
      float v = 0.f;
      for (int w = 0; w < nwarps; ++w) v += red[tid * nwarps + w];
      s_cbias[tid] = v;
    }
  }
  __syncthreads();
  stamp(6);
  if (pl.cluster) cluster_wait();  // every CTA of the cluster runs: the leader's smem may be written
  stamp(7);

  // -------- main loop ------------------------------------------------------------------------
  const uint32_t fmask = b >= 32 ? 0xffffffffu : ((1u << b) - 1u);
  const uint32_t imask = (1u << p.ib) - 1u;
  const uint32_t main_stride = uint32_t(EB) * (MAIN_SMEM ? pl.main_rep : 1);
  const uint32_t res_stride = uint32_t(EB) * pl.res_rep;
  const uint32_t s_main_lane = smem_u32(s_main) + (pl.main_rep > 1 ? (lane & 7) * EB : 0);
  const uint32_t s_res_lane = smem_u32(s_res) + (pl.res_rep > 1 ? (lane & 7) * EB : 0);
  const uint8_t* cent_bytes = reinterpret_cast<const uint8_t*>(cent_g);
  const uint32_t part_leader = pl.cluster ? mapa_shared(smem_u32(s_part), 0) : 0u;
  const uint32_t bar_leader = pl.cluster ? mapa_shared(smem_u32(part_bar), 0) : 0u;
  const T* bias = reinterpret_cast<const T*>(p.bias);
  T* y = reinterpret_cast<T*>(p.y);

  // the one place y is written: locally and, under tensor parallelism, into every peer's buffer
  bool stored_to_peers = false;
  auto store_y = [&](int t, int o, float v) {
    const T hv = DT<T>::from_float(v);
    const int64_t off = int64_t(t) * p.y_stride + o;
    y[off] = hv;
    if (p.tp_world > 0) {
      stored_to_peers = true;
#pragma unroll 1
      for (int r = 0; r < p.tp_world; ++r)
        if (r != p.tp_rank) reinterpret_cast<T*>(p.tp_peer_y[r])[off] = hv;
    }
  };

  float acc[NT][V];
#pragma unroll
  for (int t = 0; t < NT; ++t)
#pragma unroll
    for (int e = 0; e < V; ++e) acc[t][e] = 0.f;

  // field j of ring stage `sw` (0 for lanes past the end: they gather entry 0 and skip the FMAs)
  auto field_at = [&](const uint32_t* sw, int j, int nf) -> uint32_t {
    const uint32_t bit = uint32_t(j) * uint32_t(b);
    const uint32_t w = bit >> 5;
    const uint32_t f = __funnelshift_r(sw[w], sw[w + 1], bit & 31u) & fmask;
    return j < nf ? f : 0u;
  };

  // one row of this warp is complete: outlier columns, warp reduction, hand-off
  auto finish_row = [&](int krow) {
    const int r = cta_in_chunk + pl.cpc * krow;
    if (owns_outliers && wsub == 0) {
      const T* ocb = reinterpret_cast<const T*>(p.outlier_cb);
      const float* sxo = sx + ncols;
      for (int c = lane; c < p.S; c += 32) {
        float xo[NT];
#pragma unroll
        for (int t = 0; t < NT; ++t) xo[t] = sxo[t * pl.sx_stride + c];
#pragma unroll
        for (int e = 0; e < V; ++e) {
          const int o = r * V + e;
          if (o < p.O) {
            const int rol = o / p.vol, eo = o - rol * p.vol;
            const int oi = p.outlier_idx[int64_t(rol) * p.S + c];
            const float w = DT<T>::to_float(ocb[int64_t(oi) * p.vol + eo]);
#pragma unroll
            for (int t = 0; t < NT; ++t) acc[t][e] = fmaf(xo[t], w, acc[t][e]);
          }
        }
      }
    }
    float mine[NT];  // lane e < V: sum of output e of this row over this warp's columns
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      mine[t] = warp_reduce_to_lane<V>(acc[t], lane);
#pragma unroll
      for (int e = 0; e < V; ++e) acc[t][e] = 0.f;
    }
    if (wsplit > 1) {
      // the warps sharing this row meet here: each parks its V*NT sums, the last one to arrive adds
      // them up in sub-range order (deterministic) and carries on alone
      float* slot = s_wsum + (krow * wsplit) * (NT * V);
      if (lane < V) {
#pragma unroll
        for (int t = 0; t < NT; ++t) slot[(wsub * NT + t) * V + lane] = mine[t];
      }
      __threadfence_block();
      __syncwarp();
      uint32_t prev = 0;
      if (lane == 0) prev = atomicAdd(&s_wcnt[krow], 1u);
      prev = __shfl_sync(0xffffffffu, prev, 0);
      if (prev != uint32_t(wsplit - 1)) return;
      __threadfence_block();
      if (lane < V) {
#pragma unroll
        for (int t = 0; t < NT; ++t) {
          float v = 0.f;
          for (int w = 0; w < wsplit; ++w) v += slot[(w * NT + t) * V + lane];
          mine[t] = v;
        }
      }
    }
#pragma unroll
    for (int t = 0; t < NT; ++t) mine[t] += s_cbias[t];
    const int o = r * V + lane;
    const bool writer = lane < V && o < p.O;
    if (pl.nch == 1) {
      if (writer) {
        const float bv = bias ? DT<T>::to_float(bias[o]) : 0.f;
#pragma unroll
        for (int t = 0; t < NT; ++t) store_y(t, o, mine[t] + bv);
      }
    } else if (pl.cluster) {
      // DSMEM hand-off: slot [krow][chunk][t][e] of the leader's (rank 0) partial-sum table
      if (lane < V) {
#pragma unroll
        for (int t = 0; t < NT; ++t)
          st_async_f32(part_leader + uint32_t(((krow * pl.nch + chunk) * NT + t) * V + lane) * 4u, mine[t], bar_leader);
      }
    } else {
      // global-memory variant: the last chunk of a row to arrive sums all chunks in order
      const int64_t opad = int64_t(p.Ro) * V;
      if (lane < V) {
#pragma unroll
        for (int t = 0; t < NT; ++t) p.partials[(int64_t(chunk) * NT + t) * opad + r * V + lane] = mine[t];
        __threadfence();
      }
      __syncwarp();
      uint32_t prev = 0;
      if (lane == 0) prev = atomicAdd(&p.counters[r], 1u);
      prev = __shfl_sync(0xffffffffu, prev, 0);
      if (prev == uint32_t(pl.nch - 1)) {
        __threadfence();
        if (writer) {
          const float bv = bias ? DT<T>::to_float(bias[o]) : 0.f;
#pragma unroll
          for (int t = 0; t < NT; ++t) {
            float v = 0.f;
            for (int ch = 0; ch < pl.nch; ++ch) v += ldg_cg_f32(&p.partials[(int64_t(ch) * NT + t) * opad + r * V + lane]);
            store_y(t, o, v + bv);
          }
        }
        if (lane == 0) p.counters[r] = 0u;  // leave the counter region zeroed for the next launch
      }
    }
  };

  {
    // ---- rolling gather pipeline ---------------------------------------------------------------
    // The warp walks its work list in groups of 32 fields (one per lane).  U register slots hold
    // the main-codebook entries of U consecutive groups: as soon as slot k has been consumed
    // (residual gather, fp32 FMAs) the gather of group n+U is issued into it, so a lane has U-1..U
    // independent gathers in flight at all times, across segment and row boundaries.  Segment and
    // row boundaries always fall between U-blocks (rows are padded to whole blocks).
    const int gps = pl.seg_fields >> 5;                 // groups per ring segment (multiple of U)
    const int ngu = ((wcols + 32 * U - 1) / (32 * U)) * U;  // groups per unit, padded to whole U-blocks
    const int NG = nunits * ngu;                        // (padding groups decode to field 0, no FMA)
    uint32_t fld[U];
    uint32_t cw[U][V / 2];
    uint32_t rg[RES_L2 ? U : 1][V / 2];  // RES_L2: the residual entries, gathered with the main ones
    const uint8_t* res_bytes = reinterpret_cast<const uint8_t*>(res_g);
    // load side: position of the next group to fetch
    int l_gl = 0, l_st = 0, l_nf = 0;
    uint32_t l_par = 0;
    const uint32_t* l_sw = reinterpret_cast<const uint32_t*>(ring);
    auto load = [&](uint32_t& f_out, uint32_t (&c_out)[V / 2], uint32_t (&r_out)[V / 2]) {
      const int gs_ = l_gl & (gps - 1);
      if (gs_ == 0) {  // first group of a ring segment: wait for its TMA, once
        mbar_wait(&full[l_st], l_par);
        l_sw = reinterpret_cast<const uint32_t*>(ring + l_st * pl.stage_bytes);
        l_nf = min(pl.seg_fields, wcols - (l_gl / gps) * pl.seg_fields);
      }
      const uint32_t f = field_at(l_sw, gs_ * 32 + lane, l_nf);
      f_out = f;
      const uint32_t mi = f & imask;
      if constexpr (MAIN_SMEM) lds_entry<V>(c_out, s_main_lane + mi * main_stride);
      else ldg_entry<V>(c_out, cent_bytes + size_t(mi) * EB, pol_keep);
      if constexpr (RES_L2) ldg_entry<V>(r_out, res_bytes + size_t(f >> p.ib) * EB, pol_keep);
      ++l_gl;
      if (l_gl == ngu || (l_gl & (gps - 1)) == 0) {  // next group starts a new segment (and maybe a new row)
        if (++l_st == pl.stages) l_st = 0, l_par ^= 1u;
        if (l_gl == ngu) l_gl = 0;
      }
    };
    // consume side: groups done in the current unit, current unit, current flat segment
    int c_gl = 0, c_u = 0, c_q = 0;
#pragma unroll
    for (int k = 0; k < U; ++k)
      if (k < NG) load(fld[k], cw[k], rg[RES_L2 ? k : 0]);
    for (int n0 = 0; n0 < NG; n0 += U) {
#pragma unroll
      for (int k = 0; k < U; ++k) {
        const int j = (c_gl + k) * 32 + lane;  // this lane's field, relative to the warp's sub-range
        uint32_t rw[V / 2];
        if constexpr (RES_SMEM) lds_entry<V>(rw, s_res_lane + (fld[k] >> p.ib) * res_stride);
        if constexpr (RES_L2) {
#pragma unroll
          for (int i = 0; i < V / 2; ++i) rw[i] = rg[k][i];
        }
        // lanes past the end gathered entry 0 of both codebooks: they add nothing (not even 0 * entry, which an
        // inf or NaN there would turn into NaN in rows that never use the entry)
        if (j < wcols) {
#pragma unroll
          for (int t = 0; t < NT; ++t) fma_entry<T, V, RES>(acc[t], sx[t * pl.sx_stride + sf0 + j], cw[k], rw);
        }
        if (n0 + k + U < NG) load(fld[k], cw[k], rg[RES_L2 ? k : 0]);  // refill the slot: group n0+k+U
      }
      c_gl += U;
      const bool unit_done = c_gl == ngu;
      if (unit_done || (c_gl & (gps - 1)) == 0) {  // a ring segment has been consumed
        __syncwarp();  // every lane extracted all of its fields (extraction precedes consumption)
        if (c_q + pl.stages < total) issue(c_q + pl.stages);
        ++c_q;
        if (unit_done) {
          finish_row(wslot + nslots * c_u);
          c_gl = 0, ++c_u;
        }
      }
    }
  }

  stamp(8);  // warp 0 finished its rows
  if (wsplit > 1 && wcols == 0)  // (ragged last chunk) nothing to add, but the row's other warps count on us
    for (int u = 0; u < nunits; ++u) finish_row(wslot + nslots * u);

  // -------- cluster epilogue: the leader sums the chunks in order and writes y ---------------
  if (pl.cluster && chunk == 0) {
    mbar_wait(part_bar, 0);  // all nch * nrows_cta * NT * V partial sums have landed
    stamp(9);
    if constexpr (V == 8) {
      // one thread per (row, token): its 8 outputs leave as ONE 16-byte store (locally and, under
      // tensor parallelism, per peer: 8x fewer NVLink packets than element-wise stores)
      for (int i = tid; i < nrows_cta * NT; i += blockDim.x) {
        const int t = i % NT, krow = i / NT;
        const int o0 = (cta_in_chunk + pl.cpc * krow) * V;
        float v[V];
#pragma unroll
        for (int e = 0; e < V; ++e) {
          v[e] = (bias && o0 + e < p.O) ? DT<T>::to_float(bias[o0 + e]) : 0.f;
          for (int ch = 0; ch < pl.nch; ++ch) v[e] += s_part[((krow * pl.nch + ch) * NT + t) * V + e];
        }
        const int64_t off = int64_t(t) * p.y_stride + o0;
        if (o0 + V <= p.O && ((reinterpret_cast<uintptr_t>(y + off) & 15u) == 0)) {
          const uint4 pk = make_uint4(DT<T>::pack2(v[0], v[1]), DT<T>::pack2(v[2], v[3]), DT<T>::pack2(v[4], v[5]),
                                      DT<T>::pack2(v[6], v[7]));
          *reinterpret_cast<uint4*>(y + off) = pk;
          if (p.tp_world > 0) {
            stored_to_peers = true;
#pragma unroll 1
            for (int r = 0; r < p.tp_world; ++r)
              if (r != p.tp_rank) *reinterpret_cast<uint4*>(reinterpret_cast<T*>(p.tp_peer_y[r]) + off) = pk;
          }
        } else {
#pragma unroll
          for (int e = 0; e < V; ++e)
            if (o0 + e < p.O) store_y(t, o0 + e, v[e]);
        }
      }
    } else {
      const int n = nrows_cta * NT * V;
      for (int i = tid; i < n; i += blockDim.x) {
        const int e = i % V, t = (i / V) % NT, krow = i / (V * NT);
        const int o = (cta_in_chunk + pl.cpc * krow) * V + e;
        if (o < p.O) {
          float v = bias ? DT<T>::to_float(bias[o]) : 0.f;
          for (int ch = 0; ch < pl.nch; ++ch) v += s_part[((krow * pl.nch + ch) * NT + t) * V + e];
          store_y(t, o, v);
        }
      }
    }
  }

  // -------- tensor-parallel hand-off: publish this launch's epoch on every peer ------------------
  if (p.tp_world > 0) {
    if (stored_to_peers) __threadfence_system();  // this thread's peer stores are visible system-wide
    __syncthreads();
    if (tid == 0) {
      const uint32_t prev = atomicAdd(p.tp_done + p.tp_slot, 1u);
      if (prev == gdim_total - 1u) {  // the whole launch (all fused layers) has stored its outputs
        p.tp_done[p.tp_slot] = 0u;
        const uint32_t e = ld_volatile_u32(p.tp_epoch + p.tp_slot) + 1u;
        p.tp_epoch[p.tp_slot] = e;
        __threadfence_system();
        for (int r = 0; r < p.tp_world; ++r)
          if (r != p.tp_rank) st_release_sys_u32(p.tp_peer_flags[r] + p.tp_slot * p.tp_world + p.tp_rank, e);
      }
    }
  }
  stamp(10);
}

template <typename T, int V, int NT, bool MAIN_SMEM, bool RES>
__global__ void __launch_bounds__(512, 1) gemv_kernel(const __grid_constant__ GemvParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  gemv_body<T, V, NT, MAIN_SMEM, RES>(p, smem, blockIdx.x, gridDim.x, gridDim.x);
}

// the same for a residual codebook too large for shared memory (planned with GemvPlan::res_rep == 0)
template <typename T, int V, int NT, bool MAIN_SMEM>
__global__ void __launch_bounds__(512, 1) gemv_kernel_res_l2(const __grid_constant__ GemvParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  gemv_body<T, V, NT, MAIN_SMEM, true, true>(p, smem, blockIdx.x, gridDim.x, gridDim.x);
}

// Horizontal fusion: up to 4 layers that read the SAME x (q/k/v, gate/up) in ONE launch.  The grid is
// the concatenation of the layers' own grids (each planned for its share of the SMs); a CTA finds
// its layer from blockIdx.x and then runs the ordinary per-layer body.  One launch, one prologue
// latency, no idle SMs behind a small layer.
constexpr int kMaxFused = kMaxFusedLayers;  // kernels.h
struct GemvMultiParams {
  int n;
  uint32_t grid_begin[kMaxFused + 1];  // layer l owns blocks [grid_begin[l], grid_begin[l+1])
  GemvParams layer[kMaxFused];
};

template <typename T, int V, int NT, bool MAIN_SMEM, bool RES>
__global__ void __launch_bounds__(512, 1) gemv_multi_kernel(const __grid_constant__ GemvMultiParams mp) {
  extern __shared__ __align__(128) uint8_t smem[];
  int l = 0;
#pragma unroll
  for (int i = 1; i < kMaxFused; ++i)
    if (i < mp.n && blockIdx.x >= mp.grid_begin[i]) l = i;
  gemv_body<T, V, NT, MAIN_SMEM, RES>(mp.layer[l], smem, blockIdx.x - mp.grid_begin[l],
                                     mp.grid_begin[l + 1] - mp.grid_begin[l], gridDim.x);
}

template <typename T, int V, int NT, bool MAIN_SMEM>
__global__ void __launch_bounds__(512, 1) gemv_multi_kernel_res_l2(const __grid_constant__ GemvMultiParams mp) {
  extern __shared__ __align__(128) uint8_t smem[];
  int l = 0;
#pragma unroll
  for (int i = 1; i < kMaxFused; ++i)
    if (i < mp.n && blockIdx.x >= mp.grid_begin[i]) l = i;
  gemv_body<T, V, NT, MAIN_SMEM, true, true>(mp.layer[l], smem, blockIdx.x - mp.grid_begin[l],
                                             mp.grid_begin[l + 1] - mp.grid_begin[l], gridDim.x);
}

using GemvKernelFn = void (*)(const GemvParams);
using GemvMultiKernelFn = void (*)(const GemvMultiParams);
// one definition per (dtype, V) translation unit, see gemv_inst_*.cu.  res_l2 (with res): the residual codebook is
// gathered through L1/L2 instead of shared memory
GemvKernelFn gemv_kernel_v8(int dtype, int nt, bool main_smem, bool res, bool res_l2 = false);
GemvKernelFn gemv_kernel_vx(int dtype, int v, bool main_smem, bool res, bool res_l2 = false);
GemvMultiKernelFn gemv_multi_kernel_v8(int dtype, int nt, bool main_smem, bool res, bool res_l2 = false);

}  // namespace vptq_b200
