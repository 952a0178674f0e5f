// Host side of the decode GEMV: work decomposition (GemvPlan), shared-memory carve-up, launch.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <tuple>
#include <set>
#include <unordered_set>
#include <vector>

#include "gemv_kernel.cuh"

namespace vptq_b200 {

namespace {

constexpr int kMaxChunkCols = 4096;      // bounds the x' slice in shared memory (16 KB per token)
constexpr int kSmemReserve = 2048;       // head-room below the opt-in limit
constexpr int kMaxClusterPartBytes = 16384;

bool supported_vec_len(int v) { return v == 2 || v == 4 || v == 6 || v == 8 || v == 10 || v == 12 || v == 16; }

std::mutex g_mutex;
std::set<std::pair<int, const void*>> g_attr_done;  // (device, kernel): the attribute is per device
std::map<std::tuple<const void*, int, int, int>, int> g_max_clusters;

// Developer tuning knobs (not part of the ABI): VPTQ_B200_GEMV_TUNE="rep=1,stages=2,seg=512,warps=16,cpg=4,wsplit=2,cluster=0,lists=0"
struct Tune {
  int rep = -1, stages = 0, seg = 0, warps = 0, cpg = 0, cluster = -1, wsplit = 0, lists = -1;
};
const Tune& tune() {
  static Tune t = [] {
    Tune r;
    const char* e = std::getenv("VPTQ_B200_GEMV_TUNE");
    if (!e) return r;
    auto get = [&](const char* key, int& dst) {
      const char* p = std::strstr(e, key);
      if (p) dst = std::atoi(p + std::strlen(key));
    };
    get("rep=", r.rep), get("stages=", r.stages), get("seg=", r.seg), get("warps=", r.warps), get("cpg=", r.cpg),
        get("cluster=", r.cluster), get("wsplit=", r.wsplit), get("lists=", r.lists);
    return r;
  }();
  return t;
}

GemvKernelFn pick_kernel(const vptq_linear_desc& d, int nt, bool main_smem) {
  const bool res = d.num_res_centroids > 0;
  return d.vector_len == 8 ? gemv_kernel_v8(d.dtype, nt, main_smem, res)
                           : gemv_kernel_vx(d.dtype, d.vector_len, main_smem, res);
}

}  // namespace

int ensure_smem_attr(const void* fn, int bytes) {
  // cudaFuncSetAttribute applies to the CURRENT device only: a process that drives several GPUs (HF
  // device_map="auto", pipeline splits) must opt in once per (device, kernel)
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lock(g_mutex);
  if (g_attr_done.count({dev, fn})) return 0;
  cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) {
    set_error("cudaFuncSetAttribute(max dynamic smem=%d): %s", bytes, cudaGetErrorString(e));
    return VPTQ_ERR_CUDA;
  }
  g_attr_done.insert({dev, fn});
  return 0;
}

// how many clusters of `csize` CTAs (threads, smem each) the device can hold at once; <= 0: unknown
int max_active_clusters(const void* fn, int csize, int threads, int smem, int optin) {
  {
    std::lock_guard<std::mutex> lock(g_mutex);
    auto it = g_max_clusters.find({fn, csize, threads, smem});
    if (it != g_max_clusters.end()) return it->second;
  }
  if (ensure_smem_attr(fn, optin)) return -1;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(unsigned(csize));
  cfg.blockDim = dim3(unsigned(threads));
  cfg.dynamicSmemBytes = size_t(smem);
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = unsigned(csize), at[0].val.clusterDim.y = 1, at[0].val.clusterDim.z = 1;
  cfg.attrs = at, cfg.numAttrs = 1;
  int n = -1;
  if (cudaOccupancyMaxActiveClusters(&n, fn, &cfg) != cudaSuccess) {
    cudaGetLastError();
    n = -1;
  }
  std::lock_guard<std::mutex> lock(g_mutex);
  g_max_clusters[{fn, csize, threads, smem}] = n;
  return n;
}

int gemv_tune_lists() { return tune().lists; }

// developer aid: phase-stamp buffer (device pointer) handed to every subsequent GEMV launch
static unsigned long long* g_prof_buffer = nullptr;
void gemv_set_profile_buffer(void* dev_ptr) { g_prof_buffer = static_cast<unsigned long long*>(dev_ptr); }
unsigned long long* gemv_profile_buffer() { return g_prof_buffer; }

int gemv_make_plan(const vptq_linear_desc& d, int tokens, const DeviceInfo& dev, GemvPlan* out, int slots_override,
                   int force_cpg) {
  const int v = d.vector_len, G = d.num_codebooks, gs = d.group_size;
  const int Ro = (d.out_features + v - 1) / v;
  const int ib = ilog2(d.num_centroids);
  const int rb = d.num_res_centroids > 0 ? ilog2(d.num_res_centroids) : 0;
  const int b = ib + rb;
  const int S = (d.outlier_size > 0 && d.outlier_indices) ? d.outlier_size : 0;
  const int EB = 2 * v;
  const int sms = dev.sm_count;
  const Tune& tn = tune();
  if (Ro > kMaxIndexRows) {
    set_error("gemv: %d index rows exceed the supported maximum %d", Ro, kMaxIndexRows);
    return VPTQ_ERR_UNSUPPORTED;
  }

  GemvPlan pl{};
  pl.nt = (v == 8) ? (tokens >= 4 ? 4 : (tokens >= 2 ? 2 : 1)) : 1;
  pl.seg_fields = tn.seg ? tn.seg : 512;
  pl.stage_bytes = uint32_t(align_up(size_t(pl.seg_fields) * b / 8 + 16, 16));
  pl.ctas_per_sm = 1;

  const size_t main_bytes = size_t(d.num_centroids) * EB;
  const size_t res_bytes = rb ? size_t(d.num_res_centroids) * EB : 0;
  const bool main_fits = main_bytes <= 131072;
  const int main_rep_smem = (v == 8 && main_bytes * 8 <= 32768) ? 8 : 1;
  const int res_rep_want = tn.rep >= 0 ? (tn.rep ? 8 : 1) : 8;
  const int res_rep_max = (rb && v == 8 && res_bytes * 8 <= 32768) ? res_rep_want : 1;
  const int smem_limit = dev.smem_optin - kSmemReserve;
  // one CTA per SM: the whole register file and shared memory feed one pipeline; a fused launch
  // gives every layer its share of the SMs
  const int slots = slots_override > 0 ? std::min(slots_override, sms) : sms;

  // One attempt = (warps per CTA, main codebook in shared memory?).  First fit wins.
  struct Attempt { int warps; bool main_smem; };
  const Attempt attempts[] = {{16, true}, {8, true}, {16, false}, {8, false}};
  for (const Attempt& a : attempts) {
    if (a.main_smem && !main_fits) continue;
    if (tn.warps && a.warps != tn.warps) continue;

    // ---- column chunks (cpg per codebook group, multiples of 128 columns) x warps per row -------
    // A CTA streams rows_cta * cc fields; its nwarps/wsplit row slots work in parallel, each row
    // cut over wsplit warps.  Chunk counts up to 8 reduce through a cluster (the co-schedulable
    // cluster count can leave SMs idle: a cluster must fit inside one GPC), more than 8
    // through global memory.
    GemvKernelFn fn_probe = pick_kernel(d, pl.nt, a.main_smem);
    int best_cpg = 0, best_cc = 0, best_ws = 1;
    double best_cost = 1e300;
    for (int cpg = 1; cpg <= 64; cpg *= 2) {
      if (tn.cpg && cpg != tn.cpg) continue;
      if (force_cpg && cpg != force_cpg) continue;
      const int cc = int(align_up(size_t((gs + cpg - 1) / cpg), 128));
      if (cc > kMaxChunkCols) continue;
      if (cpg > 1 && cc < 256) break;
      const int real_cpg = (gs + cc - 1) / cc;
      const int nch = G * real_cpg;
      if (nch > slots) break;
      int cpc = std::max(1, std::min(slots / nch, Ro));
      if (nch >= 2 && nch <= 8 && dev.device >= 0 && fn_probe && tn.cluster != 0) {
        const int n = max_active_clusters(reinterpret_cast<const void*>(fn_probe), nch, a.warps * 32, 200 * 1024,
                                          dev.smem_optin);
        if (n > 0) cpc = std::min(cpc, n);
      }
      const int rows_cta = (Ro + cpc - 1) / cpc;
      for (int ws = 1; ws <= 4; ws *= 2) {
        if (tn.wsplit && ws != tn.wsplit) continue;
        const int sub = int(align_up(size_t((cc + ws - 1) / ws), 128));
        if (ws > 1 && (sub < 256 || (ws - 1) * sub >= cc)) continue;
        const int nslots = a.warps / ws;
        const int rounds = (rows_cta + nslots - 1) / nslots;
        const double util = double(rows_cta) * ws / (double(rounds) * a.warps);
        double cost = double(rows_cta) * cc * (1.0 + 0.5 * (1.0 - util)) + 600.0 + 0.35 * cc;
        cost += (nch <= 8 ? 24.0 : 96.0) * rows_cta + (ws > 1 ? 16.0 * rows_cta : 0.0);
        cost *= 1.0 + 0.01 * ilog2(real_cpg);  // ties go to fewer, wider chunks
        if (cost < best_cost) best_cost = cost, best_cpg = real_cpg, best_cc = cc, best_ws = ws;
      }
    }
    if (!best_cpg) {  // very wide single group: the widest legal chunk
      best_cc = kMaxChunkCols;
      best_cpg = (gs + kMaxChunkCols - 1) / kMaxChunkCols;
      best_ws = 1;
    }
    pl.chunk_cols = best_cc, pl.cpg = best_cpg, pl.nch = G * best_cpg;
    pl.wsplit = best_ws;
    pl.sub_cols = best_ws > 1 ? int(align_up(size_t((best_cc + best_ws - 1) / best_ws), 128)) : best_cc;
    if (pl.nch > slots) continue;
    pl.cpc = std::max(1, std::min(slots / pl.nch, Ro));
    const int rows_cta = (Ro + pl.cpc - 1) / pl.cpc;
    const int rows_alloc = rows_cta + rows_cta / 4 + 1;  // cpc may still be clamped below: 25% slack
    // cluster reduce: the leader holds every row's chunk partials
    const size_t part_bytes = size_t(rows_alloc) * pl.nch * pl.nt * v * 4;
    pl.cluster = (pl.nch >= 2 && pl.nch <= 8 && part_bytes <= kMaxClusterPartBytes && tn.cluster != 0) ? 1 : 0;
    pl.main_in_smem = a.main_smem ? 1 : 0;
    pl.main_rep = a.main_smem ? main_rep_smem : 1;

    // ---- shared memory carve-up ----------------------------------------------------------------
    auto carve = [&](int warps, int stages, int res_rep) -> size_t {
      pl.res_rep = res_rep;
      size_t off = 0;
      pl.off_bars = uint32_t(off);
      off += align_up(size_t(2 + warps * stages) * 8, 128);
      pl.off_cbias = uint32_t(off);
      off += align_up(size_t(pl.nt) * (1 + warps) * 4, 128);
      const int n_all = pl.chunk_cols + S;
      pl.sx_stride = int(align_up(size_t(n_all), 32));
      pl.off_pcol = uint32_t(off);
      off += align_up(size_t(n_all) * 2, 128);
      pl.off_wb = uint32_t(off);
      off += align_up(size_t(n_all) * 4, 128);
      pl.off_sx = uint32_t(off);
      off += align_up(size_t(pl.nt) * pl.sx_stride * 4, 128);
      pl.off_part = uint32_t(off);
      if (pl.cluster) off += align_up(part_bytes, 128);
      pl.off_wsum = uint32_t(off);
      if (pl.wsplit > 1) off += align_up(size_t(rows_alloc) * pl.wsplit * pl.nt * v * 4, 128);
      pl.off_wcnt = uint32_t(off);
      if (pl.wsplit > 1) off += align_up(size_t(rows_alloc) * 4, 128);
      pl.off_res = uint32_t(off);
      off += align_up(res_bytes * res_rep, 128);
      pl.off_main = uint32_t(off);
      if (a.main_smem) off += align_up(main_bytes * pl.main_rep, 128);
      pl.off_raw = uint32_t(off);
      off += align_up((res_rep > 1 ? res_bytes : 0) + (a.main_smem && pl.main_rep > 1 ? main_bytes : 0), 128);
      pl.off_ring = uint32_t(off);
      off += align_up(size_t(warps) * stages * pl.stage_bytes, 128);
      return off;
    };
    // what to shed, in order, until the layout fits.  L2-gather layers: a small footprint leaves
    // more of the 256 KB L1/shared array to cache codebook lines (measured: 2 stages beat 4);
    // smem-resident codebooks take the deeper ring.
    struct Shape { int stages, rep; };
    std::vector<Shape> shapes;
    for (int st : (a.main_smem ? std::vector<int>{4, 3, 2} : std::vector<int>{2}))
      for (int rep : {res_rep_max, 1}) shapes.push_back({st, rep});
    bool placed = false;
    for (const Shape& sh : shapes) {
      if (tn.stages && sh.stages != tn.stages) continue;
      const size_t need = carve(a.warps, sh.stages, sh.rep);
      if (need <= size_t(smem_limit)) {
        pl.threads = a.warps * 32, pl.stages = sh.stages, pl.smem_bytes = uint32_t(need);
        placed = true;
        break;
      }
    }
    if (!placed) continue;

    // ---- clusters must all be co-resident: a second wave would double the kernel ----------------
    if (pl.cluster && dev.device >= 0) {
      GemvKernelFn fn = fn_probe;
      const int n = fn ? max_active_clusters(reinterpret_cast<const void*>(fn), pl.nch, pl.threads,
                                             int(pl.smem_bytes), dev.smem_optin)
                       : -1;
      if (n > 0 && n < pl.cpc) pl.cpc = n;
      const int rows2 = (Ro + pl.cpc - 1) / pl.cpc;
      if (rows2 > rows_alloc) pl.cluster = 0;
    }
    pl.grid = pl.nch * pl.cpc;
    pl.ws_counters_bytes = kZeroRegionBytes;
    pl.ws_partials_bytes = (pl.nch > 1 && !pl.cluster) ? align_up(size_t(pl.nch) * pl.nt * Ro * v * 4, 256) : 0;
    *out = pl;
    return 0;
  }
  set_error("gemv: no shared-memory layout fits (residual codebook %zu bytes, %d column groups)", res_bytes, G);
  return VPTQ_ERR_UNSUPPORTED;
}

namespace {

void fill_params(GemvParams& p, const vptq_linear_desc& d, const GemvPlan& pl, int64_t x_stride, int64_t y_stride,
                 void* workspace) {
  p = GemvParams{};
  p.indices = reinterpret_cast<const uint32_t*>(d.indices);
  p.idx_stride_g = d.index_stride_codebook;
  p.idx_stride_r = d.index_stride_row;
  p.centroids = d.centroids;
  p.cb_stride = d.centroid_stride;
  p.res_centroids = d.res_centroids;
  p.rcb_stride = d.res_centroid_stride;
  p.I = d.in_features, p.O = d.out_features, p.G = d.num_codebooks, p.gs = d.group_size;
  p.Ro = (d.out_features + d.vector_len - 1) / d.vector_len;
  p.K = d.num_centroids, p.ib = ilog2(d.num_centroids);
  p.Kr = d.num_res_centroids > 0 ? d.num_res_centroids : 0;
  p.rb = p.Kr ? ilog2(p.Kr) : 0;
  p.S = (d.outlier_size > 0 && d.outlier_indices) ? d.outlier_size : 0;
  p.vol = p.S ? d.outlier_vector_len : 1;
  p.Kol = p.S ? d.num_outlier_centroids : 0;
  p.Rol = p.S ? (d.out_features + p.vol - 1) / p.vol : 0;
  p.outlier_idx = p.S ? d.outlier_indices : nullptr;
  p.outlier_cb = p.S ? d.outlier_centroids : nullptr;
  p.perm = d.perm;
  p.scale = d.weight_scale;
  p.wbias = d.weight_bias;
  p.scale_q = d.weight_scale_q;
  p.wbias_q = d.weight_bias_q;
  p.bias = d.bias;
  p.x_stride = x_stride, p.y_stride = y_stride;
  p.counters = reinterpret_cast<uint32_t*>(workspace);
  p.partials = workspace ? reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(workspace) + pl.ws_counters_bytes)
                         : nullptr;
  p.idx_tma_ok = ((reinterpret_cast<uintptr_t>(d.indices) & 15u) == 0 && (d.index_stride_row & 3) == 0 &&
                  (d.index_stride_codebook & 3) == 0)
                     ? 1
                     : 0;
  p.prof = g_prof_buffer;
  p.plan = pl;
}

template <typename Fn, typename Params>
int launch(Fn fn, const Params& params, int grid, int threads, uint32_t smem, int cluster, uint32_t flags,
           cudaStream_t stream) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(unsigned(grid));
  cfg.blockDim = dim3(unsigned(threads));
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int nattr = 0;
  if (flags & VPTQ_FLAG_PDL) {
    attr[nattr].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[nattr].val.programmaticStreamSerializationAllowed = 1;
    ++nattr;
  }
  if (cluster > 1) {
    attr[nattr].id = cudaLaunchAttributeClusterDimension;
    attr[nattr].val.clusterDim.x = unsigned(cluster);
    attr[nattr].val.clusterDim.y = 1;
    attr[nattr].val.clusterDim.z = 1;
    ++nattr;
  }
  cfg.attrs = attr;
  cfg.numAttrs = unsigned(nattr);
  cudaError_t e = cudaLaunchKernelEx(&cfg, fn, params);
  if (e != cudaSuccess) {
    set_error("gemv launch (grid=%d block=%d smem=%u cluster=%d): %s", grid, threads, smem, cluster, cudaGetErrorString(e));
    return VPTQ_ERR_CUDA;
  }
  return 0;
}

}  // namespace

int gemv_launch(const vptq_linear_desc& d, const void* x, int64_t x_stride, void* y, int64_t y_stride,
                int tokens, void* workspace, size_t workspace_bytes, uint32_t flags, cudaStream_t stream) {
  const DeviceInfo* dev = device_info();
  if (!dev) return VPTQ_ERR_CUDA;
  if (!supported_vec_len(d.vector_len)) {
    set_error("gemv: vector_len %d not supported (2,4,6,8,10,12,16)", d.vector_len);
    return VPTQ_ERR_UNSUPPORTED;
  }
  // decode proper (one token) of a layer that carries slice x tile lists: shared-memory gathers
  if (tokens == 1 && gemv_tune_lists() != 0 && gemv_lists_eligible(d)) {
    const vptq_linear_desc* dp = &d;
    void* yp = y;
    const int rc = gemv_lists_launch(1, &dp, x, &yp, flags, stream, workspace, workspace_bytes);
    if (rc != VPTQ_ERR_UNSUPPORTED && rc != VPTQ_ERR_WORKSPACE) return rc;
  }
  if (!d.indices) {
    set_error("gemv: this descriptor is decode-only (indices == NULL): only single-token calls through the index "
              "lists are possible (tokens %d, workspace %zu bytes)", tokens, workspace_bytes);
    return VPTQ_ERR_UNSUPPORTED;
  }
  GemvPlan pl;
  if (int rc = gemv_make_plan(d, tokens, *dev, &pl)) return rc;
  const size_t need = pl.ws_partials_bytes ? pl.ws_counters_bytes + pl.ws_partials_bytes : 0;
  if (need && (workspace_bytes < need || !workspace)) {
    set_error("gemv: workspace %zu bytes < required %zu", workspace_bytes, need);
    return VPTQ_ERR_WORKSPACE;
  }
  GemvParams p;
  fill_params(p, d, pl, x_stride, y_stride, workspace);
  const size_t esz = 2;
  for (int t0 = 0; t0 < tokens;) {
    int nt = pl.nt;
    while (nt > tokens - t0) nt >>= 1;  // tail passes: 4 -> 2 -> 1
    GemvKernelFn fn = pick_kernel(d, nt, pl.main_in_smem != 0);
    if (!fn) {
      set_error("gemv: no kernel for dtype=%d v=%d nt=%d", d.dtype, d.vector_len, nt);
      return VPTQ_ERR_UNSUPPORTED;
    }
    if (int rc = ensure_smem_attr(reinterpret_cast<const void*>(fn), dev->smem_optin)) return rc;
    p.x = reinterpret_cast<const uint8_t*>(x) + size_t(t0) * x_stride * esz;
    p.y = reinterpret_cast<uint8_t*>(y) + size_t(t0) * y_stride * esz;
    // the carve-up was sized for pl.nt tokens; a narrower tail pass fits a fortiori (the kernel's
    // partial-sum indexing uses its own template NT consistently on both sides)
    if (int rc = launch(fn, p, pl.grid, pl.threads, pl.smem_bytes, pl.cluster ? pl.nch : 1, flags, stream)) return rc;
    t0 += nt;
  }
  return 0;
}

// Several layers reading the same x in one launch (q/k/v, gate/up).  Every layer gets a share of the
// SMs proportional to its index volume and is planned for that share; the launch needs one kernel
// instantiation, one block size and one cluster size for all of them -- otherwise (or when a layer
// needs the global-memory split-K variant) VPTQ_ERR_UNSUPPORTED tells the caller to launch separately.
int gemv_multi_launch(int n, const vptq_linear_desc* const* descs, const void* x, int64_t x_stride, void* const* ys,
                      const int64_t* y_strides, int tokens, uint32_t flags, cudaStream_t stream,
                      const vptq_tp_exchange* tp, void* workspace, size_t workspace_bytes) {
  const DeviceInfo* dev = device_info();
  if (!dev) return VPTQ_ERR_CUDA;
  if (n < 1 || n > kMaxFused || tokens < 1 || tokens > 2) {
    set_error("gemv_multi: 1..%d layers and 1..2 tokens (got %d layers, %d tokens)", kMaxFused, n, tokens);
    return VPTQ_ERR_UNSUPPORTED;
  }
  if (tokens == 1 && gemv_tune_lists() != 0 && workspace) {
    bool all = true;
    for (int l = 0; l < n; ++l) all = all && gemv_lists_eligible(*descs[l]);
    if (all) {
      const int rc = gemv_lists_launch(n, descs, x, ys, flags, stream, workspace, workspace_bytes, tp);
      if (rc != VPTQ_ERR_UNSUPPORTED && rc != VPTQ_ERR_WORKSPACE) return rc;
    }
  }
  if (tp && tp->world > 1 && tp->format == VPTQ_TP_TAGGED) {
    set_error("gemv_multi: the tagged exchange format is implemented by the list kernel only (layers without index "
              "lists, several tokens or no workspace: use VPTQ_TP_PLAIN)");
    return VPTQ_ERR_UNSUPPORTED;
  }
  for (int l = 0; l < n; ++l)
    if (!descs[l]->indices) {
      set_error("gemv_multi: layer %d is decode-only (indices == NULL) and this launch cannot use the index lists", l);
      return VPTQ_ERR_UNSUPPORTED;
    }
  const vptq_linear_desc& d0 = *descs[0];
  double vol[kMaxFused], total = 0;
  for (int l = 0; l < n; ++l) {
    const vptq_linear_desc& d = *descs[l];
    if (d.vector_len != 8 || d.dtype != d0.dtype || d.in_features != d0.in_features ||
        (d.num_res_centroids > 0) != (d0.num_res_centroids > 0)) {
      set_error("gemv_multi: layers must share dtype, in_features, vector_len 8 and residual-ness");
      return VPTQ_ERR_UNSUPPORTED;
    }
    vol[l] = double((d.out_features + 7) / 8) * d.in_features;
    total += vol[l];
  }
  // plan the largest layer first: its chunking (cluster size) is imposed on the others
  int big = 0;
  for (int l = 1; l < n; ++l)
    if (vol[l] > vol[big]) big = l;
  GemvPlan plans[kMaxFused];
  // 1. provisional plan of the largest layer -> chunking / cluster size for everyone
  if (int rc = gemv_make_plan(*descs[big], tokens, *dev, &plans[big], std::max(8, int(dev->sm_count * vol[big] / total)), 0))
    return rc;
  const int cpg = plans[big].cpg, nch = plans[big].nch;
  // 2. SMs that can be used at once: all clusters of all layers must be co-resident
  int avail = dev->sm_count;
  if (plans[big].cluster) {
    GemvKernelFn probe = pick_kernel(*descs[big], plans[big].nt, plans[big].main_in_smem != 0);
    const int nmax = probe ? max_active_clusters(reinterpret_cast<const void*>(probe), nch, plans[big].threads,
                                                 200 * 1024, dev->smem_optin)
                           : -1;
    if (nmax > 0) avail = std::min(avail, nmax * nch);
  }
  // 3. shares proportional to index volume, in whole clusters
  int share[kMaxFused], used = 0;
  for (int l = 0; l < n; ++l) {
    share[l] = std::max(nch, int(avail * vol[l] / total) / nch * nch);
    used += share[l];
  }
  while (used > avail && share[big] > nch) share[big] -= nch, used -= nch;
  if (used > avail) {
    set_error("gemv_multi: %d layers do not fit %d co-resident CTAs", n, avail);
    return VPTQ_ERR_UNSUPPORTED;
  }
  while (used + nch <= avail) share[big] += nch, used += nch;  // hand the remainder to the largest layer
  for (int l = 0; l < n; ++l)
    if (int rc = gemv_make_plan(*descs[l], tokens, *dev, &plans[l], share[l], cpg)) return rc;
  GemvMultiParams mp{};
  mp.n = n;
  uint32_t smem = 0, begin = 0;
  for (int l = 0; l < n; ++l) {
    const GemvPlan& pl = plans[l];
    if (pl.nch != plans[big].nch || pl.threads != plans[big].threads || pl.cluster != plans[big].cluster ||
        pl.main_in_smem != plans[big].main_in_smem || pl.nt != plans[big].nt || pl.ws_partials_bytes) {
      set_error("gemv_multi: the layers do not admit one launch configuration");
      return VPTQ_ERR_UNSUPPORTED;
    }
    fill_params(mp.layer[l], *descs[l], pl, x_stride, y_strides[l], nullptr);
    mp.layer[l].x = x;
    mp.layer[l].y = ys[l];
    if (tp && tp->world > 1) {
      GemvParams& q = mp.layer[l];
      q.tp_world = tp->world, q.tp_rank = tp->rank, q.tp_slot = tp->slot, q.tp_wait_slot = tp->wait_slot;
      for (int r = 0; r < tp->world; ++r) q.tp_peer_y[r] = tp->peer_y[l][r], q.tp_peer_flags[r] = tp->peer_flags[r];
      q.tp_epoch = tp->epoch, q.tp_done = tp->done, q.tp_error = tp->error;
    }
    mp.grid_begin[l] = begin;
    begin += uint32_t(pl.grid);
    smem = std::max(smem, pl.smem_bytes);
  }
  for (int l = n; l <= kMaxFused; ++l) mp.grid_begin[l] = begin;
  GemvMultiKernelFn fn = gemv_multi_kernel_v8(d0.dtype, plans[big].nt, plans[big].main_in_smem != 0, d0.num_res_centroids > 0);
  if (!fn || plans[big].nt != tokens) {
    set_error("gemv_multi: no fused kernel for this configuration");
    return VPTQ_ERR_UNSUPPORTED;
  }
  if (int rc = ensure_smem_attr(reinterpret_cast<const void*>(fn), dev->smem_optin)) return rc;
  return launch(fn, mp, int(begin), plans[big].threads, smem, plans[big].cluster ? plans[big].nch : 1, flags, stream);
}

}  // namespace vptq_b200
