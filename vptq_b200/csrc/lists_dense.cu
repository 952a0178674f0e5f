// Dense 16-bit weight of a layer from its slice x tile index lists (vptq_linear_desc::lists_*), never from the
// packed index words: the prefill GEMM, dequant and the input gradient of a decode-only descriptor (C interface
// include/vptq_b200_lists_dense.h).
//
// Format (include/vptq_b200.h): unit u = (tile * NS + slice) * Ro + r lists the fields of index row r whose main
// index lies in slice s and whose ORIGINAL feature lies in tile t, as entries
//   (main index & 4095) | (perm[c] - TCW t) << 12 | residual index << 24,
// padded to whole 32-entry steps; tab[u] = first step | valid entries of the last step << 26.  The NS units of one
// (r, t) pair cover every feature of the tile exactly once, so the permutation is folded in: `perm` is never read.
//
// Arithmetic is the packed dequant kernels' (dequant.cu): fmaf(float(C) + float(R), float(scale[f]),
// float(wbias[f])) rounded once to the layer type, scale 1 and bias 0 without a norm, so W and Wt are bit-identical
// to vptq_b200_dequant and to the transposed dequant of the input-gradient GEMM.
//
// Vector length V = 8 (gemv_lists_eligible) or 16 (gemv_lists16_eligible): an index row covers V outputs, an entry
// is V elements -- H = V / 8 halves of 8, each one 16-byte codebook gather, residual read and store.
//
// Work split: one CTA per (index row r, tile t), 256 threads.  The steps of the NS units are laid end to end and
// dealt to the 8 warps step by step (LD_UNROLL steps in flight per warp: 8 independent 16-byte codebook gathers
// per lane), so skewed slices do not leave warps idle.  Residual entries come from a bank-replicated shared-memory
// table (copy k of half h of entry i at slot 8 (H i + h) + k, lane L reads copy L & 7), as in dequant.cu's fast
// paths.
//   * original order W[o][f]: half h of each entry's results (outputs V r + 8 h .. + 7 of feature f) goes to plane h
//     of H [TCW][8] shared tiles (feature slots XOR-swizzled by (f >> 3) & 7); after a barrier a thread owns 8
//     consecutive features, transposes each plane's 8x8 block in registers and writes one 16-byte vector per output
//     row.  At V = 16, TCW <= 4096: 128 KiB of planes + 64 KiB of residual table at Kr = 256.
//   * transposed Wt[f][o]: an entry is V consecutive elements of Wt row f, written as H 16-byte stores (outputs past
//     O as zeros, halves at or past ld skipped); CTAs of index rows past Ro write the zero columns [V Ro, ld).
#include "common.cuh"
#include "kernels.h"

namespace vptq_b200 {

namespace {

constexpr int LD_THREADS = 256, LD_WARPS = LD_THREADS / 32, LD_UNROLL = 8, LD_MAX_SLICES = 16;
constexpr uint32_t LD_STEP_MASK = (1u << 26) - 1u;

struct ListsDenseParams {
  const uint32_t* stream;
  const uint32_t* tab;
  const void* centroids;
  const void* res_centroids;
  const void* scale;  // [I] original order, or nullptr (no norm)
  const void* wbias;
  void* out;
  int64_t ld;
  int I, O, Ro, NS, TCW, Kr;
};

template <typename T, bool TR, int V>
__global__ void __launch_bounds__(LD_THREADS) lists_dense_kernel(const __grid_constant__ ListsDenseParams p) {
  constexpr int H = V / 8;
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ uint32_t s_first[LD_MAX_SLICES + 1], s_step0[LD_MAX_SLICES], s_nsteps[LD_MAX_SLICES],
      s_valid[LD_MAX_SLICES];
  const int r = blockIdx.x, t = blockIdx.y;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int f0 = t * p.TCW, ncols = min(p.TCW, p.I - f0);
  T* out = reinterpret_cast<T*>(p.out);

  if (TR && r >= p.Ro) {  // the zero K tail of Wt: columns [V Ro, ld) of the tile's rows
    for (int h = 0; h < H; ++h) {
      if (V > 8 && int64_t(r) * V + 8 * h >= p.ld) break;
      for (int f = tid; f < ncols; f += LD_THREADS)
        *reinterpret_cast<uint4*>(out + int64_t(f0 + f) * p.ld + int64_t(r) * V + 8 * h) = make_uint4(0u, 0u, 0u, 0u);
    }
    return;
  }

  if (tid < p.NS) {
    const int64_t u = (int64_t(t) * p.NS + tid) * p.Ro + r;
    const uint32_t a = p.tab[u], b = p.tab[u + 1];
    s_step0[tid] = a & LD_STEP_MASK;
    s_nsteps[tid] = (b & LD_STEP_MASK) - (a & LD_STEP_MASK);
    s_valid[tid] = a >> 26;
  }
  uint8_t* s_res = smem;                                   // [Kr][H][8] replicated 16-byte halves
  uint8_t* s_tile = smem + size_t(p.Kr) * 128 * H;         // H x [TCW][8] results (original order only)
  for (int slot = tid; slot < p.Kr * 8 * H; slot += LD_THREADS)
    sts_v4(smem_u32(s_res) + uint32_t(slot) * 16u,
           ldg_nc_v4(reinterpret_cast<const uint8_t*>(p.res_centroids) + size_t(slot >> 3) * 16, policy_evict_last()));
  __syncthreads();
  if (tid == 0) {
    uint32_t acc = 0;
    for (int s = 0; s < p.NS; ++s) s_first[s] = acc, acc += s_nsteps[s];
    s_first[p.NS] = acc;
  }
  __syncthreads();

  const uint32_t total = s_first[p.NS];
  const uint8_t* cb = reinterpret_cast<const uint8_t*>(p.centroids);
  const T* scale = reinterpret_cast<const T*>(p.scale);
  const T* wbias = reinterpret_cast<const T*>(p.wbias);
  const uint32_t res_lane = smem_u32(s_res) + (lane & 7) * 16;
  const uint64_t keep = policy_evict_last();
  const int o0 = r * V;

  for (uint32_t base = warp; base < total; base += LD_WARPS * LD_UNROLL) {
    uint32_t ent[LD_UNROLL], sl[LD_UNROLL];
    bool ok[LD_UNROLL];
#pragma unroll
    for (int i = 0; i < LD_UNROLL; ++i) {
      const uint32_t g = base + uint32_t(i) * LD_WARPS;  // warp-uniform
      ok[i] = false, ent[i] = 0u, sl[i] = 0u;
      if (g < total) {
        int s = 0;
        while (s + 1 < p.NS && s_first[s + 1] <= g) ++s;
        const uint32_t k = g - s_first[s];
        ok[i] = k + 1 < s_nsteps[s] || uint32_t(lane) < s_valid[s];  // padding of the unit's last step: masked
        sl[i] = uint32_t(s);
        if (ok[i]) ent[i] = ldg_nc_u32(p.stream + (size_t(s_step0[s]) + k) * 32 + lane);
      }
    }
    uint4 cw[LD_UNROLL][H];
#pragma unroll
    for (int i = 0; i < LD_UNROLL; ++i)
#pragma unroll
      for (int h = 0; h < H; ++h)
        cw[i][h] = ok[i] ? ldg_nc_v4(cb + (size_t(sl[i] << 12) | (ent[i] & 4095u)) * (16 * H) + 16 * h, keep)
                         : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
    for (int i = 0; i < LD_UNROLL; ++i) {
      if (!ok[i]) continue;
      const int col = int((ent[i] >> 12) & 4095u), f = f0 + col;
      const float sc = scale ? DT<T>::to_float(scale[f]) : 1.f, wb = scale ? DT<T>::to_float(wbias[f]) : 0.f;
#pragma unroll
      for (int h = 0; h < H; ++h) {
        uint4 rw = make_uint4(0u, 0u, 0u, 0u);
        if (p.Kr) rw = lds_v4(res_lane + (ent[i] >> 24) * (128 * H) + 128 * h);
        const uint32_t cwk[4] = {cw[i][h].x, cw[i][h].y, cw[i][h].z, cw[i][h].w}, rwk[4] = {rw.x, rw.y, rw.z, rw.w};
        uint32_t hv[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float2 c2 = DT<T>::unpack2(cwk[j]);
          if (p.Kr) {
            const float2 r2 = DT<T>::unpack2(rwk[j]);
            c2.x += r2.x, c2.y += r2.y;
          }
          hv[j] = DT<T>::pack2(fmaf(c2.x, sc, wb), fmaf(c2.y, sc, wb));
          if (TR) {  // outputs past O (padding rows of the last index row): zeros
            const int o = o0 + 8 * h + 2 * j;
            if (o >= p.O) hv[j] = 0u;
            else if (o + 1 >= p.O) hv[j] &= 0xffffu;
          }
        }
        if (TR) {
          if (V > 8 && o0 + 8 * h >= p.ld) break;  // a last half wholly past ld (ld % 16 == 8): all padding
          *reinterpret_cast<uint4*>(out + int64_t(f) * p.ld + o0 + 8 * h) = make_uint4(hv[0], hv[1], hv[2], hv[3]);
        } else {
          const uint32_t slot = uint32_t(col) ^ ((uint32_t(col) >> 3) & 7u);
          sts_v4(smem_u32(s_tile) + uint32_t(h * p.TCW) * 16u + slot * 16u, make_uint4(hv[0], hv[1], hv[2], hv[3]));
        }
      }
    }
  }
  if (TR) return;
  __syncthreads();

  // 8 consecutive features per thread: per plane an 8x8 register transpose, one 16-byte store per output row
  const int rows = min(V, p.O - o0);  // padding rows are never written
  for (int h = 0; h < H; ++h) {
    const int rh = H == 1 ? rows : min(8, rows - 8 * h);  // rows of plane h
    if (V > 8 && rh <= 0) break;
    const uint32_t plane = smem_u32(s_tile) + uint32_t(h * p.TCW) * 16u;
    const int oh = o0 + 8 * h;
    for (int j = tid; j * 8 < ncols; j += LD_THREADS) {
      uint32_t hv[8][4];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const uint4 v = lds_v4(plane + uint32_t(j * 8 + (k ^ (j & 7))) * 16u);
        hv[k][0] = v.x, hv[k][1] = v.y, hv[k][2] = v.z, hv[k][3] = v.w;
      }
      const int fb = f0 + j * 8;
      if (j * 8 + 8 <= ncols) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          if (e >= rh) break;
          const uint32_t sel = (e & 1) ? 0x7632u : 0x5410u;
          uint4 v;
          v.x = __byte_perm(hv[0][e >> 1], hv[1][e >> 1], sel);
          v.y = __byte_perm(hv[2][e >> 1], hv[3][e >> 1], sel);
          v.z = __byte_perm(hv[4][e >> 1], hv[5][e >> 1], sel);
          v.w = __byte_perm(hv[6][e >> 1], hv[7][e >> 1], sel);
          *reinterpret_cast<uint4*>(out + int64_t(oh + e) * p.ld + fb) = v;
        }
      } else {  // the last tile's ragged end (in_features % 8 != 0)
        uint16_t* o16 = reinterpret_cast<uint16_t*>(p.out);
#pragma unroll
        for (int k = 0; k < 8; ++k)
#pragma unroll
          for (int e = 0; e < 8; ++e)
            if (k < ncols - j * 8 && e < rh)
              o16[int64_t(oh + e) * p.ld + fb + k] = uint16_t(hv[k][e >> 1] >> ((e & 1) * 16));
      }
    }
  }
  if (f0 + ncols == p.I) {  // the last tile's CTAs write the zero columns [I, ld) of their rows
    uint16_t* o16 = reinterpret_cast<uint16_t*>(p.out);
    const int pad = int(p.ld - p.I);
    for (int i = tid; i < rows * pad; i += LD_THREADS) o16[int64_t(o0 + i / pad) * p.ld + p.I + i % pad] = 0;
  }
}

}  // namespace

size_t lists_dense_smem_bytes(const vptq_linear_desc& d, bool transposed) {
  const size_t H = d.vector_len / 8;
  const size_t res = d.num_res_centroids > 0 ? size_t(d.num_res_centroids) * 128 * H : 0;
  return res + (transposed ? 0 : size_t(d.lists_tile_cols) * 16 * H);
}

template <int V>
int lists_dense_launch_v(const ListsDenseParams& p, int dtype, bool transposed, dim3 grid, size_t smem,
                         cudaStream_t stream) {
  const void* fn;
  if (dtype == VPTQ_FP16)
    fn = transposed ? reinterpret_cast<const void*>(lists_dense_kernel<__half, true, V>)
                    : reinterpret_cast<const void*>(lists_dense_kernel<__half, false, V>);
  else
    fn = transposed ? reinterpret_cast<const void*>(lists_dense_kernel<__nv_bfloat16, true, V>)
                    : reinterpret_cast<const void*>(lists_dense_kernel<__nv_bfloat16, false, V>);
  if (int rc = ensure_smem_attr(fn, (V == 8 ? 100 : 200) * 1024)) return rc;
  if (dtype == VPTQ_FP16) {
    if (transposed) lists_dense_kernel<__half, true, V><<<grid, LD_THREADS, smem, stream>>>(p);
    else lists_dense_kernel<__half, false, V><<<grid, LD_THREADS, smem, stream>>>(p);
  } else {
    if (transposed) lists_dense_kernel<__nv_bfloat16, true, V><<<grid, LD_THREADS, smem, stream>>>(p);
    else lists_dense_kernel<__nv_bfloat16, false, V><<<grid, LD_THREADS, smem, stream>>>(p);
  }
  return 0;
}

int lists_dense_launch(const vptq_linear_desc& d, void* out, int64_t ld, bool transposed, cudaStream_t stream) {
  ListsDenseParams p{};
  p.stream = d.lists_stream, p.tab = d.lists_tab;
  p.centroids = d.centroids, p.res_centroids = d.res_centroids;
  p.scale = d.weight_scale, p.wbias = d.weight_scale ? d.weight_bias : nullptr;
  p.out = out, p.ld = ld;
  const int V = d.vector_len;  // 8 or 16: the caller checked gemv_lists_eligible or gemv_lists16_eligible
  p.I = d.in_features, p.O = d.out_features, p.Ro = (d.out_features + V - 1) / V;
  p.NS = d.num_centroids / 4096, p.TCW = d.lists_tile_cols;
  p.Kr = d.num_res_centroids > 0 ? d.num_res_centroids : 0;
  const int nt = (d.in_features + p.TCW - 1) / p.TCW;
  const size_t smem = lists_dense_smem_bytes(d, transposed);
  dim3 grid(unsigned(transposed ? (ld + V - 1) / V : p.Ro), unsigned(nt));
  if (int rc = V == 16 ? lists_dense_launch_v<16>(p, d.dtype, transposed, grid, smem, stream)
                       : lists_dense_launch_v<8>(p, d.dtype, transposed, grid, smem, stream))
    return rc;
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("lists dense weight launch: %s", cudaGetErrorString(e));
    return VPTQ_ERR_CUDA;
  }
  return 0;
}

}  // namespace vptq_b200
