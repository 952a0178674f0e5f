// Weight gradients of a VPTQ layer: the codebooks (main, residual, outlier), weight_scale and weight_bias
// (semantics and C interface: include/vptq_b200_grad.h).
//
// Two entry points share one reduction:
//   vptq_b200_quant_gemm_wgrad   G = dY^T x for y = x W^T + bias.  dY and x are staged transposed (dY^T [O][Tp],
//                                x'^T [I][Tp] with x'^T[c][t] = x[t][perm c], Tp = tokens rounded up to 64, zero
//                                padding) and the wgmma GEMM of gemm_wgmma.cu writes G in fp32 [O][I] (quantised
//                                column order) to the workspace.
//   vptq_b200_dequant_backward   G = the incoming 16-bit gradient of W [O][I] (original feature order).
// and then, on the caller's stream:
//   1. pre-pass   zero the accumulators; per row of dY / x / G the sums of |v| and |s_f v| (fixed order, so the
//                 bound below is the same on every run); max |C|, |R|, |Col| (order-free atomicMax).
//   2. units      one CTA: the bounds B_cb = sum |s_f G| (>=), B_bias = sum |G|, B_scale = B_bias max|Wq| in fp64
//                 and from them the power-of-two units 2^e >= B / 2^61 of the three fixed-point sums; a non-finite
//                 bound (B_scale included: inf / NaN in a codebook while d weight_scale is wanted) marks the call
//                 non-finite.
//   3. scatter    a thread owns one column and 16 index rows: it decodes the field of every (r, c) like the dequant
//                 kernels do, adds s_f G[o][f] as a 64-bit fixed-point integer into dC[k][e] (red.global.add.u64)
//                 and dR[kr][e] (a per-CTA shared-memory table for small residual codebooks, flushed once), and
//                 rounds each term G Wq and G of its column to its unit as well, summing them in registers and
//                 adding the sums once to d weight_scale[f] / d weight_bias[f].
//   4. finish     integer * 2^e rounded once to the layer's dtype: the int64 goes to fp64 with round-to-odd, so
//                 the fp64 -> 16-bit conversion is the only rounding (NaN everywhere for a non-finite call).
// Integer addition is associative, so the results do not depend on the order in which the GPU adds the terms:
// bit-identical from run to run and under CUDA-graph replay.
#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "kernels.h"

namespace vptq_b200 {

namespace {

constexpr int SC_COLS = 256;                // columns per scatter CTA (one per thread)
constexpr int SC_ROWS = 16;                 // index rows per scatter CTA
constexpr int kResTableBytes = 32 * 1024;   // per-CTA residual-gradient table in shared memory, when it fits
constexpr int kFracBits = 61;               // unit >= bound / 2^61: partial sums stay below 2^62 in magnitude

// The fused route (G never stored): v = 8, one codebook group, no outlier columns, Kr <= 256 -- every Llama shape.
bool fused_eligible(const vptq_linear_desc& d) {
  const bool outl = d.outlier_size > 0 && d.outlier_indices != nullptr;
  return d.vector_len == 8 && d.num_codebooks == 1 && !outl && d.num_res_centroids <= 256;
}

struct WgLayout {
  size_t off_hdr, off_a, off_b, off_c, off_inv, off_acc_c, off_acc_r, off_acc_col, off_acc_s, off_acc_b, off_acc_end;
  size_t off_dyt, off_xt, off_gamma, total;
  int64_t tp, ldg;
  int nrows, np;  // rows of the statistics arrays; rows of x'^T (in_features rounded up to even)
};

WgLayout wg_layout(const vptq_linear_desc& d, int tokens, int op) {
  WgLayout w{};
  const int64_t I = d.in_features, O = d.out_features, v = d.vector_len, G = d.num_codebooks;
  const int64_t Kr = d.num_res_centroids > 0 ? d.num_res_centroids : 0;
  const bool outl = d.outlier_size > 0 && d.outlier_indices != nullptr;
  const int64_t ncol = outl ? int64_t(std::max(d.num_outlier_centroids, 0)) * std::max(d.outlier_vector_len, 1) : 0;
  if (tokens < 1) tokens = 1;
  w.nrows = op == VPTQ_GRAD_OP_DEQUANT_BACKWARD ? d.out_features : tokens;
  w.np = int((I + 1) & ~int64_t(1));
  size_t off = kZeroRegionBytes;  // the zero-at-rest head of the shared workspace stays untouched
  w.off_hdr = off;
  off += 256;
  w.off_acc_c = off;  // accumulators: zeroed by every call (one memset from off_hdr to off_acc_end)
  off += align_up(size_t(G) * d.num_centroids * v * 8, 256);
  w.off_acc_r = off;
  off += align_up(size_t(G) * Kr * v * 8, 256);
  w.off_acc_col = off;
  off += align_up(size_t(ncol) * 8, 256);
  w.off_acc_s = off;
  off += align_up(size_t(I) * 8, 256);
  w.off_acc_b = off;
  off += align_up(size_t(I) * 8, 256);
  w.off_acc_end = off;
  w.off_a = off;  // per-row bound sums, fp64 (no overflow for any finite 16-bit input)
  off += align_up(size_t(w.nrows) * 8, 256);
  w.off_b = off;
  off += align_up(size_t(w.nrows) * 8, 256);
  w.off_c = off;
  off += align_up(size_t(w.nrows) * 8, 256);
  w.off_inv = off;
  if (op == VPTQ_GRAD_OP_DEQUANT_BACKWARD) {
    off += align_up(size_t(I) * 2, 256);
    w.total = align_up(off, 1024);
    return w;
  }
  off = align_up(off, 1024);
  w.tp = int64_t(align_up(size_t(tokens), 64));
  w.ldg = int64_t(align_up(size_t(I), 4));
  w.off_dyt = off;
  off += align_up(size_t(O) * w.tp * 2, 1024);
  w.off_xt = off;
  off += align_up(size_t(w.np) * w.tp * 2, 1024);
  w.off_gamma = off;
  if (op == VPTQ_GRAD_OP_WGRAD_GENERIC || !fused_eligible(d)) off += align_up(size_t(O) * w.ldg * 4, 1024);  // G
  w.total = off;
  return w;
}

__device__ __forceinline__ double block_sum_256(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < 8; ++w) s += red[w];
  __syncthreads();
  return s;
}

// abs_sum[row] = sum_i |p[row][i]|,  sabs_sum[row] = sum_i |scale[i] p[row][i]| (= abs_sum without scale), in fp64
// (finite for every finite 16-bit input).  Every thread adds a fixed strided subset, then a fixed tree: the same
// value on every run.
template <typename T>
__global__ void __launch_bounds__(256) wg_row_stats(const T* __restrict__ p, int64_t stride, int n,
                                                    const T* __restrict__ scale, double* __restrict__ abs_sum,
                                                    double* __restrict__ sabs_sum) {
  __shared__ double red[8];
  const T* row = p + int64_t(blockIdx.x) * stride;
  double a = 0.0, s = 0.0;
  for (int i = threadIdx.x; i < n; i += 256) {
    const double v = fabs(double(DT<T>::to_float(row[i])));
    a += v;
    if (scale) s += v * fabs(double(DT<T>::to_float(scale[i])));
  }
  a = block_sum_256(a, red);
  s = block_sum_256(s, red);
  if (threadIdx.x == 0) {
    abs_sum[blockIdx.x] = a;
    if (sabs_sum) sabs_sum[blockIdx.x] = scale ? s : a;
  }
}

// max that keeps NaN (fmaxf drops it): |NaN| wins over every number
__device__ __forceinline__ float max_nan(float a, float b) { return (b > a || b != b) ? b : a; }

// *out = max(*out, max |p[g][i]|) over groups g < groups, i < n (bit pattern of a non-negative float; a positive NaN
// orders above +inf, so a NaN entry reaches wg_units)
template <typename T>
__global__ void __launch_bounds__(256) wg_absmax(const T* __restrict__ p, int groups, int64_t n, int64_t stride,
                                                 uint32_t* out) {
  float m = 0.f;
  const int64_t total = int64_t(groups) * n;
  for (int64_t i = int64_t(blockIdx.x) * 256 + threadIdx.x; i < total; i += int64_t(gridDim.x) * 256) {
    const int64_t g = i / n;
    m = max_nan(m, fabsf(DT<T>::to_float(p[g * stride + (i - g * n)])));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max_nan(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && __float_as_uint(m) != 0u) atomicMax(out, __float_as_uint(m));
}

__device__ int unit_exponent(double bound) {
  if (!(bound > 0.0)) return 0;  // all terms are zero
  int k;
  frexp(bound, &k);              // bound <= 2^k
  return k - kFracBits;
}

// a == nullptr: every a[i] is 1.  B_cb = sum a b, B_bias = sum a c, B_scale = B_bias max|Wq|, in fp64, fixed order.
__global__ void __launch_bounds__(256) wg_units(const double* __restrict__ a, const double* __restrict__ b,
                                                const double* __restrict__ c, int n, WgHeader* hdr) {
  __shared__ double r1[256], r2[256];
  double s1 = 0.0, s2 = 0.0;
  for (int i = threadIdx.x; i < n; i += 256) {
    const double ai = a ? a[i] : 1.0;
    s1 += ai * b[i];
    s2 += ai * c[i];
  }
  r1[threadIdx.x] = s1, r2[threadIdx.x] = s2;
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if (threadIdx.x < h) r1[threadIdx.x] += r1[threadIdx.x + h], r2[threadIdx.x] += r2[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double bc = r1[0], bb = r2[0];
    const double mc = double(__uint_as_float(hdr->max_c)) + double(__uint_as_float(hdr->max_r));
    const double mo = double(__uint_as_float(hdr->max_col));
    const double mwq = fmax(mc, mo);
    // the maxima are 0 unless d weight_scale is wanted: a non-finite codebook matters only then.  Both are tested,
    // since fmax drops a NaN.
    hdr->nonfinite = !(isfinite(bc) && isfinite(bb) && isfinite(bb * mc) && isfinite(bb * mo));
    hdr->e_cb = unit_exponent(bc);
    hdr->e_bias = unit_exponent(bb);
    hdr->e_scale = unit_exponent(bb * mwq);
  }
}

// dst[c][t] = src[t][perm ? perm[c] : c] for c < n, t < T; zero for T <= t < Tp and for n <= c < n_out
__global__ void __launch_bounds__(256) wg_transpose(const uint16_t* __restrict__ src, int64_t stride, int T, int n,
                                                    int n_out, const uint16_t* __restrict__ perm,
                                                    uint16_t* __restrict__ dst, int64_t tp) {
  __shared__ uint16_t tile[64][66];
  const int c0 = blockIdx.x * 64, t0 = blockIdx.y * 64;
  const int cc = threadIdx.x & 63;
  const int c = c0 + cc;
  const int sc = c < n ? (perm ? int(perm[c]) : c) : 0;
  for (int i = threadIdx.x >> 6; i < 64; i += 4) {
    const int t = t0 + i;
    tile[i][cc] = (t < T && c < n) ? src[int64_t(t) * stride + sc] : uint16_t(0);
  }
  __syncthreads();
  for (int i = threadIdx.x >> 6; i < 64; i += 4) {
    const int co = c0 + i;
    if (co < n_out) dst[int64_t(co) * tp + t0 + cc] = tile[cc][i];
  }
}

__global__ void wg_invert_perm(const uint16_t* __restrict__ perm, uint16_t* __restrict__ inv, int n) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < n) inv[perm[c]] = uint16_t(c);
}

struct ScatterParams {
  const void* gamma;  // fp32 [O][ld] in quantised column order, or (16-bit input) [O][ld] in original order
  int64_t ld;
  const uint16_t* perm;      // quantised column -> original feature, or nullptr
  const uint16_t* inv_perm;  // original feature -> quantised column (16-bit input only), or nullptr
  const void* scale;         // weight_scale [I] or nullptr
  const uint32_t* indices;
  int64_t idx_stride_g, idx_stride_r;
  const void* centroids;
  int64_t cb_stride;
  const void* res_centroids;
  int64_t rcb_stride;
  const uint16_t* outlier_idx;
  const void* outlier_cb;
  unsigned long long *acc_c, *acc_r, *acc_col, *acc_s, *acc_b;  // nullptr: not wanted
  WgHeader* hdr;
  int I, O, Ro, gs, S, vol, K, Kr, ib, rb;
  int res_table;  // entries of the shared-memory dR table (G * Kr * v), 0: dR goes straight to global memory
};

__device__ __forceinline__ unsigned long long fixed(double v, double inv_unit) {
  return static_cast<unsigned long long>(to_fixed(v, inv_unit));
}

template <typename T, int V, bool G16>
__global__ void __launch_bounds__(SC_COLS) wg_scatter(const __grid_constant__ ScatterParams p) {
  extern __shared__ unsigned long long s_res[];
  const WgHeader h = *p.hdr;
  if (h.nonfinite) return;  // the finish kernel writes NaN
  const int tid = threadIdx.x;
  for (int i = tid; i < p.res_table; i += SC_COLS) s_res[i] = 0ull;
  if (p.res_table) __syncthreads();
  const double u_cb = ldexp(1.0, -h.e_cb), u_b = ldexp(1.0, -h.e_bias), u_s = ldexp(1.0, -h.e_scale);
  const int j = blockIdx.x * SC_COLS + tid;  // quantised column (fp32 input) or original feature (16-bit input)
  const int r0 = blockIdx.y * SC_ROWS, r1 = min(p.Ro, r0 + SC_ROWS);
  if (j < p.I) {
    const int c = G16 ? (p.inv_perm ? int(p.inv_perm[j]) : j) : j;
    const int f = G16 ? j : (p.perm ? int(p.perm[c]) : c);
    const int gcol = G16 ? f : c;  // column of G in memory
    const double s = p.scale ? double(DT<T>::to_float(reinterpret_cast<const T*>(p.scale)[f])) : 1.0;
    // every term is rounded to the unit on its own and summed as an integer: the same bits as the fused epilogue
    // of gemm_wgmma.cu, whatever rows each thread covers
    long long sum_s = 0, sum_b = 0;
    bool bad = false;
    const bool want_w = p.acc_s != nullptr;
    if (c < p.S) {  // outlier column: its own codebook with vector length `vol`
      const T* ocb = reinterpret_cast<const T*>(p.outlier_cb);
      const int oend = min(p.O, r1 * V);
      for (int o = r0 * V; o < oend; ++o) {
        const float gm = G16 ? DT<T>::to_float(reinterpret_cast<const T*>(p.gamma)[int64_t(o) * p.ld + gcol])
                             : reinterpret_cast<const float*>(p.gamma)[int64_t(o) * p.ld + gcol];
        const int rol = o / p.vol, eo = o - rol * p.vol;
        const int oi = p.outlier_idx[int64_t(rol) * p.S + c];
        if (gm == 0.f) continue;
        if (!isfinite(gm)) {
          bad = true;
          continue;
        }
        if (p.acc_col) atomicAdd(&p.acc_col[int64_t(oi) * p.vol + eo], fixed(s * double(gm), u_cb));
        if (want_w) sum_s += to_fixed(double(gm) * double(DT<T>::to_float(ocb[int64_t(oi) * p.vol + eo])), u_s);
        sum_b += to_fixed(double(gm), u_b);
      }
    } else {
      const int ci = c - p.S;
      const int g = ci / p.gs, jj = ci - g * p.gs;
      const int b = p.ib + p.rb;
      const uint32_t fmask = b >= 32 ? 0xffffffffu : ((1u << b) - 1u);
      const uint32_t bit = uint32_t(jj) * uint32_t(b);
      const uint32_t w0 = bit >> 5, sh = bit & 31u;
      const uint64_t pol = policy_evict_last();
      unsigned long long* acc_c = p.acc_c ? p.acc_c + int64_t(g) * p.K * V : nullptr;
      unsigned long long* acc_r = p.acc_r ? p.acc_r + int64_t(g) * p.Kr * V : nullptr;
      unsigned long long* tab_r = s_res + int64_t(g) * p.Kr * V;
      for (int r = r0; r < r1; ++r) {
        const uint32_t* row = p.indices + int64_t(g) * p.idx_stride_g + int64_t(r) * p.idx_stride_r;
        const uint32_t lo = ldg_nc_u32(row + w0);
        const uint32_t hi = (sh + b > 32) ? ldg_nc_u32(row + w0 + 1) : 0u;  // never reads past the row
        const uint32_t field = __funnelshift_r(lo, hi, sh) & fmask;
        const uint32_t mi = field & ((1u << p.ib) - 1u), ri = field >> p.ib;
        float w[V];
        if (want_w) {
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
          if (o >= p.O) break;  // padding outputs contribute nothing
          const float gm = G16 ? DT<T>::to_float(reinterpret_cast<const T*>(p.gamma)[int64_t(o) * p.ld + gcol])
                               : reinterpret_cast<const float*>(p.gamma)[int64_t(o) * p.ld + gcol];
          if (gm == 0.f) continue;
          if (!isfinite(gm)) {  // G overflowed fp32 (finite inputs): reported like a non-finite input
            bad = true;
            continue;
          }
          const unsigned long long q = fixed(s * double(gm), u_cb);
          if (acc_c) atomicAdd(&acc_c[size_t(mi) * V + e], q);
          if (acc_r) {
            if (p.res_table) atomicAdd(&tab_r[size_t(ri) * V + e], q);
            else atomicAdd(&acc_r[size_t(ri) * V + e], q);
          }
          if (want_w) sum_s += to_fixed(double(gm) * double(w[e]), u_s);
          sum_b += to_fixed(double(gm), u_b);
        }
      }
    }
    if (p.acc_s && sum_s) atomicAdd(&p.acc_s[f], static_cast<unsigned long long>(sum_s));
    if (p.acc_b && sum_b) atomicAdd(&p.acc_b[f], static_cast<unsigned long long>(sum_b));
    if (bad) atomicExch(&p.hdr->nonfinite, 1);
  }
  if (p.res_table) {
    __syncthreads();
    for (int i = tid; i < p.res_table; i += SC_COLS)
      if (s_res[i]) atomicAdd(&p.acc_r[i], s_res[i]);
  }
}

template <typename T>
__device__ __forceinline__ T from_double(double v);
template <>
__device__ __forceinline__ __half from_double<__half>(double v) { return __double2half(v); }
template <>
__device__ __forceinline__ __nv_bfloat16 from_double<__nv_bfloat16>(double v) { return __double2bfloat16(v); }

// int64 -> fp64 rounded to odd: exact up to 2^53; above, truncated with the dropped bits ORed into the last bit.  With
// 53 >= p + 2 significant bits, rounding that value to the p-bit 16-bit type (p <= 11) rounds the integer itself
// correctly: a single rounding.  (A plain conversion rounds to nearest first and can land on a tie of the 16-bit type.)
__device__ __forceinline__ double ll_to_double_odd(long long v) {
  const unsigned long long m = v < 0 ? 0ull - static_cast<unsigned long long>(v) : static_cast<unsigned long long>(v);
  if (m <= (1ull << 53)) return double(v);
  const int drop = 11 - __clzll(static_cast<long long>(m));   // bits below the 53 kept (m < 2^63)
  const unsigned long long keep = (m >> drop) | ((m & ((1ull << drop) - 1ull)) != 0ull);
  const double r = ldexp(double(keep), drop);                // exact: keep < 2^53
  return v < 0 ? -r : r;
}

// out[row * out_stride + col] = acc[row * row_len + col] * 2^e, rounded once (NaN for a non-finite call)
template <typename T>
__global__ void __launch_bounds__(256) wg_finish(const unsigned long long* __restrict__ acc, int64_t n,
                                                 int64_t row_len, int64_t out_stride, T* __restrict__ out,
                                                 const WgHeader* __restrict__ hdr, int which) {
  const WgHeader h = *hdr;
  const int e = which == 0 ? h.e_cb : (which == 1 ? h.e_bias : h.e_scale);
  for (int64_t i = int64_t(blockIdx.x) * 256 + threadIdx.x; i < n; i += int64_t(gridDim.x) * 256) {
    const int64_t row = i / row_len, col = i - row * row_len;
    const double v = h.nonfinite ? __longlong_as_double(0x7ff8000000000000ll)
                                 : ldexp(ll_to_double_odd(static_cast<long long>(acc[i])), e);
    out[row * out_stride + col] = from_double<T>(v);
  }
}

int check_launch(const char* what) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s launch: %s", what, cudaGetErrorString(e));
    return VPTQ_ERR_CUDA;
  }
  return 0;
}

unsigned grid_for(int64_t n) { return unsigned(std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, 1056))); }

// steps shared by both entry points: max |codebook| (when d weight_scale is wanted), units, then either the scatter
// kernel over G (gamma != nullptr) or `fused` (the GEMM with the weight-gradient epilogue), then finish
template <typename T, typename Fused>
int reduce_launch(const vptq_linear_desc& d, const WgLayout& w, uint8_t* ws, const vptq_linear_grads& g,
                  const void* gamma, int64_t ld, bool g16, const uint16_t* inv_perm, const double* a, Fused&& fused,
                  cudaStream_t stream) {
  WgHeader* hdr = reinterpret_cast<WgHeader*>(ws + w.off_hdr);
  const int v = d.vector_len, G = d.num_codebooks;
  const int K = d.num_centroids, Kr = d.num_res_centroids > 0 ? d.num_res_centroids : 0;
  const bool outl = d.outlier_size > 0 && d.outlier_indices != nullptr;
  const int S = outl ? d.outlier_size : 0, vol = outl ? d.outlier_vector_len : 1;
  const int64_t ncol = outl ? int64_t(d.num_outlier_centroids) * vol : 0;
  if (g.weight_scale) {
    wg_absmax<T><<<grid_for(int64_t(G) * K * v), 256, 0, stream>>>(reinterpret_cast<const T*>(d.centroids), G,
                                                                   int64_t(K) * v, d.centroid_stride, &hdr->max_c);
    if (Kr)
      wg_absmax<T><<<grid_for(int64_t(G) * Kr * v), 256, 0, stream>>>(
          reinterpret_cast<const T*>(d.res_centroids), G, int64_t(Kr) * v, d.res_centroid_stride, &hdr->max_r);
    if (ncol)
      wg_absmax<T><<<grid_for(ncol), 256, 0, stream>>>(reinterpret_cast<const T*>(d.outlier_centroids), 1, ncol, ncol,
                                                       &hdr->max_col);
  }
  wg_units<<<1, 256, 0, stream>>>(a, reinterpret_cast<const double*>(ws + w.off_b),
                                  reinterpret_cast<const double*>(ws + w.off_c), w.nrows, hdr);
  if (int rc = check_launch("weight-gradient pre-pass")) return rc;
  auto at = [&](size_t off) { return reinterpret_cast<unsigned long long*>(ws + off); };
  const int64_t tab = int64_t(G) * Kr * v;
  auto finish = [&](void* out, size_t off, int64_t n, int64_t row_len, int64_t stride, int which) {
    if (out && n > 0)
      wg_finish<T><<<grid_for(n), 256, 0, stream>>>(at(off), n, row_len, stride, reinterpret_cast<T*>(out), hdr, which);
  };
  auto finish_all = [&]() {
    finish(g.centroids, w.off_acc_c, int64_t(G) * K * v, int64_t(K) * v, d.centroid_stride, 0);
    finish(g.res_centroids, w.off_acc_r, tab, int64_t(Kr) * v, d.res_centroid_stride, 0);
    finish(g.outlier_centroids, w.off_acc_col, ncol, ncol, ncol, 0);
    finish(g.weight_scale, w.off_acc_s, d.in_features, d.in_features, d.in_features, 2);
    finish(g.weight_bias, w.off_acc_b, d.in_features, d.in_features, d.in_features, 1);
    return check_launch("weight-gradient finish");
  };
  if (!gamma) {
    WgradEpilogue ep{};
    ep.indices = reinterpret_cast<const uint32_t*>(d.indices), ep.idx_stride_r = d.index_stride_row;
    ep.centroids = d.centroids, ep.res_centroids = d.res_centroids;
    ep.scale_q = (d.weight_scale_q && d.weight_scale) ? d.weight_scale_q : nullptr;
    ep.scale = d.weight_scale, ep.perm = d.perm;
    ep.acc_c = g.centroids ? at(w.off_acc_c) : nullptr;
    ep.acc_r = g.res_centroids ? at(w.off_acc_r) : nullptr;
    ep.acc_s = g.weight_scale ? at(w.off_acc_s) : nullptr;
    ep.acc_b = g.weight_bias ? at(w.off_acc_b) : nullptr;
    ep.hdr = hdr;
    ep.I = d.in_features, ep.ib = ilog2(K), ep.rb = Kr ? ilog2(Kr) : 0;
    ep.res_table = g.res_centroids ? int(tab) : 0;
    if (int rc = fused(ep)) return rc;
    return finish_all();
  }

  ScatterParams p{};
  p.gamma = gamma, p.ld = ld, p.perm = d.perm, p.inv_perm = inv_perm, p.scale = d.weight_scale;
  p.indices = reinterpret_cast<const uint32_t*>(d.indices);
  p.idx_stride_g = d.index_stride_codebook, p.idx_stride_r = d.index_stride_row;
  p.centroids = d.centroids, p.cb_stride = d.centroid_stride;
  p.res_centroids = d.res_centroids, p.rcb_stride = d.res_centroid_stride;
  p.outlier_idx = outl ? d.outlier_indices : nullptr;
  p.outlier_cb = outl ? d.outlier_centroids : nullptr;
  unsigned long long* acc = nullptr;
  p.acc_c = g.centroids ? at(w.off_acc_c) : acc;
  p.acc_r = g.res_centroids ? at(w.off_acc_r) : acc;
  p.acc_col = g.outlier_centroids ? at(w.off_acc_col) : acc;
  p.acc_s = g.weight_scale ? at(w.off_acc_s) : acc;
  p.acc_b = g.weight_bias ? at(w.off_acc_b) : acc;
  p.hdr = hdr;
  p.I = d.in_features, p.O = d.out_features, p.Ro = (d.out_features + v - 1) / v, p.gs = d.group_size;
  p.S = S, p.vol = vol, p.K = K, p.Kr = Kr;
  p.ib = ilog2(K), p.rb = Kr ? ilog2(Kr) : 0;
  p.res_table = (g.res_centroids && tab * 8 <= kResTableBytes) ? int(tab) : 0;
  const size_t smem = size_t(p.res_table) * 8;
  dim3 grid(unsigned((d.in_features + SC_COLS - 1) / SC_COLS), unsigned((p.Ro + SC_ROWS - 1) / SC_ROWS));
  switch (v) {
#define VPTQ_CASE(VV)                                                                       \
  case VV:                                                                                  \
    if (g16) wg_scatter<T, VV, true><<<grid, SC_COLS, smem, stream>>>(p);                   \
    else wg_scatter<T, VV, false><<<grid, SC_COLS, smem, stream>>>(p);                      \
    break;
    VPTQ_CASE(2) VPTQ_CASE(4) VPTQ_CASE(6) VPTQ_CASE(8) VPTQ_CASE(10) VPTQ_CASE(12) VPTQ_CASE(16)
#undef VPTQ_CASE
    default: set_error("weight gradients: vector_len %d not supported", v); return VPTQ_ERR_UNSUPPORTED;
  }
  if (int rc = check_launch("weight-gradient scatter")) return rc;
  return finish_all();
}

bool wants_any(const vptq_linear_grads& g) {
  return g.centroids || g.res_centroids || g.outlier_centroids || g.weight_scale || g.weight_bias;
}

template <typename T>
int wgrad_impl(const vptq_linear_desc& d, const void* x, int64_t x_stride, const void* dy, int64_t dy_stride,
               int tokens, const vptq_linear_grads& g, uint8_t* ws, const WgLayout& w, bool generic,
               cudaStream_t stream) {
  const int I = d.in_features, O = d.out_features;
  cudaError_t e = cudaMemsetAsync(ws + w.off_hdr, 0, w.off_acc_end - w.off_hdr, stream);
  if (e != cudaSuccess) {
    set_error("weight gradients: cudaMemsetAsync: %s", cudaGetErrorString(e));
    return VPTQ_ERR_CUDA;
  }
  double* a = reinterpret_cast<double*>(ws + w.off_a);
  double* b = reinterpret_cast<double*>(ws + w.off_b);
  double* c = reinterpret_cast<double*>(ws + w.off_c);
  wg_row_stats<T><<<tokens, 256, 0, stream>>>(reinterpret_cast<const T*>(dy), dy_stride, O, nullptr, a, nullptr);
  wg_row_stats<T><<<tokens, 256, 0, stream>>>(reinterpret_cast<const T*>(x), x_stride, I,
                                              reinterpret_cast<const T*>(d.weight_scale), c, b);
  uint16_t* dyt = reinterpret_cast<uint16_t*>(ws + w.off_dyt);
  uint16_t* xt = reinterpret_cast<uint16_t*>(ws + w.off_xt);
  wg_transpose<<<dim3(unsigned((O + 63) / 64), unsigned(w.tp / 64)), 256, 0, stream>>>(
      reinterpret_cast<const uint16_t*>(dy), dy_stride, tokens, O, O, nullptr, dyt, w.tp);
  wg_transpose<<<dim3(unsigned((w.np + 63) / 64), unsigned(w.tp / 64)), 256, 0, stream>>>(
      reinterpret_cast<const uint16_t*>(x), x_stride, tokens, I, w.np, d.perm, xt, w.tp);
  if (int rc = check_launch("weight-gradient staging")) return rc;
  const int is_bf16 = d.dtype == VPTQ_BF16;
  auto fused = [&](const WgradEpilogue& ep) { return wgrad_fused_launch(is_bf16, dyt, xt, O, w.np, int(w.tp), ep, stream); };
  if (!generic) return reduce_launch<T>(d, w, ws, g, nullptr, 0, false, nullptr, a, fused, stream);
  float* gamma = reinterpret_cast<float*>(ws + w.off_gamma);
  if (int rc = wgrad_gamma_launch(is_bf16, dyt, xt, O, w.np, int(w.tp), gamma, w.ldg, stream)) return rc;
  return reduce_launch<T>(d, w, ws, g, gamma, w.ldg, false, nullptr, a, fused, stream);
}

template <typename T>
int dequant_backward_impl(const vptq_linear_desc& d, const void* dw, int64_t dw_stride, const vptq_linear_grads& g,
                          uint8_t* ws, const WgLayout& w, cudaStream_t stream) {
  cudaError_t e = cudaMemsetAsync(ws + w.off_hdr, 0, w.off_acc_end - w.off_hdr, stream);
  if (e != cudaSuccess) {
    set_error("weight gradients: cudaMemsetAsync: %s", cudaGetErrorString(e));
    return VPTQ_ERR_CUDA;
  }
  wg_row_stats<T><<<d.out_features, 256, 0, stream>>>(reinterpret_cast<const T*>(dw), dw_stride, d.in_features,
                                                      reinterpret_cast<const T*>(d.weight_scale),
                                                      reinterpret_cast<double*>(ws + w.off_c),
                                                      reinterpret_cast<double*>(ws + w.off_b));
  uint16_t* inv = nullptr;
  if (d.perm) {
    inv = reinterpret_cast<uint16_t*>(ws + w.off_inv);
    wg_invert_perm<<<(d.in_features + 255) / 256, 256, 0, stream>>>(d.perm, inv, d.in_features);
  }
  auto none = [](const WgradEpilogue&) { return 0; };
  return reduce_launch<T>(d, w, ws, g, dw, dw_stride, true, inv, nullptr, none, stream);
}

}  // namespace

size_t wgrad_workspace_bytes(const vptq_linear_desc& d, int tokens, int op) { return wg_layout(d, tokens, op).total; }

int wgrad_launch(const vptq_linear_desc& d, const void* x, int64_t x_stride, const void* dy, int64_t dy_stride,
                 int tokens, const vptq_linear_grads& g, void* workspace, size_t workspace_bytes, uint32_t flags,
                 cudaStream_t stream) {
  const bool generic = (flags & VPTQ_GRAD_FLAG_GENERIC) || !fused_eligible(d);
  const WgLayout w = wg_layout(d, tokens, generic ? VPTQ_GRAD_OP_WGRAD_GENERIC : VPTQ_GRAD_OP_WGRAD);
  if (!workspace || workspace_bytes < w.total) {
    set_error("quant_gemm_wgrad: workspace %zu bytes < required %zu", workspace_bytes, w.total);
    return VPTQ_ERR_WORKSPACE;
  }
  if (!wants_any(g)) return 0;
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  return d.dtype == VPTQ_BF16 ? wgrad_impl<__nv_bfloat16>(d, x, x_stride, dy, dy_stride, tokens, g, ws, w, generic, stream)
                              : wgrad_impl<__half>(d, x, x_stride, dy, dy_stride, tokens, g, ws, w, generic, stream);
}

int dequant_backward_launch(const vptq_linear_desc& d, const void* dw, int64_t dw_stride, const vptq_linear_grads& g,
                            void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  const WgLayout w = wg_layout(d, 1, VPTQ_GRAD_OP_DEQUANT_BACKWARD);
  if (!workspace || workspace_bytes < w.total) {
    set_error("dequant_backward: workspace %zu bytes < required %zu", workspace_bytes, w.total);
    return VPTQ_ERR_WORKSPACE;
  }
  if (!wants_any(g)) return 0;
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  return d.dtype == VPTQ_BF16 ? dequant_backward_impl<__nv_bfloat16>(d, dw, dw_stride, g, ws, w, stream)
                              : dequant_backward_impl<__half>(d, dw, dw_stride, g, ws, w, stream);
}

}  // namespace vptq_b200
