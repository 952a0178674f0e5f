// Gather-tier microbenchmark for the VPTQ GEMV design (SURVEY.md 7.4 H1): how many random
// 16-byte codebook gathers per second does each tier of an H100 deliver, next to plain HBM streaming?
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o gather_microbench tools/gather_microbench.cu
// Prints one JSON object per experiment.
#include <cuda_runtime.h>
#include <cooperative_groups.h>
#include <cstdint>
#include <cstdio>
#include <vector>

namespace cg = cooperative_groups;
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); return 1; } } while (0)

__device__ __forceinline__ uint32_t hash32(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16; return x;
}

// ---- 1. HBM stream ------------------------------------------------------------------------
__global__ void k_stream(const uint4* __restrict__ src, size_t n, uint32_t* sink) {
  uint32_t acc = 0;
  for (size_t i = blockIdx.x * size_t(blockDim.x) + threadIdx.x; i < n; i += size_t(gridDim.x) * blockDim.x) {
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(src + i));
    acc ^= v.x ^ v.y ^ v.z ^ v.w;
  }
  if (acc == 0x12345678u) *sink = acc;
}

// ---- 2. random 16-B gathers from global (L2 / L1) -------------------------------------------
template <int U>
__global__ void k_gather_global(const uint4* __restrict__ table, uint32_t mask, int iters, uint32_t* sink) {
  uint32_t acc = 0;
  uint32_t seed = (blockIdx.x * blockDim.x + threadIdx.x) * 2654435761u;
  for (int it = 0; it < iters; ++it) {
    uint4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const uint32_t idx = hash32(seed + it * U + u) & mask;
      v[u] = __ldg(table + idx);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) acc ^= v[u].x ^ v[u].y ^ v[u].z ^ v[u].w;
  }
  if (acc == 0x12345678u) *sink = acc;
}

// ---- 3. random 16-B gathers from shared memory ------------------------------------------------
// mode 0: random entries (bank-group conflicts).  mode 1: entry*8 + (lane&7): conflict-free replicated layout.
template <int U>
__global__ void k_gather_smem(const uint4* __restrict__ table, int entries, int mode, int iters, uint32_t* sink) {
  extern __shared__ uint4 st[];
  for (int i = threadIdx.x; i < entries; i += blockDim.x) st[i] = table[i & 0xffff];
  __syncthreads();
  uint32_t acc = 0;
  uint32_t seed = (blockIdx.x * blockDim.x + threadIdx.x) * 2654435761u;
  const uint32_t lane7 = threadIdx.x & 7;
  const uint32_t mask = mode ? (entries / 8 - 1) : (entries - 1);
  for (int it = 0; it < iters; ++it) {
    uint4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      uint32_t idx = hash32(seed + it * U + u) & mask;
      if (mode) idx = idx * 8 + lane7;
      v[u] = st[idx];
    }
#pragma unroll
    for (int u = 0; u < U; ++u) acc ^= v[u].x ^ v[u].y ^ v[u].z ^ v[u].w;
  }
  if (acc == 0x12345678u) *sink = acc;
}

// ---- 4. random 16-B gathers from distributed shared memory (cluster of CS CTAs) ------------------
template <int U>
__global__ void k_gather_dsmem(const uint4* __restrict__ table, int entries_per_cta, int iters, uint32_t* sink) {
  extern __shared__ uint4 st[];
  cg::cluster_group cluster = cg::this_cluster();
  const unsigned cs = cluster.num_blocks();
  for (int i = threadIdx.x; i < entries_per_cta; i += blockDim.x) st[i] = table[i & 0xffff];
  cluster.sync();
  uint32_t acc = 0;
  uint32_t seed = (blockIdx.x * blockDim.x + threadIdx.x) * 2654435761u;
  const uint32_t emask = entries_per_cta - 1;
  for (int it = 0; it < iters; ++it) {
    uint4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const uint32_t h = hash32(seed + it * U + u);
      const uint4* remote = cluster.map_shared_rank(st, (h >> 20) % cs);
      v[u] = remote[h & emask];
    }
#pragma unroll
    for (int u = 0; u < U; ++u) acc ^= v[u].x ^ v[u].y ^ v[u].z ^ v[u].w;
  }
  if (acc == 0x12345678u) *sink = acc;
  cluster.sync();
}

template <typename F>
float time_ms(F&& launch, int reps = 5) {
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  launch();
  cudaDeviceSynchronize();
  float best = 1e30f;
  for (int r = 0; r < reps; ++r) {
    cudaEventRecord(a); launch(); cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    if (ms < best) best = ms;
  }
  return best;
}

int main() {
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
  const int sms = prop.multiProcessorCount;
  int clk_khz = 0; cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
  printf("{\"device\": \"%s\", \"sms\": %d, \"l2_mb\": %.1f, \"clock_mhz_max\": %d}\n", prop.name, sms, prop.l2CacheSize / 1048576.0, clk_khz / 1000);
  uint32_t* sink; CK(cudaMalloc(&sink, 4));

  { // HBM stream over 4 GiB
    const size_t bytes = size_t(4) << 30; uint4* src; CK(cudaMalloc(&src, bytes)); CK(cudaMemset(src, 1, bytes));
    for (int bpsm : {8, 16, 32}) {
      float ms = time_ms([&] { k_stream<<<sms * bpsm, 256>>>(src, bytes / 16, sink); });
      printf("{\"exp\": \"hbm_stream_ldg128\", \"blocks_per_sm\": %d, \"GBps\": %.1f}\n", bpsm, bytes / ms / 1e6);
    }
    CK(cudaFree(src));
  }
  uint4* table; CK(cudaMalloc(&table, size_t(64) << 20)); CK(cudaMemset(table, 3, size_t(64) << 20));
  const int iters = 256; constexpr int U = 4;
  for (size_t tbytes : {size_t(4) << 10, size_t(64) << 10, size_t(128) << 10, size_t(1) << 20, size_t(2) << 20, size_t(32) << 20}) {
    for (int threads : {256, 512, 1024}) {
      const int blocks = sms * (2048 / threads);
      const uint32_t mask = uint32_t(tbytes / 16 - 1);
      float ms = time_ms([&] { k_gather_global<U><<<blocks, threads>>>(table, mask, iters, sink); });
      const double n = double(blocks) * threads * iters * U;
      printf("{\"exp\": \"gather16_global\", \"table_kb\": %zu, \"threads\": %d, \"Ggathers_per_s\": %.1f, \"per_sm_per_ns\": %.3f, \"eff_TBps_16B\": %.2f}\n",
             tbytes >> 10, threads, n / ms / 1e6, n / ms / 1e6 / sms, n * 16 / ms / 1e9);
    }
  }
  for (int mode : {0, 1}) {
    for (size_t tbytes : {size_t(32) << 10, size_t(128) << 10}) {
      const int entries = int(tbytes / 16);
      auto kern = k_gather_smem<U>;
      CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(tbytes)));
      for (int threads : {256, 512, 1024}) {
        const int blocks = sms;
        float ms = time_ms([&] { kern<<<blocks, threads, tbytes>>>(table, entries, mode, iters * 4, sink); });
        const double n = double(blocks) * threads * iters * 4 * U;
        printf("{\"exp\": \"gather16_smem\", \"mode\": \"%s\", \"table_kb\": %zu, \"threads\": %d, \"Ggathers_per_s\": %.1f, \"per_sm_per_ns\": %.3f, \"eff_TBps_16B\": %.2f}\n",
               mode ? "replicated_conflict_free" : "random", tbytes >> 10, threads, n / ms / 1e6, n / ms / 1e6 / sms, n * 16 / ms / 1e9);
      }
    }
  }
  for (int cs : {2, 4, 8}) {
    const size_t tbytes = size_t(128) << 10;
    auto kern = k_gather_dsmem<U>;
    CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(tbytes)));
    for (int threads : {256, 1024}) {
      cudaLaunchConfig_t cfg{}; cfg.gridDim = dim3((sms / cs) * cs); cfg.blockDim = dim3(threads); cfg.dynamicSmemBytes = tbytes;
      cudaLaunchAttribute at[1]; at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim = {unsigned(cs), 1, 1};
      cfg.attrs = at; cfg.numAttrs = 1;
      const int ent = int(tbytes / 16), it2 = iters;
      float ms = time_ms([&] { cudaLaunchKernelEx(&cfg, kern, (const uint4*)table, ent, it2, sink); });
      CK(cudaGetLastError());
      const double n = double(cfg.gridDim.x) * threads * iters * U;
      printf("{\"exp\": \"gather16_dsmem\", \"cluster\": %d, \"threads\": %d, \"Ggathers_per_s\": %.1f, \"per_sm_per_ns\": %.3f, \"eff_TBps_16B\": %.2f}\n",
             cs, threads, n / ms / 1e6, n / ms / 1e6 / cfg.gridDim.x, n * 16 / ms / 1e9);
    }
  }
  return 0;
}
