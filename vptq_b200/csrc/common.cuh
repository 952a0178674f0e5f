// Shared device helpers for the sm_100a VPTQ kernels: PTX wrappers (mbarrier, 1-D TMA bulk copy,
// cache-policy loads, programmatic dependent launch) and the 16-bit dtype traits.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace vptq_b200 {

// ------------------------------------------------------------------------------------------
// dtype traits: every kernel is instantiated for __half and __nv_bfloat16
// ------------------------------------------------------------------------------------------
template <typename T>
struct DT;

template <>
struct DT<__half> {
  // two packed elements (one 32-bit word, low element first) -> float2
  static __device__ __forceinline__ float2 unpack2(uint32_t w) {
    return __half22float2(*reinterpret_cast<const __half2*>(&w));
  }
  // packed add in 16-bit arithmetic (the reference's ADD2, csrc/util/cuda_utils.cuh:140-193)
  static __device__ __forceinline__ uint32_t add2(uint32_t a, uint32_t b) {
    __half2 r = __hadd2(*reinterpret_cast<const __half2*>(&a), *reinterpret_cast<const __half2*>(&b));
    return *reinterpret_cast<uint32_t*>(&r);
  }
  static __device__ __forceinline__ float to_float(__half v) { return __half2float(v); }
  static __device__ __forceinline__ __half from_float(float v) { return __float2half_rn(v); }
  static __device__ __forceinline__ uint32_t pack2(float lo, float hi) {
    __half2 r = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&r);
  }
};

template <>
struct DT<__nv_bfloat16> {
  static __device__ __forceinline__ float2 unpack2(uint32_t w) {
    // bf16 -> fp32 is a 16-bit left shift: two ALU ops, no conversion pipe
    return make_float2(__uint_as_float(w << 16), __uint_as_float(w & 0xffff0000u));
  }
  static __device__ __forceinline__ uint32_t add2(uint32_t a, uint32_t b) {
    __nv_bfloat162 r = __hadd2(*reinterpret_cast<const __nv_bfloat162*>(&a),
                               *reinterpret_cast<const __nv_bfloat162*>(&b));
    return *reinterpret_cast<uint32_t*>(&r);
  }
  static __device__ __forceinline__ float to_float(__nv_bfloat16 v) { return __bfloat162float(v); }
  static __device__ __forceinline__ __nv_bfloat16 from_float(float v) { return __float2bfloat16_rn(v); }
  static __device__ __forceinline__ uint32_t pack2(float lo, float hi) {
    __nv_bfloat162 r = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&r);
  }
};

// ------------------------------------------------------------------------------------------
// shared-memory addressing, mbarrier, TMA 1-D bulk copy (cp.async.bulk -> SASS UBLKCP)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
// make barrier inits visible to the async (TMA) proxy
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// L2 eviction policies: the packed index stream is read exactly once per token (evict_first) so
// that it does not push the codebooks (evict_last) out of the 126 MB L2.
__device__ __forceinline__ uint64_t policy_evict_first() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ uint64_t policy_evict_last() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}

// global -> shared bulk copy; bytes % 16 == 0, both addresses 16-B aligned; completion is
// signalled on `bar` as `bytes` of transaction count.
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes,
                                             uint64_t* bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint "
      "[%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}

// asynchronous prefetch of [p, p + bytes) into L2 (bytes % 16 == 0, p 16-byte aligned)
__device__ __forceinline__ void l2_prefetch_bulk(const void* p, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}

// ------------------------------------------------------------------------------------------
// global loads
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 ldg_nc_v4(const void* p, uint64_t policy) {
  uint4 r;
  asm volatile("ld.global.nc.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p), "l"(policy));
  return r;
}
__device__ __forceinline__ uint2 ldg_nc_v2(const void* p) {
  uint2 r;
  asm volatile("ld.global.nc.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
  return r;
}
__device__ __forceinline__ uint32_t ldg_nc_u32(const void* p) {
  uint32_t r;
  asm volatile("ld.global.nc.u32 %0, [%1];" : "=r"(r) : "l"(p));
  return r;
}
// system-scope flag traffic between GPUs (tensor-parallel epoch flags in peer memory)
__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const uint32_t* p) {
  uint32_t r;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(r) : "l"(p) : "memory");
  return r;
}
__device__ __forceinline__ void st_release_sys_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_volatile_u32(const uint32_t* p) {
  uint32_t r;
  asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(r) : "l"(p) : "memory");
  return r;
}
// L2-coherent load (bypasses L1): used to read partial sums written by other SMs
__device__ __forceinline__ float ldg_cg_f32(const float* p) {
  float r;
  asm volatile("ld.global.cg.f32 %0, [%1];" : "=f"(r) : "l"(p));
  return r;
}

// 16-byte asynchronous global -> shared copy (LDGSTS): the gather does not occupy registers while it
// is in flight, so the number of outstanding gathers per warp is bounded by shared memory only.
__device__ __forceinline__ void cp_async_16(uint32_t dst_smem, const void* src, uint64_t policy) {
  asm volatile("cp.async.ca.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(dst_smem), "l"(src), "l"(policy)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ uint4 lds_v4(uint32_t saddr) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(saddr));
  return r;
}
__device__ __forceinline__ void sts_v4(uint32_t saddr, uint4 v) {
  asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(saddr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// ------------------------------------------------------------------------------------------
// programmatic dependent launch (PDL): no-ops unless the launch carries the attribute
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_wait_prior_grid() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

// ------------------------------------------------------------------------------------------
// thread-block cluster: rank, distributed-shared-memory stores, cluster barrier
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// shared::cta address -> the same offset in CTA `rank` of this cluster (shared::cluster window)
__device__ __forceinline__ uint32_t mapa_shared(uint32_t saddr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(saddr), "r"(rank));
  return r;
}
__device__ __forceinline__ void st_cluster_f32(uint32_t addr, float v) {
  asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}
// remote shared-memory store whose completion is counted (in bytes) on an mbarrier of the SAME remote
// CTA: the consumer just waits for the expected byte count -- no fence, no closing cluster barrier.
__device__ __forceinline__ void st_async_f32(uint32_t remote_addr, float v, uint32_t remote_bar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(remote_addr),
               "r"(__float_as_uint(v)), "r"(remote_bar)
               : "memory");
}
__device__ __forceinline__ void cluster_arrive_relaxed() {
  asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");
}
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }

// v in units of 2^e (inv_unit = 2^-e), rounded to the nearest integer: one term of a 64-bit fixed-point sum
// (weight gradients, wgrad.cu).  Integer addition is associative: the sum does not depend on the order.
__device__ __forceinline__ long long to_fixed(double v, double inv_unit) { return __double2ll_rn(v * inv_unit); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Load one codebook entry of V 16-bit elements (2V bytes) as V/2 packed words with the widest
// vector access its natural alignment allows (entry address = 16B-aligned base + i * 2V).
template <int V>
__device__ __forceinline__ void lds_entry(uint32_t (&w)[V / 2], uint32_t saddr) {
  if constexpr (V % 8 == 0) {
#pragma unroll
    for (int i = 0; i < V / 8; ++i)
      asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];"
                   : "=r"(w[4 * i]), "=r"(w[4 * i + 1]), "=r"(w[4 * i + 2]), "=r"(w[4 * i + 3])
                   : "r"(saddr + 16 * i));
  } else if constexpr (V % 4 == 0) {
#pragma unroll
    for (int i = 0; i < V / 4; ++i)
      asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(w[2 * i]), "=r"(w[2 * i + 1]) : "r"(saddr + 8 * i));
  } else {
#pragma unroll
    for (int i = 0; i < V / 2; ++i) asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w[i]) : "r"(saddr + 4 * i));
  }
}

template <int V>
__device__ __forceinline__ void ldg_entry(uint32_t (&w)[V / 2], const void* p, uint64_t policy) {
  if constexpr (V % 8 == 0) {
#pragma unroll
    for (int i = 0; i < V / 8; ++i) {
      uint4 r = ldg_nc_v4(reinterpret_cast<const uint8_t*>(p) + 16 * i, policy);
      w[4 * i] = r.x, w[4 * i + 1] = r.y, w[4 * i + 2] = r.z, w[4 * i + 3] = r.w;
    }
  } else if constexpr (V % 4 == 0) {
#pragma unroll
    for (int i = 0; i < V / 4; ++i) {
      uint2 r = ldg_nc_v2(reinterpret_cast<const uint8_t*>(p) + 8 * i);
      w[2 * i] = r.x, w[2 * i + 1] = r.y;
    }
  } else {
#pragma unroll
    for (int i = 0; i < V / 2; ++i) w[i] = ldg_nc_u32(reinterpret_cast<const uint8_t*>(p) + 4 * i);
  }
}

}  // namespace vptq_b200
