// ptx.cuh -- inline-PTX wrappers shared by the sm_90a kernels: L2 cache policies, hinted
// global loads, and the 1-D TMA bulk store shared -> global (cp.async.bulk -> SASS UBLKCP).
// (tests/emu/transform.py swaps this header for tests/emu/cuemu_ptx.h.)
#pragma once
#include "common.cuh"

// ---- PTX wrappers: L2 cache policies, hinted loads, TMA bulk store -----------------
// (round 1's mbarrier + cp.async.bulk global->shared ring is gone with the kernel that used it:
// on this path a staged stream measured no faster than coalesced register loads and cost L1)
static __device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
static __device__ __forceinline__ uint64_t policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
static __device__ __forceinline__ uint64_t policy_evict_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
static __device__ __forceinline__ double ldg_f64_hint(const double* p, uint64_t policy) {
    double v;
    asm("ld.global.nc.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(policy));
    return v;
}

static __device__ __forceinline__ uint32_t ldg_stream_u32(const uint32_t* p, uint64_t policy) {
    uint32_t v;
    asm("ld.global.nc.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;"
        : "=r"(v) : "l"(p), "l"(policy));
    return v;
}
static __device__ __forceinline__ double ldg_stream_f64(const double* p, uint64_t policy) {
    double v;
    asm("ld.global.nc.L1::no_allocate.L2::cache_hint.f64 %0, [%1], %2;"
        : "=d"(v) : "l"(p), "l"(policy));
    return v;
}

// ---- GPU-scope acquire / release on a u32 flag (the triangular solve's per-row ready flags):
// the loads that follow an acquire see every store that preceded the matching release
static __device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
static __device__ __forceinline__ void st_release_u32(uint32_t* p, uint32_t v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// ---- TMA bulk store shared -> global (bulk async-group completion); the destination may be a
// peer GPU's memory or an NVSwitch multicast address
static __device__ __forceinline__ void bulk_s2g(void* dst, const void* src_smem, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst),
                 "r"(smem_u32(src_smem)), "r"(bytes)
                 : "memory");
}
static __device__ __forceinline__ void bulk_commit_group() {
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
// the shared-memory SOURCE of every committed group has been read (it may be overwritten)
static __device__ __forceinline__ void bulk_wait_group_read0() {
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
// every committed group has completed (its writes are performed)
static __device__ __forceinline__ void bulk_wait_group0() {
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}
