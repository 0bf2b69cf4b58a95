// spmv_lab.cu -- design-space probe for the SpMV gather pipe on H100 (NOT product code).
//
// "Ceiling" kernels: the SpMV's memory behaviour with the row logic removed -- stream the
// (index, value) arrays of a REAL matrix in warp tiles, gather x[col], multiply-add into one
// accumulator per lane.  Any SpMV that gathers x through L1/L2 does at least this work, so the
// best variant here is the ceiling the product kernel is measured against
// (bench.py roofline.gather_ceiling uses the library's copy of the winner, csrc/diag.cu).
//
// Variants (template parameters, selected at run time through lab_ceiling):
//   EPL   non-zeros per lane per tile (tile = 32*EPL)
//   MODE  0 direct: coalesced ld.global.nc.L1::no_allocate of index and value (no smem)
//         1 TMA ring, 1 stage (what the round-1 product kernel does)
//         2 direct with the NEXT tile's indices prefetched into registers
//         3 TMA ring, 2 stages
//   GOP   gather instruction: 0 ld.global.nc + L2 evict_last, 1 + L1::no_allocate,
//         2 plain ld.global.nc, 3 L1::evict_last + L2 evict_last
//   MINB  resident CTAs per SM (8 warps each) -- sets the register budget
// cmode: 0 real columns, 1 columns & mask (shrinks the x range), 2 sequential columns.
//
// Build: make -C tools lab   (nvcc -shared, sm_90a)
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>

namespace {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ uint64_t policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t policy_evict_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint32_t ldg_stream_u32(const uint32_t* p, uint64_t policy) {
    uint32_t v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;"
                 : "=r"(v) : "l"(p), "l"(policy));
    return v;
}
__device__ __forceinline__ double ldg_stream_f64(const double* p, uint64_t policy) {
    double v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.f64 %0, [%1], %2;"
                 : "=d"(v) : "l"(p), "l"(policy));
    return v;
}
template <int GOP>
__device__ __forceinline__ double gather(const double* p, uint64_t pol) {
    double v;
    if (GOP == 0)
        asm volatile("ld.global.nc.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(pol));
    else if (GOP == 1)
        asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.f64 %0, [%1], %2;"
                     : "=d"(v) : "l"(p), "l"(pol));
    else if (GOP == 2)
        asm volatile("ld.global.nc.f64 %0, [%1];" : "=d"(v) : "l"(p));
    else
        asm volatile("ld.global.nc.L1::evict_last.L2::cache_hint.f64 %0, [%1], %2;"
                     : "=d"(v) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n.reg .pred p;\nLAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra LAB_DONE;\nbra LAB_WAIT;\nLAB_DONE:\n}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint "
        "[%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy) : "memory");
}

template <int EPL, int MODE, int GOP, int MINB>
__global__ void __launch_bounds__(256, MINB)
    ceil_kernel(const uint32_t* __restrict__ idx, const double* __restrict__ val,
                const double* __restrict__ x, double* __restrict__ out, uint64_t n_tiles,
                int cmode, uint32_t mask, uint32_t ncols) {
    constexpr int WT = EPL * 32;
    constexpr int NW = 8;
    constexpr bool TMA = MODE == 1 || MODE == 3;
    constexpr int NST = MODE == 3 ? 2 : 1;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ __align__(8) uint64_t bars[NW][2];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t gw = (uint64_t)blockIdx.x * NW + warp, GW = (uint64_t)gridDim.x * NW;
    const uint64_t pol_s = policy_evict_first(), pol_x = policy_evict_last();
    double acc = 0.0;
    auto col = [&](uint32_t c, uint64_t k) -> uint32_t {
        if (cmode == 1) return c & mask;
        if (cmode == 2) return (uint32_t)(k % ncols);
        return c;
    };
    if (!TMA) {
        uint32_t cn[EPL];
        if (MODE == 2 && gw < n_tiles) {
#pragma unroll
            for (int i = 0; i < EPL; ++i) cn[i] = ldg_stream_u32(idx + gw * WT + lane + 32 * i, pol_s);
        }
        for (uint64_t t = gw; t < n_tiles; t += GW) {
            const uint64_t k0 = t * WT;
            uint32_t c[EPL];
            double v[EPL], xv[EPL];
            if (MODE == 2) {
#pragma unroll
                for (int i = 0; i < EPL; ++i) c[i] = cn[i];
            } else {
#pragma unroll
                for (int i = 0; i < EPL; ++i) c[i] = ldg_stream_u32(idx + k0 + lane + 32 * i, pol_s);
            }
#pragma unroll
            for (int i = 0; i < EPL; ++i) xv[i] = gather<GOP>(x + col(c[i], k0 + lane + 32 * i), pol_x);
#pragma unroll
            for (int i = 0; i < EPL; ++i) v[i] = ldg_stream_f64(val + k0 + lane + 32 * i, pol_s);
            if (MODE == 2 && t + GW < n_tiles) {
#pragma unroll
                for (int i = 0; i < EPL; ++i)
                    cn[i] = ldg_stream_u32(idx + (t + GW) * WT + lane + 32 * i, pol_s);
            }
#pragma unroll
            for (int i = 0; i < EPL; ++i) acc = __dadd_rn(acc, __dmul_rn(v[i], xv[i]));
        }
    } else {
        unsigned char* wsm = smem_raw + (size_t)warp * NST * WT * 12;
        if (lane == 0) {
            for (int s = 0; s < NST; ++s) mbar_init(&bars[warp][s], 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncwarp();
        auto issue = [&](uint64_t t, int s) {
            unsigned char* st = wsm + (size_t)s * WT * 12;
            mbar_expect_tx(&bars[warp][s], WT * 12);
            bulk_g2s(st, val + t * WT, WT * 8, &bars[warp][s], pol_s);
            bulk_g2s(st + WT * 8, idx + t * WT, WT * 4, &bars[warp][s], pol_s);
        };
        if (lane == 0)
            for (int s = 0; s < NST; ++s)
                if (gw + s * GW < n_tiles) issue(gw + s * GW, s);
        uint32_t phases = 0;
        int s = 0;
        for (uint64_t t = gw; t < n_tiles; t += GW) {
            const uint64_t k0 = t * WT;
            const double* sval = (const double*)(wsm + (size_t)s * WT * 12);
            const uint32_t* sidx = (const uint32_t*)(wsm + (size_t)s * WT * 12 + WT * 8);
            mbar_wait(&bars[warp][s], (phases >> s) & 1u);
            phases ^= 1u << s;
            uint32_t c[EPL];
            double xv[EPL];
#pragma unroll
            for (int i = 0; i < EPL; ++i) c[i] = sidx[lane + 32 * i];
#pragma unroll
            for (int i = 0; i < EPL; ++i) xv[i] = gather<GOP>(x + col(c[i], k0 + lane + 32 * i), pol_x);
#pragma unroll
            for (int i = 0; i < EPL; ++i) acc = __dadd_rn(acc, __dmul_rn(sval[lane + 32 * i], xv[i]));
            __syncwarp();
            const uint64_t tn = t + (uint64_t)NST * GW;
            if (lane == 0 && tn < n_tiles) {
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                issue(tn, s);
            }
            s = (s + 1 == NST) ? 0 : s + 1;
        }
    }
    out[gw * 32 + lane] = acc;
}

template <int EPL, int MODE, int GOP, int MINB>
int run(const uint32_t* idx, const double* val, const double* x, double* out, uint64_t nnz,
        int carve_pct, int cmode, uint32_t mask, uint32_t ncols, int iters, int sm_count, float* ms) {
    auto kern = ceil_kernel<EPL, MODE, GOP, MINB>;
    constexpr int WT = EPL * 32;
    const size_t smem = (MODE == 1) ? (size_t)8 * WT * 12 : (MODE == 3 ? (size_t)16 * WT * 12 : 0);
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return 2;
    int carve = carve_pct;
    if (carve < 0) carve = (int)(((smem + 1024) * MINB * 100 + 228 * 1024 - 1) / (228 * 1024));
    if (carve > 100) carve = 100;
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, carve);
    const uint64_t n_tiles = nnz / WT;
    int occ = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, 256, smem);
    const unsigned grid = (unsigned)(sm_count * (occ < MINB ? occ : MINB));
    if (grid == 0) return 3;
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    for (int i = 0; i < 2; ++i) kern<<<grid, 256, smem>>>(idx, val, x, out, n_tiles, cmode, mask, ncols);
    cudaEventRecord(e0);
    for (int i = 0; i < iters; ++i) kern<<<grid, 256, smem>>>(idx, val, x, out, n_tiles, cmode, mask, ncols);
    cudaEventRecord(e1);
    cudaError_t e = cudaEventSynchronize(e1);
    if (e != cudaSuccess) {
        fprintf(stderr, "lab: %s\n", cudaGetErrorString(e));
        return 4;
    }
    cudaEventElapsedTime(ms, e0, e1);
    *ms /= iters;
    ms[1] = (float)occ;
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    return 0;
}

}  // namespace

extern "C" int lab_ceiling(int epl, int mode, int gop, int minb, int carve_pct, int cmode,
                           uint32_t mask, uint32_t ncols, const uint32_t* idx, const double* val,
                           const double* x, double* out, uint64_t nnz, int iters, float* ms) {
    int dev = 0, sm = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, dev);
#define CASE(E, M, G, B)                                                                     \
    if (epl == E && mode == M && gop == G && minb == B)                                      \
        return run<E, M, G, B>(idx, val, x, out, nnz, carve_pct, cmode, mask, ncols, iters, sm, ms);
#define CASES_B(E, M, G) CASE(E, M, G, 2) CASE(E, M, G, 3) CASE(E, M, G, 4) CASE(E, M, G, 6)
#define CASES_G(E, M) CASES_B(E, M, 0) CASES_B(E, M, 1) CASES_B(E, M, 2) CASES_B(E, M, 3)
#define CASES_M(E) CASES_G(E, 0) CASES_G(E, 1) CASES_G(E, 2) CASES_G(E, 3)
    CASES_M(8)
    CASES_M(12)
    CASES_M(16)
    return 1;
}
