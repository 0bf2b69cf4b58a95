// diag.cu -- measurement aid, not a product path: the "gather ceiling" of a matrix.
//
// The SpMV of spmv.cu is bound by the x gathers (L1TEX line rate and the L1 lines in-flight
// gathers hold), not by HBM.  This kernel is the SpMV's memory behaviour with the row logic
// removed: it streams the mirror's (index, value) arrays in the same warp tiles with the same
// loads (ld.global.nc.L1::no_allocate, L2 evict_first), gathers x[col] with the same
// instruction (ld.global.nc, L2 evict_last), multiplies (unfused) and adds into ONE accumulator
// per lane -- no row boundaries, no reduction, no y.  Any SpMV that gathers x through L1/L2
// does at least this work, so its rate on the bench's own matrix is the ceiling the product
// kernel is held against (bench.py roofline.gather_ceiling; tools/spmv_lab.cu has the whole
// design space this variant -- "e8 m2 b2": 256-nnz tiles, next tile's indices prefetched, two
// CTAs of 8 warps per SM -- is the fastest of).
#include "common.cuh"
#include "ptx.cuh"

namespace {

constexpr int DIAG_EPL = 8, DIAG_NWARPS = 8, DIAG_CTAS = 2;

__global__ void __launch_bounds__(DIAG_NWARPS * 32, DIAG_CTAS)
    gather_ceiling_kernel(const uint32_t* __restrict__ idx, const double* __restrict__ val,
                          const double* __restrict__ x, double* __restrict__ out,
                          uint64_t n_tiles) {
    constexpr int WT = DIAG_EPL * 32;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t gw = (uint64_t)blockIdx.x * DIAG_NWARPS + warp;
    const uint64_t GW = (uint64_t)gridDim.x * DIAG_NWARPS;
    const uint64_t pol_s = policy_evict_first(), pol_x = policy_evict_last();
    double acc = 0.0;
    uint32_t cn[DIAG_EPL];
    if (gw < n_tiles) {
#pragma unroll
        for (int i = 0; i < DIAG_EPL; ++i) cn[i] = ldg_stream_u32(idx + gw * WT + lane + 32 * i, pol_s);
    }
    for (uint64_t t = gw; t < n_tiles; t += GW) {
        const uint64_t k0 = t * WT;
        double v[DIAG_EPL], xv[DIAG_EPL];
#pragma unroll
        for (int i = 0; i < DIAG_EPL; ++i) xv[i] = ldg_f64_hint(x + cn[i], pol_x);
#pragma unroll
        for (int i = 0; i < DIAG_EPL; ++i) v[i] = ldg_stream_f64(val + k0 + lane + 32 * i, pol_s);
        if (t + GW < n_tiles) {
#pragma unroll
            for (int i = 0; i < DIAG_EPL; ++i)
                cn[i] = ldg_stream_u32(idx + (t + GW) * WT + lane + 32 * i, pol_s);
        }
#pragma unroll
        for (int i = 0; i < DIAG_EPL; ++i) acc = __dadd_rn(acc, __dmul_rn(v[i], xv[i]));
    }
    out[gw * 32 + lane] = acc;
}

}  // namespace

extern "C" int sprs_b200_diag_gather_ceiling(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat,
                                             const double* d_x, int iters, double* ms_per_pass,
                                             uint64_t* nnz_covered) {
    if (!ctx || !mat || !d_x || !ms_per_pass || iters < 1) return SPRS_B200_ERR_ARGUMENT;
    if (mat->storage != SPRS_B200_CSR)
        SPRS_FAIL(ctx, SPRS_B200_ERR_STORAGE, "Storage mismatch: diag needs a CSR mirror");
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    constexpr int WT = DIAG_EPL * 32;
    const uint64_t n_tiles = mat->nnz / WT;  // whole tiles only (the ragged tail is < 0.001 %)
    if (nnz_covered) *nnz_covered = n_tiles * WT;
    *ms_per_pass = 0.0;
    if (n_tiles == 0) return SPRS_B200_OK;
    cudaStream_t s = ctx->stream;
    uint64_t grid = (uint64_t)ctx->sm_count * DIAG_CTAS;
    const uint64_t need = (n_tiles + DIAG_NWARPS - 1) / DIAG_NWARPS;
    if (grid > need) grid = need;
    void* d_out = nullptr;
    SPRS_TRY(ctx_scratch(ctx, 3, grid * DIAG_NWARPS * 32 * sizeof(double), &d_out));
    SPRS_CUDA(ctx, cudaFuncSetAttribute(gather_ceiling_kernel,
                                        cudaFuncAttributePreferredSharedMemoryCarveout, 0));
    cudaEvent_t e0, e1;
    SPRS_CUDA(ctx, cudaEventCreate(&e0));
    SPRS_CUDA(ctx, cudaEventCreate(&e1));
    for (int i = 0; i < 2; ++i)
        gather_ceiling_kernel<<<(unsigned)grid, DIAG_NWARPS * 32, 0, s>>>(
            mat->d_indices, mat->d_data, d_x, (double*)d_out, n_tiles);
    cudaEventRecord(e0, s);
    for (int i = 0; i < iters; ++i)
        gather_ceiling_kernel<<<(unsigned)grid, DIAG_NWARPS * 32, 0, s>>>(
            mat->d_indices, mat->d_data, d_x, (double*)d_out, n_tiles);
    cudaEventRecord(e1, s);
    cudaError_t e = cudaEventSynchronize(e1);
    float ms = 0.f;
    if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, e0, e1);
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    if (e != cudaSuccess) SPRS_FAIL(ctx, SPRS_B200_ERR_CUDA, "diag: %s", cudaGetErrorString(e));
    ctx->launches += (uint64_t)iters + 2;
    *ms_per_pass = (double)ms / iters;
    return SPRS_B200_OK;
}
