// gather_bench.cu -- microbenchmarks that bound the SpMV design on H100 (DESIGN.md):
//   copy     : streaming read+write bandwidth (the HBM roofline denominator's cousin)
//   stream   : read-only stream of 12 B/element (index + value), like the CSR arrays
//   gather   : random 8-byte gathers from a table of T bytes (x of an SpMV)
//   spmvlike : stream 12 B + 1 random gather per element (no reduction)
// Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a tools/gather_bench.cu -o gather_bench
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

__device__ __forceinline__ uint64_t mix64(uint64_t z) {
    z += 0x9E3779B97F4A7C15ull; z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; return z ^ (z >> 31);
}
__global__ void fill_idx(uint32_t* idx, uint64_t n, uint32_t range, int mode) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t h = mix64(i);
    if (mode == 0) idx[i] = (uint32_t)__umul64hi(h, range);                // uniform random
    else { // clustered: runs of 4 consecutive columns (FEM-like)
        uint64_t h4 = mix64(i >> 2); idx[i] = (uint32_t)((__umul64hi(h4, range - 4)) + (i & 3)); }
}
__global__ void fill_val(double* v, uint64_t n) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n) v[i] = 1.0 + (double)(i & 1023) * 1e-3;
}
__global__ void copy_k(const double4* __restrict__ a, double4* __restrict__ b, uint64_t n4) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (; i < n4; i += stride) b[i] = a[i];
}
template <int U>
__global__ void gather_k(const uint32_t* __restrict__ idx, const double* __restrict__ x, double* out, uint64_t n, int withval, const double* __restrict__ val) {
    uint64_t tile = (uint64_t)blockIdx.x * blockDim.x * U;
    double acc = 0;
    for (; tile < n; tile += (uint64_t)gridDim.x * blockDim.x * U) {
        uint32_t c[U]; double v[U];
#pragma unroll
        for (int u = 0; u < U; ++u) { uint64_t e = tile + threadIdx.x + (uint64_t)u * blockDim.x; c[u] = e < n ? idx[e] : 0; }
        if (withval) {
#pragma unroll
            for (int u = 0; u < U; ++u) { uint64_t e = tile + threadIdx.x + (uint64_t)u * blockDim.x; v[u] = e < n ? val[e] : 0; }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) acc += (withval ? v[u] : 1.0) * __ldg(x + c[u]);
    }
    if (acc == 123.456) out[0] = acc;
}
__global__ void stream_k(const uint32_t* __restrict__ idx, const double* __restrict__ val, double* out, uint64_t n) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    double acc = 0;
    const uint4* i4 = (const uint4*)idx; const double2* v2 = (const double2*)val;
    for (; i < n / 4; i += stride) { uint4 c = i4[i]; double2 a = v2[2 * i], b = v2[2 * i + 1]; acc += a.x + a.y + b.x + b.y + (double)(c.x ^ c.y ^ c.z ^ c.w); }
    if (acc == 123.456) out[0] = acc;
}
template <typename F> float timeit(F f, int reps = 10) {
    cudaEvent_t a, b; CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
    f(); f(); CK(cudaDeviceSynchronize());
    float best = 1e30f;
    for (int r = 0; r < reps; ++r) { CK(cudaEventRecord(a)); f(); CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b)); float ms; CK(cudaEventElapsedTime(&ms, a, b)); if (ms < best) best = ms; }
    return best;
}
int main() {
    const uint64_t n = 1ull << 28;  // 268M elements: 1 GB idx + 2 GB val
    uint32_t* idx; double *val, *x, *out, *cp;
    CK(cudaMalloc(&idx, n * 4)); CK(cudaMalloc(&val, n * 8)); CK(cudaMalloc(&x, 1ull << 30)); CK(cudaMalloc(&out, 64)); CK(cudaMalloc(&cp, n * 8));
    fill_val<<<(unsigned)((n + 255) / 256), 256>>>(val, n);
    fill_val<<<(unsigned)(((1ull << 27) + 255) / 256), 256>>>(x, 1ull << 27);
    int sms = 132; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    float ms = timeit([&] { copy_k<<<sms * 16, 512>>>((const double4*)val, (double4*)cp, n / 4); });
    printf("copy      : %.3f ms  %.1f GB/s (read+write)\n", ms, 2.0 * n * 8 / ms / 1e6);
    ms = timeit([&] { stream_k<<<sms * 16, 512>>>(idx, val, out, n); });
    printf("stream12  : %.3f ms  %.1f GB/s (read only)\n", ms, 12.0 * n / ms / 1e6);
    const uint64_t tables[] = {1ull << 17, 1ull << 20, 10ull * 1000 * 1000, 1ull << 25, 1ull << 27};  // elements: 1MB, 8MB, 80MB, 256MB, 1GB
    for (int mode = 0; mode < 2; ++mode)
        for (uint64_t T : tables) {
            fill_idx<<<(unsigned)((n + 255) / 256), 256>>>(idx, n, (uint32_t)T, mode);
            CK(cudaDeviceSynchronize());
            for (int occ : {4, 8}) {
                float g = timeit([&] { gather_k<8><<<sms * occ, 256>>>(idx, x, out, n, 0, val); }, 5);
                float s = timeit([&] { gather_k<8><<<sms * occ, 256>>>(idx, x, out, n, 1, val); }, 5);
                printf("%s table %7.1f MB occ %d: gather-only %.3f ms %.1f Gelem/s | spmv-like %.3f ms %.1f Gelem/s = %.1f GB/s of 12B/nnz\n",
                       mode ? "clustered4" : "uniform   ", T * 8 / 1e6, occ, g, n / g / 1e6, s, n / s / 1e6, 12.0 * n / s / 1e6);
            }
        }
    return 0;
}
