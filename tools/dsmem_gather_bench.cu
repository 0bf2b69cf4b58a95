// dsmem_gather_bench.cu -- how fast can a thread-block CLUSTER gather random 8-byte words out
// of its distributed shared memory?  (round-2 question behind DESIGN.md 4.1: the SpMV sits on
// the L1TEX ceiling of one gathered line per clock per SM and on the L2->SM sector traffic;
// a cluster of 16 CTAs holds 16 x 128 KB = 2 MB of x on chip, reachable without either.)
//
// Every CTA fills PER_CTA doubles of shared memory; the cluster-wide table is the concatenation.
// Threads stream random indices from global memory (coalesced, 4 B each) and gather table
// entries with ld.shared::cluster (cluster.map_shared_rank), U loads in flight per thread.
// Cluster size 1 measures plain shared-memory random reads (bank conflicts only).
// Prints G elements/s and elements per clock per SM; compare with tools/gather_bench.cu's global
// gathers.
// Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a tools/dsmem_gather_bench.cu -o dsmem_gather_bench
#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
namespace cg = cooperative_groups;
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

constexpr int PER_CTA_LOG2 = 14;               // 16384 doubles = 128 KB per CTA
constexpr uint32_t PER_CTA = 1u << PER_CTA_LOG2;
constexpr int NT = 512;

__device__ __forceinline__ uint64_t mix64(uint64_t z) {
    z += 0x9E3779B97F4A7C15ull; z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; return z ^ (z >> 31);
}
__global__ void fill_idx(uint32_t* idx, uint64_t n, uint32_t range) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n) idx[i] = (uint32_t)__umul64hi(mix64(i), range);
}

template <int U>
__global__ void __launch_bounds__(NT) dsmem_gather_k(const uint32_t* __restrict__ idx, uint64_t n, double* out) {
    extern __shared__ double tab[];
    cg::cluster_group cl = cg::this_cluster();
    const unsigned nb = cl.num_blocks(), rk = cl.block_rank();
    for (uint32_t i = threadIdx.x; i < PER_CTA; i += NT) tab[i] = 1.0 + (double)((rk << PER_CTA_LOG2) + i) * 1e-6;
    cl.sync();
    // the table of this cluster has nb * PER_CTA entries; idx was drawn in [0, 16 * PER_CTA)
    const uint32_t mask = nb * PER_CTA - 1;  // nb is a power of two
    double acc = 0;
    for (uint64_t tile = (uint64_t)blockIdx.x * NT * U; tile < n; tile += (uint64_t)gridDim.x * NT * U) {
        uint32_t c[U];
#pragma unroll
        for (int u = 0; u < U; ++u) { uint64_t e = tile + threadIdx.x + (uint64_t)u * NT; c[u] = e < n ? (idx[e] & mask) : 0; }
        double v[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {  // mapa + ld.shared::cluster (not a generic load)
            const uint32_t local = (uint32_t)__cvta_generic_to_shared(tab + (c[u] & (PER_CTA - 1)));
            uint32_t remote;
            asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local), "r"(c[u] >> PER_CTA_LOG2));
            asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v[u]) : "r"(remote));
        }
#pragma unroll
        for (int u = 0; u < U; ++u) acc += v[u];
    }
    cl.sync();  // nobody leaves while a peer may still read its shared memory
    if (acc == 123.456) out[0] = acc;
}

int main() {
    const uint64_t n = 1ull << 28;
    uint32_t* idx; double* out;
    CK(cudaMalloc(&idx, n * 4)); CK(cudaMalloc(&out, 64));
    fill_idx<<<(unsigned)((n + 255) / 256), 256>>>(idx, n, 16u * PER_CTA);
    CK(cudaDeviceSynchronize());
    int sms = 132, khz = 1980000;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    auto kern = dsmem_gather_k<8>;
    const size_t smem = (size_t)PER_CTA * 8;
    CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CK(cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    for (int cs : {1, 2, 4, 8, 16}) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned)(sms / cs * cs));  // one CTA per SM, whole clusters
        cfg.blockDim = dim3(NT);
        cfg.dynamicSmemBytes = smem;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = (unsigned)cs; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        int max_clusters = 0;
        cudaError_t qe = cudaOccupancyMaxActiveClusters(&max_clusters, kern, &cfg);
        if (qe != cudaSuccess || max_clusters == 0) { printf("cluster %2d: not launchable (%s)\n", cs, cudaGetErrorString(qe)); cudaGetLastError(); continue; }
        cudaEvent_t a, b; CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
        CK(cudaLaunchKernelEx(&cfg, kern, (const uint32_t*)idx, n, out));  // warm-up
        CK(cudaDeviceSynchronize());
        CK(cudaEventRecord(a));
        for (int r = 0; r < 5; ++r) CK(cudaLaunchKernelEx(&cfg, kern, (const uint32_t*)idx, n, out));
        CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b));
        float ms = 0; CK(cudaEventElapsedTime(&ms, a, b)); ms /= 5;
        const double gel = n / ms / 1e6;
        printf("cluster %2d (%4.1f MB table, %d active clusters): %.3f ms  %.1f Gelem/s  = %.2f elem/clk/SM (index stream %.0f GB/s)\n",
               cs, cs * smem / 1e6, max_clusters, ms, gel, gel * 1e9 / ((double)cfg.gridDim.x * khz * 1e3), 4.0 * n / ms / 1e6);
    }
    return 0;
}
