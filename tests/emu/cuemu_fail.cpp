// TEST INFRASTRUCTURE ONLY: the emulator (cuemu.cpp) with an allocation-failure hook, linked in
// place of cuemu.o by tests/test_emu_alloc_failure.py.  The emulator's allocation functions are
// compiled under other names and wrapped: the n-th next cudaMalloc / cudaMallocAsync /
// cudaMallocHost fails like an exhausted device, and live allocations are counted so that a test
// sees leaks.
#define cudaMalloc cuemu_base_cudaMalloc
#define cudaFree cuemu_base_cudaFree
#define cudaMallocHost cuemu_base_cudaMallocHost
#define cudaFreeHost cuemu_base_cudaFreeHost
#include "cuemu.cpp"
#undef cudaMalloc
#undef cudaFree
#undef cudaMallocHost
#undef cudaFreeHost

namespace {
long g_fail_after = -1;
long g_live_allocs = 0;

bool alloc_fails() {
    if (g_fail_after < 0 || g_fail_after-- > 0) return false;
    cuemu::g_last_error = cudaErrorMemoryAllocation;  // like the runtime: the error stays behind
    return true;
}
}  // namespace

// n < 0: no failure armed.  Returns what was still armed: < 0 once the armed failure happened.
extern "C" long cuemu_fail_alloc_after(long n) {
    const long left = g_fail_after;
    g_fail_after = n;
    return left;
}
// allocations minus frees
extern "C" long cuemu_live_allocs() { return g_live_allocs; }

cudaError_t cudaMalloc(void** p, size_t bytes) {
    if (alloc_fails()) return cudaErrorMemoryAllocation;
    const cudaError_t e = cuemu_base_cudaMalloc(p, bytes);
    if (e == cudaSuccess) ++g_live_allocs;
    return e;
}
cudaError_t cudaFree(void* p) {
    if (p) --g_live_allocs;
    return cuemu_base_cudaFree(p);
}
cudaError_t cudaMallocHost(void** p, size_t bytes) {
    if (alloc_fails()) return cudaErrorMemoryAllocation;
    const cudaError_t e = cuemu_base_cudaMallocHost(p, bytes);
    if (e == cudaSuccess) ++g_live_allocs;
    return e;
}
cudaError_t cudaFreeHost(void* p) {
    if (p) --g_live_allocs;
    return cuemu_base_cudaFreeHost(p);
}
