// cuemu.cpp -- TEST INFRASTRUCTURE ONLY (see cuemu.h): fibers, the block scheduler, warp
// collectives, and the handful of CUDA runtime calls the library's host code makes.
#include "cuemu.h"

#include <sys/mman.h>

#include <vector>

// ---- context switch (x86-64 SysV): callee-saved registers + stack pointer -------------------
extern "C" void cuemu_switch(void** save_sp, void* new_sp);
asm(R"(
.text
.globl cuemu_switch
.type cuemu_switch,@function
cuemu_switch:
    pushq %rbp
    pushq %rbx
    pushq %r12
    pushq %r13
    pushq %r14
    pushq %r15
    movq %rsp, (%rdi)
    movq %rsi, %rsp
    popq %r15
    popq %r14
    popq %r13
    popq %r12
    popq %rbx
    popq %rbp
    ret
.size cuemu_switch,.-cuemu_switch
)");

namespace cuemu {

Fiber* g_cur = nullptr;
dim3 g_block_dim, g_grid_dim;
uint3 g_block_idx{0, 0, 0};

namespace {

constexpr size_t STACK_BYTES = 256 * 1024;
constexpr unsigned MAX_THREADS = 1024;

struct WarpSync {
    unsigned alive = 0;      // lanes that exist and have not returned
    unsigned arrived = 0;    // lanes waiting at the current collective
    unsigned lane_mask[32];  // the mask each waiting lane named
    unsigned released = 0;   // lanes allowed to leave
    uint64_t slot[32];
    unsigned ballot = 0;
};

std::vector<Fiber> g_fibers;
std::vector<WarpSync> g_warps;
void* g_sched_sp = nullptr;
const std::function<void()>* g_body = nullptr;
unsigned g_live = 0;
unsigned g_barrier_arrived = 0;
unsigned long long g_barrier_gen = 0;
unsigned long long g_progress = 0;
std::vector<unsigned char> g_smem;
void* g_smem_aligned = nullptr;
cudaError_t g_last_error = cudaSuccess;
unsigned long long g_rng = 0x9E3779B97F4A7C15ull;

void release_block_barrier_if_complete() {
    if (g_live > 0 && g_barrier_arrived == g_live) {
        g_barrier_arrived = 0;
        ++g_barrier_gen;
        ++g_progress;
    }
}

// Release every group of waiting lanes (a group = the lanes that named the same mask) whose
// live members have all arrived.
void release_warp_if_complete(WarpSync& w) {
    unsigned todo = w.arrived;
    while (todo) {
        const int l = __builtin_ctz(todo);
        const unsigned m = w.lane_mask[l];
        unsigned group = 0;
        for (int k = 0; k < 32; ++k)
            if ((w.arrived >> k & 1u) && w.lane_mask[k] == m) group |= 1u << k;
        const unsigned need = m & w.alive;
        if ((group & need) == need) {
            w.released |= group;
            w.arrived &= ~group;
            ++g_progress;
        }
        todo &= ~group;
    }
}

void fiber_exit() {
    Fiber* f = g_cur;
    f->done = true;
    --g_live;
    ++g_progress;
    WarpSync& w = g_warps[f->warp];
    w.alive &= ~(1u << f->lane);
    release_warp_if_complete(w);
    release_block_barrier_if_complete();
    void* dummy;
    cuemu_switch(&dummy, g_sched_sp);  // never resumed
    abort();
}

extern "C" void cuemu_fiber_main() {
    (*g_body)();
    fiber_exit();
}

void prepare_fiber(Fiber& f) {
    if (!f.stack) {
        void* m = mmap(nullptr, STACK_BYTES, PROT_READ | PROT_WRITE,
                       MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
        if (m == MAP_FAILED) {
            perror("cuemu: mmap");
            abort();
        }
        f.stack = (char*)m;
    }
    // initial frame: six callee-saved slots, the entry address, a null return address
    uintptr_t top = ((uintptr_t)f.stack + STACK_BYTES) & ~(uintptr_t)15;
    void** sp = (void**)top;
    *--sp = nullptr;                          // fake return address of cuemu_fiber_main
    *--sp = (void*)&cuemu_fiber_main;         // popped by `ret` in cuemu_switch
    for (int i = 0; i < 6; ++i) *--sp = nullptr;
    f.sp = sp;
    f.done = false;
}

void run_block(unsigned nthreads) {
    g_live = nthreads;
    g_barrier_arrived = 0;
    const unsigned nwarps = (nthreads + 31) / 32;
    g_warps.assign(nwarps, WarpSync());
    for (unsigned t = 0; t < nthreads; ++t) {
        Fiber& f = g_fibers[t];
        f.linear = t;
        f.lane = t & 31;
        f.warp = t >> 5;
        f.tid.x = t % g_block_dim.x;
        f.tid.y = (t / g_block_dim.x) % g_block_dim.y;
        f.tid.z = t / (g_block_dim.x * g_block_dim.y);
        g_warps[f.warp].alive |= 1u << f.lane;
        prepare_fiber(f);
    }
    // Order in which the runnable threads get the CPU in each round.  Any order is a legal
    // CUDA schedule, so results must not depend on it: CUEMU_SCHEDULE=reverse | random[:seed]
    // (default: forward) lets the test-suite look for missing barriers under other schedules.
    static const int mode = [] {
        const char* e = getenv("CUEMU_SCHEDULE");
        if (!e || !*e || !strncmp(e, "forward", 7)) return 0;
        if (!strncmp(e, "reverse", 7)) return 1;
        if (!strncmp(e, "random", 6)) {
            if (e[6] == ':') g_rng = strtoull(e + 7, nullptr, 10) * 2654435761ull + 1;
            return 2;
        }
        fprintf(stderr, "cuemu: unknown CUEMU_SCHEDULE '%s'\n", e);
        abort();
    }();
    static std::vector<unsigned> order;
    order.resize(nthreads);
    for (unsigned t = 0; t < nthreads; ++t) order[t] = mode == 1 ? nthreads - 1 - t : t;
    unsigned idle_rounds = 0;
    while (g_live) {
        const unsigned long long before = g_progress;
        if (mode == 2)
            for (unsigned t = nthreads; t > 1; --t) {  // Fisher-Yates with a 64-bit LCG
                g_rng = g_rng * 6364136223846793005ull + 1442695040888963407ull;
                std::swap(order[t - 1], order[(g_rng >> 33) % t]);
            }
        for (unsigned k = 0; k < nthreads; ++k) {
            const unsigned t = order[k];
            Fiber& f = g_fibers[t];
            if (f.done) continue;
            g_cur = &f;
            cuemu_switch(&g_sched_sp, f.sp);
        }
        g_cur = nullptr;
        if (g_progress == before) {
            if (++idle_rounds > 4) {
                fprintf(stderr,
                        "cuemu: DEADLOCK in block (%u,%u,%u): %u threads alive, %u at "
                        "__syncthreads, none can proceed\n",
                        g_block_idx.x, g_block_idx.y, g_block_idx.z, g_live, g_barrier_arrived);
                abort();
            }
        } else {
            idle_rounds = 0;
        }
    }
}

}  // namespace

void note_progress() { ++g_progress; }

void yield() {
    Fiber* f = g_cur;
    cuemu_switch(&f->sp, g_sched_sp);
    g_cur = f;
}

void* dyn_smem() { return g_smem_aligned; }

void block_barrier() {
    ++g_barrier_arrived;
    ++g_progress;
    const unsigned long long gen = g_barrier_gen;
    release_block_barrier_if_complete();
    while (g_barrier_gen == gen) yield();
}

void warp_barrier(unsigned mask) {
    Fiber* f = g_cur;
    WarpSync& w = g_warps[f->warp];
    const unsigned bit = 1u << f->lane;
    if (!(mask & bit)) {
        fprintf(stderr, "cuemu: lane %u calls a warp collective whose mask 0x%08x omits it\n",
                f->lane, mask);
        abort();
    }
    w.arrived |= bit;
    w.lane_mask[f->lane] = mask;
    ++g_progress;
    release_warp_if_complete(w);
    while (!(w.released & bit)) yield();
    w.released &= ~bit;
}

uint64_t warp_exchange(unsigned mask, uint64_t mine, int src_lane) {
    Fiber* f = g_cur;
    WarpSync& w = g_warps[f->warp];
    w.slot[f->lane] = mine;
    warp_barrier(mask);
    const uint64_t got = w.slot[src_lane & 31];
    warp_barrier(mask);  // nobody overwrites a slot before every lane has read
    return got;
}

unsigned warp_ballot(unsigned mask, bool pred) {
    Fiber* f = g_cur;
    WarpSync& w = g_warps[f->warp];
    const unsigned bit = 1u << f->lane;
    w.ballot = pred ? (w.ballot | bit) : (w.ballot & ~bit);
    warp_barrier(mask);
    const unsigned got = w.ballot & mask & (w.alive | bit);
    warp_barrier(mask);
    return got;
}

unsigned warp_match_any(unsigned mask, uint64_t value) {
    Fiber* f = g_cur;
    WarpSync& w = g_warps[f->warp];
    w.slot[f->lane] = value;
    warp_barrier(mask);
    unsigned got = 0;
    for (int l = 0; l < 32; ++l)
        if ((mask >> l & 1u) && (w.alive >> l & 1u) && w.slot[l] == value) got |= 1u << l;
    warp_barrier(mask);
    return got;
}

void launch(const Cfg& c, const std::function<void()>& thread_body) {
    const unsigned nthreads = c.block.x * c.block.y * c.block.z;
    if (nthreads == 0 || nthreads > MAX_THREADS || c.grid.x == 0 || c.grid.y == 0 ||
        c.grid.z == 0 || c.smem > 227 * 1024) {
        g_last_error = 9;  // cudaErrorInvalidConfiguration
        return;
    }
    if (g_cur) {
        fprintf(stderr, "cuemu: kernel launch from device code is not supported\n");
        abort();
    }
    if (g_fibers.size() < nthreads) g_fibers.resize(MAX_THREADS);
    g_smem.assign(c.smem + 256, 0xA5);  // shared memory starts out as garbage
    g_smem_aligned = (void*)(((uintptr_t)g_smem.data() + 127) & ~(uintptr_t)127);
    g_block_dim = c.block;
    g_grid_dim = c.grid;
    g_body = &thread_body;
    for (unsigned z = 0; z < c.grid.z; ++z)
        for (unsigned y = 0; y < c.grid.y; ++y)
            for (unsigned x = 0; x < c.grid.x; ++x) {
                g_block_idx = uint3{x, y, z};
                std::memset(g_smem.data(), 0xA5, g_smem.size());
                run_block(nthreads);
            }
    g_body = nullptr;
}

}  // namespace cuemu

// ---- runtime API -----------------------------------------------------------------------------
const char* cudaGetErrorString(cudaError_t e) {
    switch (e) {
        case cudaSuccess: return "no error";
        case cudaErrorMemoryAllocation: return "out of memory";
        case 9: return "invalid configuration argument";
        case cudaErrorNotSupported: return "operation not supported (cuemu)";
        default: return "cuemu error";
    }
}
cudaError_t cudaGetLastError() {
    const cudaError_t e = cuemu::g_last_error;
    cuemu::g_last_error = cudaSuccess;
    return e;
}
cudaError_t cudaMalloc(void** p, size_t bytes) {
    // like the device allocator: 256-byte aligned, contents undefined (poisoned here); the
    // size is exact so that an address-sanitizer build sees out-of-bounds accesses
    void* m = nullptr;
    if (posix_memalign(&m, 256, bytes ? bytes : 1) != 0) return cudaErrorMemoryAllocation;
    std::memset(m, 0xA5, bytes);
    *p = m;
    return cudaSuccess;
}
cudaError_t cudaFree(void* p) {
    free(p);
    return cudaSuccess;
}
cudaError_t cudaMallocHost(void** p, size_t bytes) {
    *p = malloc(bytes ? bytes : 1);
    return *p ? cudaSuccess : cudaErrorMemoryAllocation;
}
cudaError_t cudaFreeHost(void* p) {
    free(p);
    return cudaSuccess;
}
cudaError_t cudaMemcpy(void* dst, const void* src, size_t bytes, cudaMemcpyKind) {
    if (bytes) std::memmove(dst, src, bytes);
    return cudaSuccess;
}
cudaError_t cudaMemcpyAsync(void* dst, const void* src, size_t bytes, cudaMemcpyKind k,
                            cudaStream_t) {
    return cudaMemcpy(dst, src, bytes, k);
}
cudaError_t cudaMemsetAsync(void* dst, int value, size_t bytes, cudaStream_t) {
    if (bytes) std::memset(dst, value, bytes);
    return cudaSuccess;
}
cudaError_t cudaMemset(void* dst, int value, size_t bytes) {
    return cudaMemsetAsync(dst, value, bytes, nullptr);
}
cudaError_t cudaStreamCreateWithPriority(cudaStream_t* s, unsigned flags, int) {
    return cudaStreamCreateWithFlags(s, flags);
}
cudaError_t cudaDeviceGetStreamPriorityRange(int* least, int* greatest) {
    *least = 0;
    *greatest = -5;
    return cudaSuccess;
}
cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) {
    *e = (cudaEvent_t)malloc(8);
    return cudaSuccess;
}
cudaError_t cudaEventDestroy(cudaEvent_t e) {
    free(e);
    return cudaSuccess;
}
// kernels run to completion inside the launch call: every event has already happened
cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return cudaSuccess; }
cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
long long clock64() {
    static long long t = 0;
    return t += 1000;
}
cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) {
    *s = (cudaStream_t)malloc(8);
    return cudaSuccess;
}
cudaError_t cudaStreamDestroy(cudaStream_t s) {
    free(s);
    return cudaSuccess;
}
cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
cudaError_t cudaSetDevice(int d) { return d == 0 ? cudaSuccess : 101; }
cudaError_t cudaGetDeviceCount(int* n) {
    *n = 1;
    return cudaSuccess;
}
cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int) {
    std::memset(p, 0, sizeof(*p));
    std::snprintf(p->name, sizeof(p->name), "cuemu (CPU emulation, tests only)");
    p->multiProcessorCount = 4;  // small grids keep the emulation quick
    p->l2CacheSize = 1 << 20;
    p->totalGlobalMem = (size_t)1 << 32;
    p->major = 9;  // the compute capability the library is built for (sm_90a)
    p->minor = 0;
    return cudaSuccess;
}
// every host pointer is "pinned and mapped" here (device memory IS host memory)
cudaError_t cudaPointerGetAttributes(cudaPointerAttributes* a, const void* p) {
    a->type = cudaMemoryTypeHost;
    a->device = 0;
    a->devicePointer = const_cast<void*>(p);
    a->hostPointer = const_cast<void*>(p);
    return cudaSuccess;
}
cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t*, void*) { return cudaErrorNotSupported; }
cudaError_t cudaIpcOpenMemHandle(void**, cudaIpcMemHandle_t, unsigned) {
    return cudaErrorNotSupported;
}
cudaError_t cudaIpcCloseMemHandle(void*) { return cudaErrorNotSupported; }
