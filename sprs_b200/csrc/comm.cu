// comm.cu -- multi-GPU plumbing of the row-partitioned products behind the C ABI (no torch,
// no NCCL): rendezvous of the ranks of ONE node, symmetric device buffers every rank can
// store into (CUDA IPC, or CUDA VMM + an NVSwitch multicast object when the devices have
// one), a stream-ordered device barrier (flags in peer memory), and the row-partitioned
// SpMV entry points (SURVEY 8b "comm_init / spmv_rowpart", 8e).
//
// The reference has no multi-device code (SURVEY 2.4); its shard primitive is slice_outer
// (sprs/src/sparse/slicing.rs:65-89), which sprs_b200_partition_rows cuts by cost.
//
// Rendezvous: rank 0 creates a POSIX shared-memory segment named after a 64-byte id the
// caller ships to the other ranks by any transport (the way an ncclUniqueId travels); the
// segment carries a sense-reversing host barrier and one 512-byte mailbox per rank, enough to
// all-gather IPC handles, pids and partition bounds.  File descriptors (VMM shareable handles)
// travel over abstract unix sockets (SCM_RIGHTS).  Ranks may be processes (one per GPU, the
// torchrun layout) or threads of one process (then peers are reached by direct peer access
// instead of IPC) -- two ranks may even share one device, which is how the multi-rank logic is
// tested on a single-GPU box.
#include <cuda.h>

#include <atomic>
#include <chrono>
#include <cstdlib>
#include <thread>

#include <errno.h>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/socket.h>
#include <sys/stat.h>
#include <sys/un.h>
#include <time.h>
#include <unistd.h>

#include "common.cuh"

constexpr int COMM_MAX_RANKS = SPRS_B200_MAX_RANKS;
constexpr size_t COMM_BLOB = 512;
constexpr uint32_t COMM_MAGIC = 0x5B200C01u;

struct CommShm {
    std::atomic<uint32_t> magic;
    uint32_t world;
    std::atomic<uint32_t> bar_count;
    std::atomic<uint32_t> bar_gen;
    std::atomic<uint32_t> failed;  // a rank gave up: everybody else stops waiting
    unsigned char blob[COMM_MAX_RANKS][COMM_BLOB];
};

struct sprs_b200_symm {
    sprs_b200_comm* comm = nullptr;
    uint64_t bytes = 0;
    void* ptr[COMM_MAX_RANKS] = {};  // rank g's buffer as mapped in this process
    void* mc_ptr = nullptr;          // NVSwitch multicast address of all of them, or null
    bool vmm = false;
    bool ipc_opened[COMM_MAX_RANKS] = {};
    // VMM flavour
    size_t map_bytes = 0;
    CUmemGenericAllocationHandle mem[COMM_MAX_RANKS] = {};
    CUmemGenericAllocationHandle mc = 0;
};

struct sprs_b200_comm {
    sprs_b200_ctx* ctx = nullptr;
    int rank = 0, world = 1;
    char id[64] = {};
    CommShm* shm = nullptr;
    int pid[COMM_MAX_RANKS] = {};
    int device[COMM_MAX_RANKS] = {};
    int multicast_ok = 0;  // every rank's device supports multicast and devices are distinct
    int listen_fd = -1;
    sprs_b200_symm* flags = nullptr;  // device barrier: COMM_MAX_RANKS u64 per rank
    unsigned long long* d_err = nullptr;
    uint64_t epoch = 0;
    double timeout_s = 120.0;
};

namespace {

double now_s() {
    timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return ts.tv_sec + 1e-9 * ts.tv_nsec;
}

std::string shm_name(const char* id) { return std::string("/sprs_b200_") + id; }

// ---- host barrier + mailbox all-gather over the shared segment ----------------------
int host_barrier(sprs_b200_comm* c) {
    if (c->world == 1) return SPRS_B200_OK;
    CommShm* h = c->shm;
    const uint32_t gen = h->bar_gen.load(std::memory_order_acquire);
    if (h->bar_count.fetch_add(1, std::memory_order_acq_rel) + 1 == (uint32_t)c->world) {
        h->bar_count.store(0, std::memory_order_relaxed);
        h->bar_gen.store(gen + 1, std::memory_order_release);
        return SPRS_B200_OK;
    }
    const double t0 = now_s();
    unsigned spins = 0;
    while (h->bar_gen.load(std::memory_order_acquire) == gen) {
        if (h->failed.load(std::memory_order_relaxed))
            SPRS_FAIL(c->ctx, SPRS_B200_ERR_COMM, "comm: another rank failed");
        if (++spins > 2000) {
            std::this_thread::sleep_for(std::chrono::microseconds(50));
            if (now_s() - t0 > c->timeout_s) {
                h->failed.store(1);
                SPRS_FAIL(c->ctx, SPRS_B200_ERR_COMM, "comm: host barrier timed out after %.0f s",
                          c->timeout_s);
            }
        }
    }
    return SPRS_B200_OK;
}

int host_allgather(sprs_b200_comm* c, const void* mine, size_t bytes, void* all) {
    if (bytes > COMM_BLOB) SPRS_FAIL(c->ctx, SPRS_B200_ERR_ARGUMENT, "comm: blob too large");
    if (c->world == 1) {
        memcpy(all, mine, bytes);
        return SPRS_B200_OK;
    }
    memcpy(c->shm->blob[c->rank], mine, bytes);
    SPRS_TRY(host_barrier(c));
    for (int g = 0; g < c->world; ++g) memcpy((char*)all + g * bytes, c->shm->blob[g], bytes);
    SPRS_TRY(host_barrier(c));  // nobody overwrites a mailbox before everyone has read it
    return SPRS_B200_OK;
}

// ---- file descriptors between ranks (abstract unix sockets, SCM_RIGHTS) -----------------
void sock_addr(const sprs_b200_comm* c, int rank, sockaddr_un* a, socklen_t* len) {
    memset(a, 0, sizeof(*a));
    a->sun_family = AF_UNIX;
    const int n = snprintf(a->sun_path + 1, sizeof(a->sun_path) - 1, "sprs_b200_%s_%d", c->id, rank);
    *len = (socklen_t)(offsetof(sockaddr_un, sun_path) + 1 + n);
}

int sock_listen(sprs_b200_comm* c) {
    if (c->listen_fd >= 0) return SPRS_B200_OK;
    const int fd = socket(AF_UNIX, SOCK_STREAM, 0);
    if (fd < 0) SPRS_FAIL(c->ctx, SPRS_B200_ERR_COMM, "comm: socket(): %s", strerror(errno));
    sockaddr_un a;
    socklen_t len;
    sock_addr(c, c->rank, &a, &len);
    if (bind(fd, (sockaddr*)&a, len) != 0 || listen(fd, COMM_MAX_RANKS) != 0) {
        close(fd);
        SPRS_FAIL(c->ctx, SPRS_B200_ERR_COMM, "comm: bind/listen: %s", strerror(errno));
    }
    c->listen_fd = fd;
    return SPRS_B200_OK;
}

int send_fd(sprs_b200_comm* c, int to_rank, int fd_to_send) {
    const int s = socket(AF_UNIX, SOCK_STREAM, 0);
    if (s < 0) SPRS_FAIL(c->ctx, SPRS_B200_ERR_COMM, "comm: socket(): %s", strerror(errno));
    sockaddr_un a;
    socklen_t len;
    sock_addr(c, to_rank, &a, &len);
    if (connect(s, (sockaddr*)&a, len) != 0) {
        close(s);
        SPRS_FAIL(c->ctx, SPRS_B200_ERR_COMM, "comm: connect to rank %d: %s", to_rank, strerror(errno));
    }
    int from = c->rank;
    iovec iov{&from, sizeof(from)};
    alignas(cmsghdr) char ctrl[CMSG_SPACE(sizeof(int))] = {};
    msghdr msg{};
    msg.msg_iov = &iov;
    msg.msg_iovlen = 1;
    msg.msg_control = ctrl;
    msg.msg_controllen = sizeof(ctrl);
    cmsghdr* cm = CMSG_FIRSTHDR(&msg);
    cm->cmsg_level = SOL_SOCKET;
    cm->cmsg_type = SCM_RIGHTS;
    cm->cmsg_len = CMSG_LEN(sizeof(int));
    memcpy(CMSG_DATA(cm), &fd_to_send, sizeof(int));
    const ssize_t n = sendmsg(s, &msg, 0);
    close(s);
    if (n != (ssize_t)sizeof(from))
        SPRS_FAIL(c->ctx, SPRS_B200_ERR_COMM, "comm: sendmsg: %s", strerror(errno));
    return SPRS_B200_OK;
}

int recv_fd(sprs_b200_comm* c, int* from_rank, int* fd_out) {
    const int s = accept(c->listen_fd, nullptr, nullptr);
    if (s < 0) SPRS_FAIL(c->ctx, SPRS_B200_ERR_COMM, "comm: accept: %s", strerror(errno));
    int from = -1;
    iovec iov{&from, sizeof(from)};
    alignas(cmsghdr) char ctrl[CMSG_SPACE(sizeof(int))] = {};
    msghdr msg{};
    msg.msg_iov = &iov;
    msg.msg_iovlen = 1;
    msg.msg_control = ctrl;
    msg.msg_controllen = sizeof(ctrl);
    const ssize_t n = recvmsg(s, &msg, 0);
    close(s);
    cmsghdr* cm = CMSG_FIRSTHDR(&msg);
    if (n != (ssize_t)sizeof(from) || !cm || cm->cmsg_type != SCM_RIGHTS)
        SPRS_FAIL(c->ctx, SPRS_B200_ERR_COMM, "comm: recvmsg without a descriptor");
    memcpy(fd_out, CMSG_DATA(cm), sizeof(int));
    *from_rank = from;
    return SPRS_B200_OK;
}

// every rank with send_mask bit set sends `my_fd` to every other rank; fds[g] receives rank
// g's descriptor (-1 where none is due); collective
int fd_exchange(sprs_b200_comm* c, int my_fd, uint32_t send_mask, int* fds) {
    for (int g = 0; g < c->world; ++g) fds[g] = -1;
    SPRS_TRY(sock_listen(c));
    SPRS_TRY(host_barrier(c));  // every rank listens
    if (send_mask & (1u << c->rank))
        for (int g = 0; g < c->world; ++g)
            if (g != c->rank && c->pid[g] != c->pid[c->rank]) SPRS_TRY(send_fd(c, g, my_fd));
    for (int g = 0; g < c->world; ++g) {
        if (g == c->rank || !(send_mask & (1u << g)) || c->pid[g] == c->pid[c->rank]) continue;
        int from = -1, fd = -1;
        SPRS_TRY(recv_fd(c, &from, &fd));
        if (from < 0 || from >= c->world || fds[from] != -1) {
            close(fd);
            SPRS_FAIL(c->ctx, SPRS_B200_ERR_COMM, "comm: unexpected descriptor from rank %d", from);
        }
        fds[from] = fd;
    }
    SPRS_TRY(host_barrier(c));
    return SPRS_B200_OK;
}

// ---- CUDA driver entry points (VMM + multicast), resolved through the runtime ----------
struct DriverApi {
    bool ok = false;
    CUresult (*DeviceGet)(CUdevice*, int) = nullptr;
    CUresult (*DeviceGetAttribute)(int*, CUdevice_attribute, CUdevice) = nullptr;
    CUresult (*MemCreate)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long) = nullptr;
    CUresult (*MemRelease)(CUmemGenericAllocationHandle) = nullptr;
    CUresult (*MemAddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
    CUresult (*MemAddressFree)(CUdeviceptr, size_t) = nullptr;
    CUresult (*MemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long) = nullptr;
    CUresult (*MemUnmap)(CUdeviceptr, size_t) = nullptr;
    CUresult (*MemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t) = nullptr;
    CUresult (*MemExport)(void*, CUmemGenericAllocationHandle, CUmemAllocationHandleType, unsigned long long) = nullptr;
    CUresult (*MemImport)(CUmemGenericAllocationHandle*, void*, CUmemAllocationHandleType) = nullptr;
    CUresult (*MemGetGranularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags) = nullptr;
    CUresult (*MulticastCreate)(CUmemGenericAllocationHandle*, const CUmulticastObjectProp*) = nullptr;
    CUresult (*MulticastAddDevice)(CUmemGenericAllocationHandle, CUdevice) = nullptr;
    CUresult (*MulticastBindMem)(CUmemGenericAllocationHandle, size_t, CUmemGenericAllocationHandle, size_t, size_t, unsigned long long) = nullptr;
    CUresult (*MulticastUnbind)(CUmemGenericAllocationHandle, CUdevice, size_t, size_t) = nullptr;
    CUresult (*MulticastGetGranularity)(size_t*, const CUmulticastObjectProp*, CUmulticastGranularity_flags) = nullptr;
    CUresult (*GetErrorString)(CUresult, const char**) = nullptr;
};

const DriverApi& driver() {
    static DriverApi api = [] {
        DriverApi a;
        bool ok = true;
        auto get = [&](const char* name, void** fn) {
            cudaDriverEntryPointQueryResult q;
            if (cudaGetDriverEntryPoint(name, fn, cudaEnableDefault, &q) != cudaSuccess ||
                q != cudaDriverEntryPointSuccess || !*fn) {
                cudaGetLastError();
                ok = false;
            }
        };
        get("cuDeviceGet", (void**)&a.DeviceGet);
        get("cuDeviceGetAttribute", (void**)&a.DeviceGetAttribute);
        get("cuMemCreate", (void**)&a.MemCreate);
        get("cuMemRelease", (void**)&a.MemRelease);
        get("cuMemAddressReserve", (void**)&a.MemAddressReserve);
        get("cuMemAddressFree", (void**)&a.MemAddressFree);
        get("cuMemMap", (void**)&a.MemMap);
        get("cuMemUnmap", (void**)&a.MemUnmap);
        get("cuMemSetAccess", (void**)&a.MemSetAccess);
        get("cuMemExportToShareableHandle", (void**)&a.MemExport);
        get("cuMemImportFromShareableHandle", (void**)&a.MemImport);
        get("cuMemGetAllocationGranularity", (void**)&a.MemGetGranularity);
        get("cuMulticastCreate", (void**)&a.MulticastCreate);
        get("cuMulticastAddDevice", (void**)&a.MulticastAddDevice);
        get("cuMulticastBindMem", (void**)&a.MulticastBindMem);
        get("cuMulticastUnbind", (void**)&a.MulticastUnbind);
        get("cuMulticastGetGranularity", (void**)&a.MulticastGetGranularity);
        get("cuGetErrorString", (void**)&a.GetErrorString);
        a.ok = ok;
        return a;
    }();
    return api;
}

#define SPRS_CU(ctx, expr)                                                                 \
    do {                                                                                   \
        CUresult _r = (expr);                                                              \
        if (_r != CUDA_SUCCESS) {                                                          \
            const char* _m = nullptr;                                                      \
            if (driver().GetErrorString) driver().GetErrorString(_r, &_m);                 \
            SPRS_FAIL((ctx), SPRS_B200_ERR_CUDA, "%s failed: %s (%s:%d)", #expr,           \
                      _m ? _m : "?", __FILE__, __LINE__);                                  \
        }                                                                                  \
    } while (0)

int device_multicast_supported(int device) {
    const DriverApi& d = driver();
    if (!d.ok) return 0;
    CUdevice dev;
    int v = 0;
    if (d.DeviceGet(&dev, device) != CUDA_SUCCESS) return 0;
    if (d.DeviceGetAttribute(&v, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, dev) != CUDA_SUCCESS) return 0;
    return v;
}

// ---- device barrier: every rank stores its epoch into a slot of every peer's flag array and
// waits until all of its own slots have reached the epoch.  Stream ordered: whatever the
// peers enqueued BEFORE their barrier (the stores of their y rows into this rank's buffers)
// has completed when this rank's barrier kernel returns.
struct BarrierArgs {
    unsigned long long* peer_flags[COMM_MAX_RANKS];  // flags array of rank g (g == rank: own)
    int rank, world;
    unsigned long long epoch;
    unsigned long long* err;
    long long timeout_cycles;
};

__global__ void comm_barrier_kernel(BarrierArgs a) {
    const int t = threadIdx.x;
    if (t >= a.world) return;
    __threadfence_system();
    unsigned long long* dst = a.peer_flags[t] + a.rank;
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(dst), "l"(a.epoch) : "memory");
    const unsigned long long* src = a.peer_flags[a.rank] + t;
    const long long start = clock64();
    unsigned backoff = 32;
    for (;;) {
        unsigned long long v;
        asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(src) : "memory");
        if (v >= a.epoch) break;
        __nanosleep(backoff);
        if (backoff < 1024) backoff <<= 1;
        if (clock64() - start > a.timeout_cycles) {  // a peer never arrived: report, do not hang
            atomicExch(a.err, 1ull);
            break;
        }
    }
}

int symm_free_impl(sprs_b200_symm* s);

int symm_alloc_ipc(sprs_b200_comm* c, uint64_t bytes, sprs_b200_symm* s) {
    sprs_b200_ctx* ctx = c->ctx;
    void* p = nullptr;
    SPRS_CUDA(ctx, cudaMalloc(&p, bytes ? bytes : 256));
    SPRS_CUDA(ctx, cudaMemset(p, 0, bytes ? bytes : 256));
    SPRS_CUDA(ctx, cudaDeviceSynchronize());
    s->ptr[c->rank] = p;
    struct Rec {
        cudaIpcMemHandle_t h;
        uint64_t raw;
    } mine{}, all[COMM_MAX_RANKS];
    mine.raw = (uint64_t)(uintptr_t)p;
    bool need_ipc = false;
    for (int g = 0; g < c->world; ++g) need_ipc |= c->pid[g] != c->pid[c->rank];
    if (need_ipc) SPRS_CUDA(ctx, cudaIpcGetMemHandle(&mine.h, p));
    SPRS_TRY(host_allgather(c, &mine, sizeof(mine), all));
    for (int g = 0; g < c->world; ++g) {
        if (g == c->rank) continue;
        if (c->pid[g] == c->pid[c->rank]) {  // ranks are threads of one process: direct access
            if (c->device[g] != c->device[c->rank]) {
                cudaError_t e = cudaDeviceEnablePeerAccess(c->device[g], 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled)
                    SPRS_FAIL(ctx, SPRS_B200_ERR_CUDA, "cudaDeviceEnablePeerAccess(%d): %s",
                              c->device[g], cudaGetErrorString(e));
                cudaGetLastError();
            }
            s->ptr[g] = (void*)(uintptr_t)all[g].raw;
        } else {
            SPRS_CUDA(ctx, cudaIpcOpenMemHandle(&s->ptr[g], all[g].h, cudaIpcMemLazyEnablePeerAccess));
            s->ipc_opened[g] = true;
        }
    }
    SPRS_TRY(host_barrier(c));
    return SPRS_B200_OK;
}

int symm_alloc_vmm(sprs_b200_comm* c, uint64_t bytes, sprs_b200_symm* s) {
    sprs_b200_ctx* ctx = c->ctx;
    const DriverApi& d = driver();
    CUdevice dev;
    SPRS_CU(ctx, d.DeviceGet(&dev, ctx->device));
    CUmulticastObjectProp mp{};
    mp.numDevices = (unsigned)c->world;
    mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    CUmemAllocationProp ap{};
    ap.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    ap.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    ap.location.id = ctx->device;
    ap.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    size_t g_mc = 0, g_mem = 0;
    mp.size = bytes ? bytes : 256;
    SPRS_CU(ctx, d.MulticastGetGranularity(&g_mc, &mp, CU_MULTICAST_GRANULARITY_RECOMMENDED));
    SPRS_CU(ctx, d.MemGetGranularity(&g_mem, &ap, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED));
    const size_t gran = g_mc > g_mem ? g_mc : g_mem;
    const size_t size = ((bytes ? bytes : 256) + gran - 1) / gran * gran;
    mp.size = size;
    s->map_bytes = size;
    // 1. the multicast object: created by rank 0, imported by the others
    int fds[COMM_MAX_RANKS];
    int mc_fd = -1;
    if (c->rank == 0) {
        SPRS_CU(ctx, d.MulticastCreate(&s->mc, &mp));
        SPRS_CU(ctx, d.MemExport(&mc_fd, s->mc, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
    }
    SPRS_TRY(fd_exchange(c, mc_fd, 1u, fds));
    if (c->rank == 0) {
        close(mc_fd);
    } else if (c->pid[0] != c->pid[c->rank]) {
        SPRS_CU(ctx, d.MemImport(&s->mc, (void*)(uintptr_t)fds[0], CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR));
        close(fds[0]);
    } else {
        SPRS_FAIL(ctx, SPRS_B200_ERR_UNSUPPORTED, "comm: multicast needs one process per rank");
    }
    SPRS_CU(ctx, d.MulticastAddDevice(s->mc, dev));
    SPRS_TRY(host_barrier(c));  // every device is in the team before anything is bound
    // 2. this rank's physical memory, bound into the object
    SPRS_CU(ctx, d.MemCreate(&s->mem[c->rank], size, &ap, 0));
    SPRS_CU(ctx, d.MulticastBindMem(s->mc, 0, s->mem[c->rank], 0, size, 0));
    // 3. everybody's memory mapped here (unicast), then the multicast address
    int my_fd = -1;
    SPRS_CU(ctx, d.MemExport(&my_fd, s->mem[c->rank], CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
    SPRS_TRY(fd_exchange(c, my_fd, (1u << c->world) - 1u, fds));
    close(my_fd);
    CUmemAccessDesc acc{};
    acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    acc.location.id = ctx->device;
    acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    for (int g = 0; g < c->world; ++g) {
        if (g != c->rank) {
            SPRS_CU(ctx, d.MemImport(&s->mem[g], (void*)(uintptr_t)fds[g], CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR));
            close(fds[g]);
        }
        CUdeviceptr va = 0;
        SPRS_CU(ctx, d.MemAddressReserve(&va, size, gran, 0, 0));
        SPRS_CU(ctx, d.MemMap(va, size, 0, s->mem[g], 0));
        SPRS_CU(ctx, d.MemSetAccess(va, size, &acc, 1));
        s->ptr[g] = (void*)va;
    }
    CUdeviceptr mva = 0;
    SPRS_CU(ctx, d.MemAddressReserve(&mva, size, gran, 0, 0));
    SPRS_CU(ctx, d.MemMap(mva, size, 0, s->mc, 0));
    SPRS_CU(ctx, d.MemSetAccess(mva, size, &acc, 1));
    s->mc_ptr = (void*)mva;
    s->vmm = true;
    SPRS_CUDA(ctx, cudaMemset(s->ptr[c->rank], 0, size));
    SPRS_CUDA(ctx, cudaDeviceSynchronize());
    SPRS_TRY(host_barrier(c));
    return SPRS_B200_OK;
}

int symm_free_impl(sprs_b200_symm* s) {
    sprs_b200_comm* c = s->comm;
    cudaSetDevice(c->ctx->device);
    cudaDeviceSynchronize();
    if (s->vmm) {
        const DriverApi& d = driver();
        if (s->mc_ptr) {
            d.MemUnmap((CUdeviceptr)s->mc_ptr, s->map_bytes);
            d.MemAddressFree((CUdeviceptr)s->mc_ptr, s->map_bytes);
        }
        for (int g = 0; g < c->world; ++g)
            if (s->ptr[g]) {
                d.MemUnmap((CUdeviceptr)s->ptr[g], s->map_bytes);
                d.MemAddressFree((CUdeviceptr)s->ptr[g], s->map_bytes);
            }
        CUdevice dev;
        if (s->mc && d.DeviceGet(&dev, c->ctx->device) == CUDA_SUCCESS)
            d.MulticastUnbind(s->mc, dev, 0, s->map_bytes);
        for (int g = 0; g < c->world; ++g)
            if (s->mem[g]) d.MemRelease(s->mem[g]);
        if (s->mc) d.MemRelease(s->mc);
    } else {
        for (int g = 0; g < c->world; ++g)
            if (g != c->rank && s->ipc_opened[g] && s->ptr[g]) cudaIpcCloseMemHandle(s->ptr[g]);
    }
    return SPRS_B200_OK;
}

}  // namespace

extern "C" {

int sprs_b200_comm_unique_id(char id[64]) {
    if (!id) return SPRS_B200_ERR_ARGUMENT;
    timespec ts;
    clock_gettime(CLOCK_REALTIME, &ts);
    uint64_t r = ((uint64_t)getpid() << 32) ^ (uint64_t)ts.tv_nsec ^ ((uint64_t)ts.tv_sec << 20);
    r += 0x9E3779B97F4A7C15ull;  // splitmix64 finaliser: spread the clock bits
    r = (r ^ (r >> 30)) * 0xBF58476D1CE4E5B9ull;
    r = (r ^ (r >> 27)) * 0x94D049BB133111EBull;
    r ^= r >> 31;
    static std::atomic<uint32_t> counter{0};
    memset(id, 0, 64);
    snprintf(id, 64, "%x-%llx-%x", (unsigned)getpid(), (unsigned long long)r, counter.fetch_add(1));
    return SPRS_B200_OK;
}

int sprs_b200_comm_init_rank(sprs_b200_ctx* ctx, const char id[64], int rank, int world,
                             sprs_b200_comm** out) {
    if (!ctx || !id || !out) return SPRS_B200_ERR_ARGUMENT;
    *out = nullptr;
    if (world < 1 || world > COMM_MAX_RANKS || rank < 0 || rank >= world)
        SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "comm: world must be 1..%d and 0 <= rank < world",
                  COMM_MAX_RANKS);
    if (memchr(id, 0, 64) == nullptr || id[0] == 0)
        SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "comm: id is not a NUL-terminated string");
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    auto* c = new sprs_b200_comm();
    c->ctx = ctx;
    c->rank = rank;
    c->world = world;
    memcpy(c->id, id, 64);
    if (const char* e = getenv("SPRS_B200_COMM_TIMEOUT_S")) c->timeout_s = atof(e) > 0 ? atof(e) : c->timeout_s;
    int st = SPRS_B200_OK;
    do {
        if (world > 1) {
            const std::string name = shm_name(id);
            int fd = -1;
            if (rank == 0) {
                fd = shm_open(name.c_str(), O_CREAT | O_EXCL | O_RDWR, 0600);
                if (fd < 0 || ftruncate(fd, sizeof(CommShm)) != 0) {
                    sprs_b200_set_error(ctx, (std::string("comm: shm_open/ftruncate: ") + strerror(errno)).c_str());
                    if (fd >= 0) close(fd);
                    st = SPRS_B200_ERR_COMM;
                    break;
                }
            } else {
                const double t0 = now_s();
                while ((fd = shm_open(name.c_str(), O_RDWR, 0600)) < 0) {
                    if (now_s() - t0 > c->timeout_s) break;
                    std::this_thread::sleep_for(std::chrono::milliseconds(2));
                }
                if (fd >= 0) {  // wait until rank 0 has sized it
                    struct stat sb;
                    while (fstat(fd, &sb) == 0 && (size_t)sb.st_size < sizeof(CommShm) &&
                           now_s() - t0 <= c->timeout_s)
                        std::this_thread::sleep_for(std::chrono::milliseconds(1));
                }
                if (fd < 0) {
                    sprs_b200_set_error(ctx, "comm: rank 0's rendezvous segment never appeared");
                    st = SPRS_B200_ERR_COMM;
                    break;
                }
            }
            void* p = mmap(nullptr, sizeof(CommShm), PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
            close(fd);
            if (p == MAP_FAILED) {
                sprs_b200_set_error(ctx, "comm: mmap of the rendezvous segment failed");
                st = SPRS_B200_ERR_COMM;
                break;
            }
            c->shm = (CommShm*)p;
            if (rank == 0) {  // fresh segments are zero-filled; publish last
                c->shm->world = (uint32_t)world;
                c->shm->magic.store(COMM_MAGIC, std::memory_order_release);
            } else {
                const double t0 = now_s();
                while (c->shm->magic.load(std::memory_order_acquire) != COMM_MAGIC) {
                    if (now_s() - t0 > c->timeout_s) break;
                    std::this_thread::sleep_for(std::chrono::milliseconds(1));
                }
                if (c->shm->magic.load() != COMM_MAGIC || c->shm->world != (uint32_t)world) {
                    sprs_b200_set_error(ctx, "comm: rendezvous segment not initialised / world mismatch");
                    st = SPRS_B200_ERR_COMM;
                    break;
                }
            }
        }
        struct Hello {
            int pid, device, mc;
        } mine{(int)getpid(), ctx->device, device_multicast_supported(ctx->device)}, all[COMM_MAX_RANKS];
        if ((st = host_allgather(c, &mine, sizeof(mine), all)) != SPRS_B200_OK) break;
        if (world > 1 && rank == 0) shm_unlink(shm_name(id).c_str());  // everyone is attached
        int mc = world > 1 ? 1 : 0;
        for (int g = 0; g < world; ++g) {
            c->pid[g] = all[g].pid;
            c->device[g] = all[g].device;
            mc &= all[g].mc;
            for (int h = 0; h < g; ++h)
                if (all[h].device == all[g].device || all[h].pid == all[g].pid) mc = 0;
        }
        if (const char* e = getenv("SPRS_B200_COMM_MULTICAST")) mc &= atoi(e) != 0;
        c->multicast_ok = mc;
        // device barrier state
        cudaError_t e = cudaMalloc((void**)&c->d_err, 8);
        if (e == cudaSuccess) e = cudaMemset(c->d_err, 0, 8);
        if (e != cudaSuccess) {
            sprs_b200_set_error(ctx, cudaGetErrorString(e));
            st = SPRS_B200_ERR_CUDA;
            break;
        }
        c->flags = new sprs_b200_symm();
        c->flags->comm = c;
        c->flags->bytes = COMM_MAX_RANKS * 8;
        if ((st = symm_alloc_ipc(c, c->flags->bytes, c->flags)) != SPRS_B200_OK) break;
    } while (0);
    if (st != SPRS_B200_OK) {
        if (c->shm) c->shm->failed.store(1);
        return st;  // the handle is leaked on purpose: peers may still be mapped into it
    }
    *out = c;
    return SPRS_B200_OK;
}

int sprs_b200_comm_free(sprs_b200_comm* c) {
    if (!c) return SPRS_B200_OK;
    cudaSetDevice(c->ctx->device);
    cudaDeviceSynchronize();
    if (c->world > 1 && c->shm && !c->shm->failed.load()) host_barrier(c);  // nobody unmaps early
    if (c->flags) {
        symm_free_impl(c->flags);
        if (c->flags->ptr[c->rank]) cudaFree(c->flags->ptr[c->rank]);
        delete c->flags;
    }
    if (c->d_err) cudaFree(c->d_err);
    if (c->listen_fd >= 0) close(c->listen_fd);
    if (c->shm) munmap(c->shm, sizeof(CommShm));
    delete c;
    return SPRS_B200_OK;
}

int sprs_b200_comm_rank(const sprs_b200_comm* c) { return c ? c->rank : -1; }
int sprs_b200_comm_world(const sprs_b200_comm* c) { return c ? c->world : 0; }
int sprs_b200_comm_multicast_supported(const sprs_b200_comm* c) { return c ? c->multicast_ok : 0; }

int sprs_b200_comm_allgather_host(sprs_b200_comm* c, const void* mine, uint64_t bytes, void* all) {
    if (!c || !mine || !all) return SPRS_B200_ERR_ARGUMENT;
    return host_allgather(c, mine, (size_t)bytes, all);
}

int sprs_b200_comm_barrier_host(sprs_b200_comm* c) {
    if (!c) return SPRS_B200_ERR_ARGUMENT;
    return host_barrier(c);
}

int sprs_b200_comm_barrier_dev(sprs_b200_comm* c, void* stream) {
    if (!c) return SPRS_B200_ERR_ARGUMENT;
    if (c->world == 1) return SPRS_B200_OK;
    BarrierArgs a{};
    for (int g = 0; g < c->world; ++g) a.peer_flags[g] = (unsigned long long*)c->flags->ptr[g];
    a.rank = c->rank;
    a.world = c->world;
    a.epoch = ++c->epoch;
    a.err = c->d_err;
    a.timeout_cycles = (long long)(c->timeout_s * 1.9e9);
    comm_barrier_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(a);
    c->ctx->launches += 1;
    SPRS_CUDA(c->ctx, cudaGetLastError());
    return SPRS_B200_OK;
}

int sprs_b200_comm_check(sprs_b200_comm* c, void* stream) {
    if (!c) return SPRS_B200_ERR_ARGUMENT;
    unsigned long long err = 0;
    SPRS_CUDA(c->ctx, cudaMemcpyAsync(&err, c->d_err, 8, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    SPRS_CUDA(c->ctx, cudaStreamSynchronize((cudaStream_t)stream));
    if (err) SPRS_FAIL(c->ctx, SPRS_B200_ERR_COMM, "comm: a device barrier timed out (a peer never arrived)");
    return SPRS_B200_OK;
}

int sprs_b200_symm_alloc(sprs_b200_comm* c, uint64_t bytes, int want_multicast,
                         sprs_b200_symm** out) {
    if (!c || !out) return SPRS_B200_ERR_ARGUMENT;
    *out = nullptr;
    SPRS_CUDA(c->ctx, cudaSetDevice(c->ctx->device));
    auto* s = new sprs_b200_symm();
    s->comm = c;
    s->bytes = bytes;
    int st;
    if (want_multicast && c->multicast_ok)
        st = symm_alloc_vmm(c, bytes, s);
    else
        st = symm_alloc_ipc(c, bytes, s);
    if (st != SPRS_B200_OK) {
        if (c->shm) c->shm->failed.store(1);
        return st;
    }
    *out = s;
    return SPRS_B200_OK;
}

void* sprs_b200_symm_ptr(const sprs_b200_symm* s, int rank) {
    return (s && rank >= 0 && rank < s->comm->world) ? s->ptr[rank] : nullptr;
}
void* sprs_b200_symm_multicast_ptr(const sprs_b200_symm* s) { return s ? s->mc_ptr : nullptr; }
uint64_t sprs_b200_symm_bytes(const sprs_b200_symm* s) { return s ? s->bytes : 0; }

int sprs_b200_symm_free(sprs_b200_symm* s) {
    if (!s) return SPRS_B200_OK;
    sprs_b200_comm* c = s->comm;
    cudaSetDevice(c->ctx->device);
    cudaDeviceSynchronize();
    if (c->world > 1 && c->shm && !c->shm->failed.load()) host_barrier(c);  // peers have stopped storing
    symm_free_impl(s);
    if (!s->vmm && s->ptr[c->rank]) cudaFree(s->ptr[c->rank]);
    delete s;
    return SPRS_B200_OK;
}

// slice_outer cut points (slicing.rs:65-89) balanced on cost(rows [a,b)) = nnz + row_cost*rows
int sprs_b200_partition_rows(const void* indptr, int indptr_bytes, uint64_t rows, int nparts,
                             double row_cost, uint64_t* bounds) {
    if (!indptr || !bounds || nparts < 1 || (indptr_bytes != 4 && indptr_bytes != 8))
        return SPRS_B200_ERR_ARGUMENT;
    auto ip = [&](uint64_t r) -> uint64_t {
        return indptr_bytes == 4 ? (uint64_t)((const uint32_t*)indptr)[r] : ((const uint64_t*)indptr)[r];
    };
    const uint64_t base = ip(0);
    if (row_cost < 0) row_cost = 0;
    auto cost = [&](uint64_t r) -> double { return (double)(ip(r) - base) + row_cost * (double)r; };
    const double total = cost(rows);
    bounds[0] = 0;
    for (int g = 1; g < nparts; ++g) {
        const double target = total * g / nparts;
        uint64_t lo = 0, hi = rows;  // first r with cost(r) >= target
        while (lo < hi) {
            const uint64_t mid = lo + (hi - lo) / 2;
            if (cost(mid) >= target)
                hi = mid;
            else
                lo = mid + 1;
        }
        bounds[g] = lo < bounds[g - 1] ? bounds[g - 1] : lo;
    }
    bounds[nparts] = rows;
    return SPRS_B200_OK;
}

// ---- row-partitioned SpMV: y[row_offset .. row_offset + rows_local) = A_local x on this rank,
// all-gathered into EVERY rank's y (a symmetric buffer of n doubles) and followed by the device
// barrier, all on `stream`: when the call's work has completed on a rank, that rank's y holds
// the full product.  `exchange` picks how the rows travel (see sprs_b200.h).
int sprs_b200_spmv_rowpart(sprs_b200_comm* c, const sprs_b200_csmat* mat, const double* d_x,
                           sprs_b200_symm* y, uint64_t row_offset, int exchange, void* stream) {
    if (!c || !mat || !y) return SPRS_B200_ERR_ARGUMENT;
    sprs_b200_ctx* ctx = c->ctx;
    if ((row_offset + mat->rows) * 8 > y->bytes)
        SPRS_FAIL(ctx, SPRS_B200_ERR_DIMENSION, "Dimension mismatch: row block exceeds y");
    cudaStream_t s = (cudaStream_t)stream;
    const bool mc = y->mc_ptr != nullptr;
    const bool no_barrier = (exchange & SPRS_B200_EXCHANGE_NO_BARRIER) != 0;
    exchange &= ~SPRS_B200_EXCHANGE_NO_BARRIER;
    if (exchange == SPRS_B200_EXCHANGE_AUTO)  // tools/scale_modes.py times every mode
        exchange = SPRS_B200_EXCHANGE_FUSED;
    SpmvTargets yt;
    yt.n = 1;
    for (int q = 0; q < SPMV_MAX_TARGETS; ++q) yt.p[q] = nullptr;
    double* own = (double*)y->ptr[c->rank] + row_offset;
    yt.p[0] = own;
    SpmvTargets remote;  // where the rows go besides the local y
    remote.n = 0;
    for (int q = 0; q < SPMV_MAX_TARGETS; ++q) remote.p[q] = nullptr;
    if (c->world > 1) {
        if (mc) {
            remote.p[remote.n++] = (double*)y->mc_ptr + row_offset;  // the switch replicates
        } else {
            for (int g = 0; g < c->world; ++g)
                if (g != c->rank) {
                    if (remote.n >= SPMV_MAX_TARGETS - 1)
                        SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "comm: too many peers");
                    remote.p[remote.n++] = (double*)y->ptr[g] + row_offset;
                }
        }
    }
    if (exchange == SPRS_B200_EXCHANGE_FUSED) {
        for (int q = 0; q < remote.n; ++q) yt.p[yt.n++] = remote.p[q];
        SPRS_TRY(spmv_launch_targets(ctx, mat, d_x, yt, 0, s));
    } else if (exchange == SPRS_B200_EXCHANGE_PUSH) {
        SPRS_TRY(spmv_launch_targets(ctx, mat, d_x, yt, 0, s));
        if (remote.n) SPRS_TRY(peer_push_launch(ctx, own, remote, mat->rows, s));
    } else {
        SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "comm: unknown exchange mode %d", exchange);
    }
    return no_barrier ? SPRS_B200_OK : sprs_b200_comm_barrier_dev(c, stream);
}

// `&A * &x` on a row-partitioned matrix with HOST vectors, every rank handling only its own
// slices: x_slice (x[col_offset .. col_offset+col_count)) is uploaded into this rank's part of
// the symmetric x buffer and pushed to the peers (all-gather of x over NVLink), then the local
// block is multiplied and y_slice (this rank's rows) downloaded.  Blocking, like the operator.
int sprs_b200_mul_mat_vec_rowpart(sprs_b200_comm* c, const sprs_b200_csmat* mat,
                                  sprs_b200_symm* x, const double* x_slice, uint64_t col_offset,
                                  uint64_t col_count, double* y_slice, uint64_t y_len) {
    if (!c || !mat || !x || (col_count && !x_slice) || (y_len && !y_slice))
        return SPRS_B200_ERR_ARGUMENT;
    sprs_b200_ctx* ctx = c->ctx;
    if (mat->storage != SPRS_B200_CSR)
        SPRS_FAIL(ctx, SPRS_B200_ERR_STORAGE, "Storage mismatch: spmv needs a CSR mirror");
    if (y_len != mat->rows || (col_offset + col_count) > mat->cols || mat->cols * 8 > x->bytes)
        SPRS_FAIL(ctx, SPRS_B200_ERR_DIMENSION, "Dimension mismatch");
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    double* x_own = (double*)x->ptr[c->rank];
    if (col_count)
        SPRS_CUDA(ctx, cudaMemcpyAsync(x_own + col_offset, x_slice, col_count * 8,
                                       cudaMemcpyHostToDevice, s));
    if (c->world > 1) {
        SpmvTargets remote;
        remote.n = 0;
        for (int q = 0; q < SPMV_MAX_TARGETS; ++q) remote.p[q] = nullptr;
        if (x->mc_ptr) {
            remote.p[remote.n++] = (double*)x->mc_ptr + col_offset;
        } else {
            for (int g = 0; g < c->world; ++g)
                if (g != c->rank) remote.p[remote.n++] = (double*)x->ptr[g] + col_offset;
        }
        if (col_count) SPRS_TRY(peer_push_launch(ctx, x_own + col_offset, remote, col_count, s));
        SPRS_TRY(sprs_b200_comm_barrier_dev(c, s));  // every slice of x has landed here
    }
    void* d_y = nullptr;
    SPRS_TRY(ctx_scratch(ctx, 1, (mat->rows ? mat->rows : 1) * 8, &d_y));
    SPRS_TRY(spmv_launch(ctx, mat, x_own, (double*)d_y, 0, s));
    if (y_len)
        SPRS_CUDA(ctx, cudaMemcpyAsync(y_slice, d_y, y_len * 8, cudaMemcpyDeviceToHost, s));
    if (c->world > 1)  // nobody overwrites x for the next call while a peer still gathers from it
        SPRS_TRY(sprs_b200_comm_barrier_dev(c, s));
    SPRS_CUDA(ctx, cudaStreamSynchronize(s));
    return SPRS_B200_OK;
}

}  // extern "C"
