// peer.cu -- multi-GPU plumbing of the row-partitioned SpMV (one process per GPU).
//
// The reference has no multi-device code (SURVEY 2.4); the natural sharding primitive is
// slice_outer (slicing.rs:65-89).  Each rank owns a contiguous row block of A, x is
// replicated, and the single exchange step is an all-gather of y.  Here the all-gather is
// FUSED into the SpMV kernel: every rank maps the other ranks' y buffers through CUDA IPC
// (NVLink/NVSwitch peer access) and the kernel stores each finished row into all of them,
// so the transfer overlaps the rest of the compute; only a stream-ordered barrier remains.
#include <algorithm>
#include <cstdlib>

#include "common.cuh"

namespace {
// Push `count` doubles from this GPU's y into the same position of every target buffer (the
// all-gather "put"): peer mappings over NVLink, or ONE NVSwitch multicast address the switch
// replicates.  16-byte loads and stores on the aligned body (all buffers share the alignment of
// their common row offset), scalar head / tail.
__global__ void __launch_bounds__(256)
    peer_push_kernel(const double* __restrict__ src, SpmvTargets dst, uint64_t count) {
    const uint64_t head = (((uintptr_t)src & 15) && count) ? 1 : 0;  // 8-byte aligned, not 16
    const uint64_t pairs = (count - head) / 2;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const uint64_t tid = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    const double2* s2 = (const double2*)(src + head);
    for (uint64_t i = tid; i < pairs; i += 4 * stride) {
        double2 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u)
            v[u] = (i + u * stride < pairs) ? s2[i + u * stride] : make_double2(0.0, 0.0);
#pragma unroll
        for (int q = 0; q < SPMV_MAX_TARGETS; ++q)
            if (q < dst.n) {
                double2* d2 = (double2*)(dst.p[q] + head);
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    if (i + u * stride < pairs) d2[i + u * stride] = v[u];
            }
    }
    if (tid == 0) {
        if (head)
            for (int q = 0; q < dst.n; ++q) dst.p[q][0] = src[0];
        if ((count - head) & 1)
            for (int q = 0; q < dst.n; ++q) dst.p[q][count - 1] = src[count - 1];
    }
}

// The put kernel takes its scalar head from the source address alone and stores double2 through
// every target, so each target must be non-null and share the source's 16-byte parity.
int check_push_targets(sprs_b200_ctx* ctx, const double* src, const SpmvTargets& dst) {
    for (int q = 0; q < dst.n; ++q) {
        if (!dst.p[q]) SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "peer push: target %d is null", q);
        if ((((uintptr_t)dst.p[q]) & 15) != (((uintptr_t)src) & 15))
            SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "peer push: buffers must share their 16-byte alignment");
    }
    return SPRS_B200_OK;
}

// dst = bufs[0 .. n) + offset, checked against the put's source `src` (the same offset into the
// rank's own buffer).  A null buffer is caught before the offset makes it look valid.
int push_targets(sprs_b200_ctx* ctx, const double* src, double* const* bufs, int n, uint64_t offset,
                 SpmvTargets* dst) {
    dst->n = n;
    for (int q = 0; q < SPMV_MAX_TARGETS; ++q) {
        if (q < n && !bufs[q]) SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "peer push: target %d is null", q);
        dst->p[q] = q < n ? bufs[q] + offset : nullptr;
    }
    return check_push_targets(ctx, src, *dst);
}
}  // namespace

int peer_push_launch(sprs_b200_ctx* ctx, const double* src, const SpmvTargets& dst, uint64_t count,
                     cudaStream_t s) {
    if (dst.n == 0) return SPRS_B200_OK;
    SPRS_TRY(check_push_targets(ctx, src, dst));
    if (count == 0) return SPRS_B200_OK;
    uint64_t blocks = (count / 2 + 1023) / 1024;
    if (blocks == 0) blocks = 1;
    const uint64_t cap = (uint64_t)ctx->sm_count * 2;
    if (blocks > cap) blocks = cap;
    peer_push_kernel<<<(unsigned)blocks, 256, 0, s>>>(src, dst, count);
    ctx->launches += 1;
    SPRS_CUDA(ctx, cudaGetLastError());
    return SPRS_B200_OK;
}

extern "C" {

int sprs_b200_peer_push_dev(sprs_b200_ctx* ctx, const double* d_y_own, uint64_t row_offset,
                            uint64_t rows, int n_peers, double* const* d_y_peers, void* stream) {
    if (!ctx || !d_y_own || (n_peers && !d_y_peers)) return SPRS_B200_ERR_ARGUMENT;
    if (n_peers < 0 || n_peers > SPMV_MAX_TARGETS)
        SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "n_peers must be 0..%d", SPMV_MAX_TARGETS);
    SpmvTargets dst;
    SPRS_TRY(push_targets(ctx, d_y_own + row_offset, d_y_peers, n_peers, row_offset, &dst));
    return peer_push_launch(ctx, d_y_own + row_offset, dst, rows, (cudaStream_t)stream);
}

int sprs_b200_peer_alloc(sprs_b200_ctx* ctx, uint64_t bytes, void** d_ptr,
                         unsigned char ipc_handle[64]) {
    if (!ctx || !d_ptr || !ipc_handle) return SPRS_B200_ERR_ARGUMENT;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handles are 64 bytes");
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    void* p = nullptr;
    SPRS_CUDA(ctx, cudaMalloc(&p, bytes ? bytes : 16));
    cudaIpcMemHandle_t h;
    cudaError_t e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess) {
        cudaFree(p);
        SPRS_FAIL(ctx, SPRS_B200_ERR_CUDA, "cudaIpcGetMemHandle: %s", cudaGetErrorString(e));
    }
    memcpy(ipc_handle, &h, 64);
    *d_ptr = p;
    return SPRS_B200_OK;
}

int sprs_b200_peer_open(sprs_b200_ctx* ctx, const unsigned char ipc_handle[64], void** d_ptr) {
    if (!ctx || !d_ptr || !ipc_handle) return SPRS_B200_ERR_ARGUMENT;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaIpcMemHandle_t h;
    memcpy(&h, ipc_handle, 64);
    SPRS_CUDA(ctx, cudaIpcOpenMemHandle(d_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return SPRS_B200_OK;
}

int sprs_b200_peer_close(sprs_b200_ctx* ctx, void* d_ptr) {
    if (!ctx) return SPRS_B200_ERR_ARGUMENT;
    if (d_ptr) SPRS_CUDA(ctx, cudaIpcCloseMemHandle(d_ptr));
    return SPRS_B200_OK;
}

int sprs_b200_peer_free(sprs_b200_ctx* ctx, void* d_ptr) {
    if (!ctx) return SPRS_B200_ERR_ARGUMENT;
    if (d_ptr) SPRS_CUDA(ctx, cudaFree(d_ptr));
    return SPRS_B200_OK;
}

int sprs_b200_copy_dev(sprs_b200_ctx* ctx, void* dst, const void* src, uint64_t bytes,
                       void* stream) {
    if (!ctx || (bytes && (!dst || !src))) return SPRS_B200_ERR_ARGUMENT;
    SPRS_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice,
                                   (cudaStream_t)stream));
    return SPRS_B200_OK;
}

int sprs_b200_copy_to_device(sprs_b200_ctx* ctx, void* d_dst, const void* h_src, uint64_t bytes,
                             void* stream) {
    if (!ctx || (bytes && (!d_dst || !h_src))) return SPRS_B200_ERR_ARGUMENT;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    SPRS_CUDA(ctx, cudaMemcpyAsync(d_dst, h_src, bytes, cudaMemcpyHostToDevice, (cudaStream_t)stream));
    SPRS_CUDA(ctx, cudaStreamSynchronize((cudaStream_t)stream));
    return SPRS_B200_OK;
}

int sprs_b200_copy_to_host(sprs_b200_ctx* ctx, void* h_dst, const void* d_src, uint64_t bytes,
                           void* stream) {
    if (!ctx || (bytes && (!h_dst || !d_src))) return SPRS_B200_ERR_ARGUMENT;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    SPRS_CUDA(ctx, cudaMemcpyAsync(h_dst, d_src, bytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    SPRS_CUDA(ctx, cudaStreamSynchronize((cudaStream_t)stream));
    return SPRS_B200_OK;
}

int sprs_b200_spmv_allgather_dev(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat,
                                 const double* d_x, uint64_t row_offset, int n_targets,
                                 double* const* d_y_bufs, int accumulate, void* stream) {
    if (!ctx || !mat || !d_y_bufs) return SPRS_B200_ERR_ARGUMENT;
    if (n_targets < 1 || n_targets > SPMV_MAX_TARGETS)
        SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "n_targets must be 1..%d", SPMV_MAX_TARGETS);
    SpmvTargets yt;
    yt.n = n_targets;
    for (int q = 0; q < SPMV_MAX_TARGETS; ++q)
        yt.p[q] = q < n_targets ? d_y_bufs[q] + row_offset : nullptr;
    return spmv_launch_targets(ctx, mat, d_x, yt, accumulate, (cudaStream_t)stream);
}

// Pipelined all-gather without any kernel waiting on another (plan B of the stream push): the
// rank's tile stream is launched in a few chunks of decreasing size; behind each chunk's event
// the side stream runs a put kernel that copies the rows that chunk completed into the peer
// buffers while the next chunk computes.  Only the put of the (small) last chunk is exposed.
int sprs_b200_spmv_chunked_push_dev(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat,
                                    const double* d_x, uint64_t row_offset, int n_targets,
                                    double* const* d_y_bufs, int accumulate, int n_chunks,
                                    void* stream) {
    if (!ctx || !mat || !d_y_bufs) return SPRS_B200_ERR_ARGUMENT;
    if (n_targets < 1 || n_targets > SPMV_MAX_TARGETS)
        SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "n_targets must be 1..%d", SPMV_MAX_TARGETS);
    if (!d_y_bufs[0]) SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "d_y_bufs[0] is null");
    double* y_own = d_y_bufs[0] + row_offset;
    // every put of the chunks below reads y_own + r0 and stores to d_y_bufs[q] + row_offset + r0:
    // one check of the targets at r0 = 0 covers all of them
    SpmvTargets dst;
    SPRS_TRY(push_targets(ctx, y_own, d_y_bufs + 1, n_targets - 1, row_offset, &dst));
    if (mat->storage != SPRS_B200_CSR)
        SPRS_FAIL(ctx, SPRS_B200_ERR_STORAGE, "Storage mismatch: spmv needs a CSR mirror");
    if (mat->rows == 0) return SPRS_B200_OK;
    cudaStream_t s = (cudaStream_t)stream;
    if (n_chunks <= 0) n_chunks = 4;
    if (const char* e = getenv("SPRS_B200_PUSH_CHUNKS")) n_chunks = atoi(e) > 0 ? atoi(e) : n_chunks;
    if (n_chunks > SPRS_E2E_MAX_CHUNKS) n_chunks = SPRS_E2E_MAX_CHUNKS;
    if (mat->push_tiles.empty() || (int)mat->push_tiles.size() - 1 != std::min<int>(n_chunks, (int)mat->n_tiles)) {
        std::vector<uint64_t> tiles, rows;
        SPRS_TRY(csmat_chunk_table(ctx, mat, (uint64_t)n_chunks, true, s, &tiles, &rows));
        mat->push_tiles = tiles;
        mat->push_rows = rows;
    }
    SPRS_TRY(ctx_side_stream(ctx));
    if (!ctx->ev_chunk[0])
        for (int i = 0; i < SPRS_E2E_MAX_CHUNKS; ++i)
            SPRS_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_chunk[i], cudaEventDisableTiming));
    const size_t nc = mat->push_tiles.size() - 1;
    for (size_t c = 0; c < nc; ++c) {
        SPRS_TRY(spmv_launch_tile_range(ctx, mat, d_x, y_own, accumulate, mat->push_tiles[c],
                                        mat->push_tiles[c + 1], s));
        if (n_targets == 1) continue;
        const uint64_t r0 = mat->push_rows[c], r1 = mat->push_rows[c + 1];
        SPRS_CUDA(ctx, cudaEventRecord(ctx->ev_chunk[c], s));
        SPRS_CUDA(ctx, cudaStreamWaitEvent(ctx->side_stream, ctx->ev_chunk[c], 0));
        if (r1 == r0) continue;
        for (int q = 0; q < dst.n; ++q) dst.p[q] = d_y_bufs[q + 1] + row_offset + r0;
        uint64_t blocks = (r1 - r0 + 1023) / 1024;
        const uint64_t cap = (uint64_t)ctx->sm_count / 4;  // a few SMs' worth: the next chunk computes
        if (blocks > cap) blocks = cap;
        peer_push_kernel<<<(unsigned)blocks, 256, 0, ctx->side_stream>>>(y_own + r0, dst, r1 - r0);
        ctx->launches += 1;
        SPRS_CUDA(ctx, cudaGetLastError());
    }
    if (n_targets > 1) {
        SPRS_CUDA(ctx, cudaEventRecord(ctx->ev_join, ctx->side_stream));
        SPRS_CUDA(ctx, cudaStreamWaitEvent(s, ctx->ev_join, 0));
    }
    return SPRS_B200_OK;
}

}  // extern "C"
