// api.cu -- the extern "C" surface declared in include/sprs_b200.h: context, device
// mirrors of CsMatBase, and the host-buffer entry points that mirror the reference's
// free functions (sprs/src/sparse/prod.rs).  Shape / storage checks happen here,
// before any device work, exactly where the reference asserts (prod.rs:114-118,
// 198-201, 283-286).  There is no CPU implementation behind any of these calls.

#include <algorithm>
#include <mutex>
#include <vector>

#include <cstdlib>

#include "common.cuh"
#include "ptx.cuh"

namespace {

__global__ void make_policies_kernel(uint64_t* out) {
    out[0] = policy_evict_first();
    out[1] = policy_evict_last();
}

thread_local std::string g_create_error;

template <typename Src, typename Dst>
__global__ void convert_rebase_kernel(const Src* __restrict__ in, Dst* __restrict__ out,
                                      uint64_t n, uint64_t base) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n) out[i] = (Dst)((uint64_t)in[i] - base);
}

inline unsigned grid_for(uint64_t n) { return (unsigned)((n + 255) / 256); }

template <typename P>
__global__ void check_structure_kernel(const P* __restrict__ indptr,
                                       const uint32_t* __restrict__ indices, uint64_t outer,
                                       uint64_t inner, unsigned long long* __restrict__ bad) {
    const int lane = threadIdx.x & 31;
    const uint64_t w0 = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
    const uint64_t nw = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t r = w0; r < outer; r += nw) {  // one warp per outer dimension
        const uint64_t s = indptr[r], e = indptr[r + 1];
        bool viol = e < s;
        if (!viol)
            for (uint64_t k = s + lane; k < e; k += 32) {
                const uint32_t c = indices[k];
                if (c >= inner || (k > s && indices[k - 1] >= c)) viol = true;
            }
        if (__any_sync(0xffffffffu, viol) && lane == 0) atomicAdd(bad, 1ull);
    }
}

int upload_indexlike(sprs_b200_ctx* ctx, const void* host, int host_bytes, uint64_t n,
                     uint64_t base, void* d_out, int dev_bytes, cudaStream_t s) {
    if (n == 0) return SPRS_B200_OK;
    if (host_bytes == dev_bytes && base == 0) {
        SPRS_CUDA(ctx, cudaMemcpyAsync(d_out, host, n * (size_t)dev_bytes,
                                       cudaMemcpyHostToDevice, s));
        return SPRS_B200_OK;
    }
    void* d_raw = nullptr;
    SPRS_TRY(ctx_scratch(ctx, 0, n * (size_t)host_bytes, &d_raw));
    SPRS_CUDA(ctx, cudaMemcpyAsync(d_raw, host, n * (size_t)host_bytes, cudaMemcpyHostToDevice, s));
    const unsigned g = grid_for(n);
    if (host_bytes == 4 && dev_bytes == 4)
        convert_rebase_kernel<uint32_t, uint32_t><<<g, 256, 0, s>>>((const uint32_t*)d_raw,
                                                                    (uint32_t*)d_out, n, base);
    else if (host_bytes == 8 && dev_bytes == 4)
        convert_rebase_kernel<uint64_t, uint32_t><<<g, 256, 0, s>>>((const uint64_t*)d_raw,
                                                                    (uint32_t*)d_out, n, base);
    else if (host_bytes == 4 && dev_bytes == 8)
        convert_rebase_kernel<uint32_t, uint64_t><<<g, 256, 0, s>>>((const uint32_t*)d_raw,
                                                                    (uint64_t*)d_out, n, base);
    else
        convert_rebase_kernel<uint64_t, uint64_t><<<g, 256, 0, s>>>((const uint64_t*)d_raw,
                                                                    (uint64_t*)d_out, n, base);
    ctx->launches += 1;
    SPRS_CUDA(ctx, cudaGetLastError());
    SPRS_CUDA(ctx, cudaStreamSynchronize(s));  // scratch slot 0 is reused by the next call
    return SPRS_B200_OK;
}

int download_indexlike(sprs_b200_ctx* ctx, const void* d_in, int dev_bytes, uint64_t n,
                       void* host, int host_bytes, cudaStream_t s) {
    if (n == 0) return SPRS_B200_OK;
    if (host_bytes == dev_bytes) {
        SPRS_CUDA(ctx, cudaMemcpyAsync(host, d_in, n * (size_t)dev_bytes, cudaMemcpyDeviceToHost, s));
        SPRS_CUDA(ctx, cudaStreamSynchronize(s));
        return SPRS_B200_OK;
    }
    void* d_tmp = nullptr;
    SPRS_TRY(ctx_scratch(ctx, 0, n * (size_t)host_bytes, &d_tmp));
    const unsigned g = grid_for(n);
    if (dev_bytes == 4 && host_bytes == 8)
        convert_rebase_kernel<uint32_t, uint64_t><<<g, 256, 0, s>>>((const uint32_t*)d_in,
                                                                    (uint64_t*)d_tmp, n, 0);
    else
        convert_rebase_kernel<uint64_t, uint32_t><<<g, 256, 0, s>>>((const uint64_t*)d_in,
                                                                    (uint32_t*)d_tmp, n, 0);
    ctx->launches += 1;
    SPRS_CUDA(ctx, cudaGetLastError());
    SPRS_CUDA(ctx, cudaMemcpyAsync(host, d_tmp, n * (size_t)host_bytes, cudaMemcpyDeviceToHost, s));
    SPRS_CUDA(ctx, cudaStreamSynchronize(s));
    return SPRS_B200_OK;
}

uint64_t read_index(const void* p, int bytes, uint64_t i) {
    return bytes == 4 ? (uint64_t)((const uint32_t*)p)[i] : ((const uint64_t*)p)[i];
}

}  // namespace

void sprs_b200_set_error(const sprs_b200_ctx* ctx, const char* msg) {
    if (ctx)
        const_cast<sprs_b200_ctx*>(ctx)->last_error = msg;
    else
        g_create_error = msg;
}

int ctx_scratch(sprs_b200_ctx* ctx, int i, size_t bytes, void** out) {
    if (bytes < 256) bytes = 256;
    if (ctx->d_scratch_bytes[i] < bytes) {
        if (ctx->d_scratch[i]) {
            SPRS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            SPRS_CUDA(ctx, cudaFree(ctx->d_scratch[i]));
            ctx->d_scratch[i] = nullptr;
            ctx->d_scratch_bytes[i] = 0;
        }
        const size_t want = bytes + bytes / 4;
        SPRS_CUDA(ctx, cudaMalloc(&ctx->d_scratch[i], want));
        ctx->d_scratch_bytes[i] = want;
    }
    *out = ctx->d_scratch[i];
    return SPRS_B200_OK;
}

int ctx_side_stream(sprs_b200_ctx* ctx) {
    if (ctx->side_stream) return SPRS_B200_OK;
    int lo = 0, hi = 0;  // numerically lower = higher priority
    SPRS_CUDA(ctx, cudaDeviceGetStreamPriorityRange(&lo, &hi));
    SPRS_CUDA(ctx, cudaStreamCreateWithPriority(&ctx->side_stream, cudaStreamNonBlocking, hi));
    SPRS_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming));
    SPRS_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_join, cudaEventDisableTiming));
    return SPRS_B200_OK;
}

int csmat_chunk_table(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, uint64_t n_chunks, bool taper,
                      cudaStream_t s, std::vector<uint64_t>* tiles, std::vector<uint64_t>* rows) {
    n_chunks = std::max<uint64_t>(1, std::min<uint64_t>(n_chunks, SPRS_E2E_MAX_CHUNKS));
    n_chunks = std::min<uint64_t>(n_chunks, m->n_tiles);
    tiles->assign(n_chunks + 1, 0);
    rows->assign(n_chunks + 1, 0);
    const uint64_t wsum = taper ? n_chunks * (n_chunks + 1) / 2 : n_chunks;
    uint64_t acc = 0;
    for (uint64_t c = 0; c < n_chunks; ++c) {
        (*tiles)[c] = m->n_tiles * acc / wsum;
        acc += taper ? n_chunks - c : 1;
    }
    (*tiles)[n_chunks] = m->n_tiles;
    // never an empty chunk: strictly increasing cut points (n_chunks <= n_tiles, so they
    // exist) -- push duplicates up, then pull anything that ran into the end back down
    for (uint64_t c = 1; c < n_chunks; ++c)
        if ((*tiles)[c] <= (*tiles)[c - 1]) (*tiles)[c] = (*tiles)[c - 1] + 1;
    for (uint64_t c = n_chunks; c-- > 1;)
        if ((*tiles)[c] >= (*tiles)[c + 1]) (*tiles)[c] = (*tiles)[c + 1] - 1;
    for (uint64_t c = 0; c <= n_chunks; ++c) {
        uint32_t r = 0;  // tile_row[0] == 0, tile_row[n_tiles] == rows
        SPRS_CUDA(ctx, cudaMemcpyAsync(&r, m->d_tile_row + (*tiles)[c], sizeof(r),
                                       cudaMemcpyDeviceToHost, s));
        SPRS_CUDA(ctx, cudaStreamSynchronize(s));
        (*rows)[c] = r;
    }
    return SPRS_B200_OK;
}

int ctx_stage(sprs_b200_ctx* ctx, size_t bytes, void** out) {
    if (bytes < 256) bytes = 256;
    if (ctx->h_stage_bytes < bytes) {
        if (ctx->h_stage) {
            SPRS_CUDA(ctx, cudaFreeHost(ctx->h_stage));
            ctx->h_stage = nullptr;
            ctx->h_stage_bytes = 0;
        }
        SPRS_CUDA(ctx, cudaMallocHost(&ctx->h_stage, bytes));
        ctx->h_stage_bytes = bytes;
    }
    *out = ctx->h_stage;
    return SPRS_B200_OK;
}

extern "C" {

int sprs_b200_version(void) { return 100; }

int sprs_b200_ctx_create(int device, sprs_b200_ctx** out) {
    if (!out) return SPRS_B200_ERR_ARGUMENT;
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        g_create_error = std::string("no CUDA device: ") + cudaGetErrorString(e);
        cudaGetLastError();
        return SPRS_B200_ERR_CUDA;
    }
    if (device < 0 || device >= n) {
        g_create_error = "device ordinal out of range";
        return SPRS_B200_ERR_ARGUMENT;
    }
    auto* ctx = new sprs_b200_ctx();
    ctx->device = device;
    cudaDeviceProp prop;
    if ((e = cudaSetDevice(device)) != cudaSuccess ||
        (e = cudaGetDeviceProperties(&prop, device)) != cudaSuccess ||
        (e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking)) != cudaSuccess) {
        g_create_error = std::string("ctx_create: ") + cudaGetErrorString(e);
        delete ctx;
        return SPRS_B200_ERR_CUDA;
    }
    // architecture-specific sm_90a code loads on compute capability 9.0 only
    if (prop.major != 9 || prop.minor != 0) {
        g_create_error = "sprs_b200 kernels are built for sm_90a (H100) only; device is sm_" +
                         std::to_string(prop.major) + std::to_string(prop.minor);
        cudaStreamDestroy(ctx->stream);
        delete ctx;
        return SPRS_B200_ERR_CUDA;
    }
    ctx->sm_count = prop.multiProcessorCount;
    ctx->l2_bytes = (size_t)prop.l2CacheSize;
    {
        uint64_t* d_pol = nullptr;
        uint64_t h_pol[2] = {0, 0};
        if ((e = cudaMalloc((void**)&d_pol, 16)) == cudaSuccess) {
            make_policies_kernel<<<1, 1, 0, ctx->stream>>>(d_pol);
            e = cudaMemcpyAsync(h_pol, d_pol, 16, cudaMemcpyDeviceToHost, ctx->stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
            cudaFree(d_pol);
        }
        if (e != cudaSuccess) {
            g_create_error = std::string("ctx_create (cache policies): ") + cudaGetErrorString(e);
            cudaStreamDestroy(ctx->stream);
            delete ctx;
            return SPRS_B200_ERR_CUDA;
        }
        ctx->pol_evict_first = h_pol[0];
        ctx->pol_evict_last = h_pol[1];
    }
    {   // the stream-ordered allocator keeps what the SpGEMM frees (a 42 GB product is
        // re-allocated by the next call instead of being mapped again)
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
            uint64_t keep = ~0ull;
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
        }
        cudaGetLastError();
    }
    *out = ctx;
    return SPRS_B200_OK;
}

int sprs_b200_ctx_destroy(sprs_b200_ctx* ctx) {
    if (!ctx) return SPRS_B200_OK;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    for (int i = 0; i < 4; ++i)
        if (ctx->d_scratch[i]) cudaFree(ctx->d_scratch[i]);
    if (ctx->h_stage) cudaFreeHost(ctx->h_stage);
    if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
    if (ctx->ev_join) cudaEventDestroy(ctx->ev_join);
    if (ctx->side_stream) cudaStreamDestroy(ctx->side_stream);
    for (int i = 0; i < SPRS_E2E_MAX_CHUNKS; ++i)
        if (ctx->ev_chunk[i]) cudaEventDestroy(ctx->ev_chunk[i]);
    if (ctx->ev_copied) cudaEventDestroy(ctx->ev_copied);
    if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
    cudaStreamDestroy(ctx->stream);
    {
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, ctx->device) == cudaSuccess) cudaMemPoolTrimTo(pool, 0);
        cudaGetLastError();
    }
    delete ctx;
    return SPRS_B200_OK;
}

const char* sprs_b200_last_error(const sprs_b200_ctx* ctx) {
    return ctx ? ctx->last_error.c_str() : g_create_error.c_str();
}
int sprs_b200_ctx_device(const sprs_b200_ctx* ctx) { return ctx ? ctx->device : -1; }
int sprs_b200_ctx_sm_count(const sprs_b200_ctx* ctx) { return ctx ? ctx->sm_count : 0; }
int sprs_b200_ctx_synchronize(sprs_b200_ctx* ctx) {
    if (!ctx) return SPRS_B200_ERR_ARGUMENT;
    SPRS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SPRS_B200_OK;
}
uint64_t sprs_b200_launch_count(const sprs_b200_ctx* ctx) { return ctx ? ctx->launches : 0; }

// ---------------------------------------------------------------------------------
int sprs_b200_csmat_upload(sprs_b200_ctx* ctx, int storage, uint64_t rows, uint64_t cols,
                           const void* indptr, int indptr_bytes, const void* indices,
                           int index_bytes, const double* data, sprs_b200_csmat** out) {
    if (!ctx || !out || !indptr) return SPRS_B200_ERR_ARGUMENT;
    *out = nullptr;
    if ((indptr_bytes != 4 && indptr_bytes != 8) || (index_bytes != 4 && index_bytes != 8) ||
        (storage != SPRS_B200_CSR && storage != SPRS_B200_CSC))
        SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "bad storage or index width");
    if (rows > 0xffffffffull || cols > 0xffffffffull)
        SPRS_FAIL(ctx, SPRS_B200_ERR_INDEX_RANGE,
                  "Index type is not large enough: device mirrors use u32 indices");
    const uint64_t outer = storage == SPRS_B200_CSR ? rows : cols;
    const uint64_t base = read_index(indptr, indptr_bytes, 0);
    const uint64_t last = read_index(indptr, indptr_bytes, outer);
    if (last < base) SPRS_FAIL(ctx, SPRS_B200_ERR_STRUCTURE, "indptr not monotone");
    const uint64_t nnz = last - base;
    if (nnz > 0 && (!indices || !data)) return SPRS_B200_ERR_ARGUMENT;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    CsmatPtr m = new_result(ctx, storage, rows, cols, nnz, indptr_bytes_for(nnz), Arrays::owned);
    cudaStream_t s = ctx->stream;
    SPRS_TRY(alloc_result(ctx, m.get(), s, "upload"));
    SPRS_TRY(upload_indexlike(ctx, indptr, indptr_bytes, outer + 1, base, m->d_indptr,
                              m->indptr_bytes, s));
    SPRS_TRY(upload_indexlike(ctx, indices, index_bytes, nnz, 0, m->d_indices, 4, s));
    if (nnz > 0)
        SPRS_CUDA(ctx, cudaMemcpyAsync(m->d_data, data, nnz * sizeof(double),
                                       cudaMemcpyHostToDevice, s));
    return finish_result(ctx, m, s, "upload", true, out);
}

int sprs_b200_csmat_from_device(sprs_b200_ctx* ctx, int storage, uint64_t rows, uint64_t cols,
                                uint64_t nnz, const uint32_t* d_indptr,
                                const uint32_t* d_indices, const double* d_data,
                                sprs_b200_csmat** out) {
    if (!ctx || !out || !d_indptr) return SPRS_B200_ERR_ARGUMENT;
    *out = nullptr;
    if (nnz >= 0xffffffffull || rows > 0xffffffffull || cols > 0xffffffffull)
        SPRS_FAIL(ctx, SPRS_B200_ERR_INDEX_RANGE, "from_device takes u32 arrays only");
    if (((uintptr_t)d_indices | (uintptr_t)d_data) & 15)
        SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "device arrays must be 16-byte aligned");
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    CsmatPtr m = new_result(ctx, storage, rows, cols, nnz, 4, Arrays::borrowed);
    m->d_indptr = const_cast<uint32_t*>(d_indptr);
    m->d_indices = const_cast<uint32_t*>(d_indices);
    m->d_data = const_cast<double*>(d_data);
    return finish_result(ctx, m, ctx->stream, "from_device", true, out);
}

int sprs_b200_csmat_free(sprs_b200_csmat* m) {
    if (!m) return SPRS_B200_OK;
    if (m->ctx) cudaSetDevice(m->ctx->device);
    if (m->owns && m->pooled && m->ctx) {  // back to the pool, ordered on the ctx stream
        cudaDeviceSynchronize();  // (readers on other streams -- a caller's views of C -- are done)
        if (m->d_indptr) cudaFreeAsync(m->d_indptr, m->ctx->stream);
        if (m->d_indices) cudaFreeAsync(m->d_indices, m->ctx->stream);
        if (m->d_data) cudaFreeAsync(m->d_data, m->ctx->stream);
    } else if (m->owns) {
        if (m->d_indptr) cudaFree(m->d_indptr);
        if (m->d_indices) cudaFree(m->d_indices);
        if (m->d_data) cudaFree(m->d_data);
    }
    if (m->d_tile_row) cudaFree(m->d_tile_row);
    if (m->d_tile_k) cudaFree(m->d_tile_k);
    if (m->d_carry) cudaFree(m->d_carry);
    if (m->d_hot_col) cudaFree(m->d_hot_col);
    if (m->d_hot_idx) cudaFree(m->d_hot_idx);
    if (m->csr_cache) sprs_b200_csmat_free(m->csr_cache);
    delete m;
    return SPRS_B200_OK;
}

int sprs_b200_csmat_storage(const sprs_b200_csmat* m) { return m ? m->storage : -1; }
uint64_t sprs_b200_csmat_rows(const sprs_b200_csmat* m) { return m ? m->rows : 0; }
uint64_t sprs_b200_csmat_cols(const sprs_b200_csmat* m) { return m ? m->cols : 0; }
uint64_t sprs_b200_csmat_nnz(const sprs_b200_csmat* m) { return m ? m->nnz : 0; }

int sprs_b200_csmat_download(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, void* indptr,
                             int indptr_bytes, void* indices, int index_bytes, double* data) {
    if (!ctx || !m || !indptr) return SPRS_B200_ERR_ARGUMENT;
    if ((indptr_bytes != 4 && indptr_bytes != 8) || (index_bytes != 4 && index_bytes != 8))
        SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "bad index width");
    if (indptr_bytes == 4 && m->nnz > 0xffffffffull)
        SPRS_FAIL(ctx, SPRS_B200_ERR_INDEX_RANGE, "Index type is not large enough for nnz");
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    SPRS_TRY(download_indexlike(ctx, m->d_indptr, m->indptr_bytes, m->outer + 1, indptr,
                                indptr_bytes, s));
    if (m->nnz) {
        if (!indices || !data) return SPRS_B200_ERR_ARGUMENT;
        SPRS_TRY(download_indexlike(ctx, m->d_indices, 4, m->nnz, indices, index_bytes, s));
        SPRS_CUDA(ctx, cudaMemcpyAsync(data, m->d_data, m->nnz * sizeof(double),
                                       cudaMemcpyDeviceToHost, s));
        SPRS_CUDA(ctx, cudaStreamSynchronize(s));
    }
    return SPRS_B200_OK;
}

int sprs_b200_csmat_device_arrays(const sprs_b200_csmat* m, const void** d_indptr,
                                  int* indptr_bytes, const uint32_t** d_indices,
                                  const double** d_data) {
    if (!m) return SPRS_B200_ERR_ARGUMENT;
    if (d_indptr) *d_indptr = m->d_indptr;
    if (indptr_bytes) *indptr_bytes = m->indptr_bytes;
    if (d_indices) *d_indices = m->d_indices;
    if (d_data) *d_data = m->d_data;
    return SPRS_B200_OK;
}

int sprs_b200_csmat_from_triplets_dev(sprs_b200_ctx* ctx, uint64_t rows, uint64_t cols,
                                      uint64_t n, const uint32_t* d_row, const uint32_t* d_col,
                                      const double* d_val, sprs_b200_csmat** out) {
    if (!ctx || !out || (n && (!d_row || !d_col || !d_val))) return SPRS_B200_ERR_ARGUMENT;
    *out = nullptr;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    CsmatPtr t;
    SPRS_TRY(triplets_to_csr_launch(ctx, rows, cols, n, d_row, d_col, d_val, &t, ctx->stream));
    return finish_result(ctx, t, ctx->stream, "from_triplets", true, out);
}

int sprs_b200_csmat_from_triplets(sprs_b200_ctx* ctx, uint64_t rows, uint64_t cols, uint64_t n,
                                  const void* row_inds, const void* col_inds, int index_bytes,
                                  const double* data, sprs_b200_csmat** out) {
    if (!ctx || !out || (n && (!row_inds || !col_inds || !data))) return SPRS_B200_ERR_ARGUMENT;
    *out = nullptr;
    if (index_bytes != 4 && index_bytes != 8)
        SPRS_FAIL(ctx, SPRS_B200_ERR_ARGUMENT, "bad index width");
    if (rows > 0xffffffffull || cols > 0xffffffffull || n >= 0xffffffffull)
        SPRS_FAIL(ctx, SPRS_B200_ERR_INDEX_RANGE, "from_triplets: needs nnz, rows, cols < 2^32");
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    CsmatPtr t;
    {   // the device copies of the triplets live until the CSR mirror is built
        Owned<uint32_t> d_row, d_col;
        Owned<double> d_val;
        SPRS_TRY(d_row.alloc(ctx, n * 4 + 16, "from_triplets"));
        SPRS_TRY(d_col.alloc(ctx, n * 4 + 16, "from_triplets"));
        SPRS_TRY(d_val.alloc(ctx, n * 8 + 16, "from_triplets"));
        SPRS_TRY(upload_indexlike(ctx, row_inds, index_bytes, n, 0, d_row, 4, s));
        SPRS_TRY(upload_indexlike(ctx, col_inds, index_bytes, n, 0, d_col, 4, s));
        if (n) SPRS_CUDA(ctx, cudaMemcpyAsync(d_val, data, n * 8, cudaMemcpyHostToDevice, s));
        SPRS_TRY(triplets_to_csr_launch(ctx, rows, cols, n, d_row, d_col, d_val, &t, s));
    }
    return finish_result(ctx, t, s, "from_triplets", true, out);
}

int sprs_b200_csmat_check_structure(sprs_b200_ctx* ctx, const sprs_b200_csmat* m,
                                    uint64_t* n_violations) {
    if (!ctx || !m || !n_violations) return SPRS_B200_ERR_ARGUMENT;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    void* d_bad = nullptr;
    SPRS_TRY(ctx_scratch(ctx, 0, 8, &d_bad));
    SPRS_CUDA(ctx, cudaMemsetAsync(d_bad, 0, 8, s));
    if (m->outer) {
        const unsigned g = (unsigned)std::min<uint64_t>((m->outer + 7) / 8,
                                                        (uint64_t)ctx->sm_count * 32);
        if (m->indptr_bytes == 4)
            check_structure_kernel<uint32_t><<<g, 256, 0, s>>>(
                (const uint32_t*)m->d_indptr, m->d_indices, m->outer, m->inner,
                (unsigned long long*)d_bad);
        else
            check_structure_kernel<uint64_t><<<g, 256, 0, s>>>(
                (const uint64_t*)m->d_indptr, m->d_indices, m->outer, m->inner,
                (unsigned long long*)d_bad);
        ctx->launches += 1;
    }
    SPRS_CUDA(ctx, cudaMemcpyAsync(n_violations, d_bad, 8, cudaMemcpyDeviceToHost, s));
    SPRS_CUDA(ctx, cudaStreamSynchronize(s));
    return SPRS_B200_OK;
}

int sprs_b200_csmat_to_other_storage(sprs_b200_ctx* ctx, const sprs_b200_csmat* m,
                                     sprs_b200_csmat** out) {
    if (!ctx || !m || !out) return SPRS_B200_ERR_ARGUMENT;
    *out = nullptr;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    CsmatPtr t;
    SPRS_TRY(transpose_launch(ctx, m, &t, ctx->stream));
    return finish_result(ctx, t, ctx->stream, "to_other_storage", true, out);
}

// ---------------------------------------------------------------------------------
// device-resident entry points
int sprs_b200_spmv_dev(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat, const double* d_x,
                       double* d_y, int accumulate, void* stream) {
    if (!ctx || !mat || (!d_x && mat->cols) || (!d_y && mat->rows)) return SPRS_B200_ERR_ARGUMENT;
    return spmv_launch(ctx, mat, d_x, d_y, accumulate, pick_stream(ctx, stream));
}

int sprs_b200_spmm_rowmaj_dev(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat, const double* d_b,
                              uint64_t ldb, uint64_t k, double* d_c, uint64_t ldc,
                              int accumulate, void* stream) {
    if (!ctx || !mat) return SPRS_B200_ERR_ARGUMENT;
    if (ldb < k || ldc < k) SPRS_FAIL(ctx, SPRS_B200_ERR_DIMENSION, "Dimension mismatch: ld < k");
    return spmm_rowmaj_launch(ctx, mat, d_b, ldb, k, d_c, ldc, accumulate,
                              pick_stream(ctx, stream));
}

// ---------------------------------------------------------------------------------
// host-buffer entry points.  x / y travel through cudaMemcpyAsync on the ctx stream
// (true DMA when the caller's buffers are pinned); the call blocks until y is visible.

// Chunked variant of the host path: the tile stream is cut into a few chunks; each chunk's
// SpMV + carry kernel is followed by an event, and a second stream copies the rows that chunk
// completed to the host while the next chunk computes -- plain stream/event ordering, no kernel
// waits on another.  Only the last chunk's copy is left after the SpMV.  Bit-identical to the
// one-shot SpMV (spmv_launch_tile_range).
static int spmv_host_chunked(sprs_b200_ctx* ctx, const sprs_b200_csmat* csr, const double* d_x,
                             double* d_y, double* y, int accumulate, int n_chunks_want,
                             cudaStream_t s) {
    if (!ctx->copy_stream) {
        SPRS_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
        SPRS_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_copied, cudaEventDisableTiming));
    }
    if (!ctx->ev_chunk[0])
        for (int i = 0; i < SPRS_E2E_MAX_CHUNKS; ++i)
            SPRS_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_chunk[i], cudaEventDisableTiming));
    if (csr->e2e_tiles.empty()) {
        std::vector<uint64_t> tiles, rows;
        SPRS_TRY(csmat_chunk_table(ctx, csr, (uint64_t)n_chunks_want, false, s, &tiles, &rows));
        csr->e2e_rows = rows;
        csr->e2e_tiles = tiles;
    }
    const size_t n_chunks = csr->e2e_tiles.size() - 1;
    for (size_t c = 0; c < n_chunks; ++c) {
        SPRS_TRY(spmv_launch_tile_range(ctx, csr, d_x, d_y, accumulate, csr->e2e_tiles[c],
                                        csr->e2e_tiles[c + 1], s));
        SPRS_CUDA(ctx, cudaEventRecord(ctx->ev_chunk[c], s));
    }
    for (size_t c = 0; c < n_chunks; ++c) {
        const uint64_t r0 = csr->e2e_rows[c], r1 = csr->e2e_rows[c + 1];
        SPRS_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_chunk[c], 0));
        if (r1 > r0)
            SPRS_CUDA(ctx, cudaMemcpyAsync(y + r0, d_y + r0, (r1 - r0) * sizeof(double),
                                           cudaMemcpyDeviceToHost, ctx->copy_stream));
    }
    // join: the ctx stream (and the caller, who synchronises it) waits for the last copy
    SPRS_CUDA(ctx, cudaEventRecord(ctx->ev_copied, ctx->copy_stream));
    SPRS_CUDA(ctx, cudaStreamWaitEvent(s, ctx->ev_copied, 0));
    return SPRS_B200_OK;
}

static int spmv_host(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat, int want_storage,
                     const double* x, uint64_t x_len, double* y, uint64_t y_len,
                     int accumulate) {
    if (!ctx || !mat) return SPRS_B200_ERR_ARGUMENT;
    // the reference asserts dimensions first, then storage (prod.rs:114-118)
    if (mat->cols != x_len || mat->rows != y_len)
        SPRS_FAIL(ctx, SPRS_B200_ERR_DIMENSION, "Dimension mismatch");
    if (mat->storage != want_storage) SPRS_FAIL(ctx, SPRS_B200_ERR_STORAGE, "Storage mismatch");
    if ((x_len && !x) || (y_len && !y)) return SPRS_B200_ERR_ARGUMENT;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    const sprs_b200_csmat* csr = nullptr;
    SPRS_TRY(csmat_csr_view(ctx, mat, &csr));
    void *d_x = nullptr, *d_y = nullptr;
    SPRS_TRY(ctx_scratch(ctx, 1, x_len * sizeof(double), &d_x));
    SPRS_TRY(ctx_scratch(ctx, 2, y_len * sizeof(double), &d_y));
    if (x_len)
        SPRS_CUDA(ctx, cudaMemcpyAsync(d_x, x, x_len * sizeof(double), cudaMemcpyHostToDevice, s));
    if (accumulate && y_len)
        SPRS_CUDA(ctx, cudaMemcpyAsync(d_y, y, y_len * sizeof(double), cudaMemcpyHostToDevice, s));
    // SPRS_B200_E2E_CHUNKS=n (n > 1): the tile stream runs in n chunks and each chunk's
    // finished rows leave for the host behind its event while the next chunk computes
    // (spmv_host_chunked); default: one launch, one D2H copy.
    static const int chunks = [] {
        const char* v = getenv("SPRS_B200_E2E_CHUNKS");
        return v ? atoi(v) : SPRS_E2E_DEFAULT_CHUNKS;
    }();
    // (a chunk is worth its launch only with >= ~1000 tiles; SPRS_B200_E2E_MIN_TILES is a TEST
    // hook that lets small matrices take the chunked path)
    static const uint64_t min_tiles = [] {
        const char* v = getenv("SPRS_B200_E2E_MIN_TILES");
        return v ? (uint64_t)atoll(v) : (uint64_t)1024;
    }();
    if (chunks > 1 && y_len >= 4096 && csr->n_tiles >= (uint64_t)chunks * min_tiles) {
        SPRS_TRY(spmv_host_chunked(ctx, csr, (const double*)d_x, (double*)d_y, y, accumulate,
                                   chunks, s));
    } else {
        SPRS_TRY(spmv_launch(ctx, csr, (const double*)d_x, (double*)d_y, accumulate, s));
        if (y_len)
            SPRS_CUDA(ctx, cudaMemcpyAsync(y, d_y, y_len * sizeof(double), cudaMemcpyDeviceToHost, s));
    }
    SPRS_CUDA(ctx, cudaStreamSynchronize(s));
    return SPRS_B200_OK;
}

int sprs_b200_mul_acc_mat_vec_csr(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat,
                                  const double* in_vec, uint64_t in_len, double* res_vec,
                                  uint64_t res_len) {
    return spmv_host(ctx, mat, SPRS_B200_CSR, in_vec, in_len, res_vec, res_len, 1);
}
int sprs_b200_mul_acc_mat_vec_csc(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat,
                                  const double* in_vec, uint64_t in_len, double* res_vec,
                                  uint64_t res_len) {
    return spmv_host(ctx, mat, SPRS_B200_CSC, in_vec, in_len, res_vec, res_len, 1);
}
int sprs_b200_mul_mat_vec(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat, const double* x,
                          uint64_t x_len, double* y, uint64_t y_len) {
    if (!mat) return SPRS_B200_ERR_ARGUMENT;
    return spmv_host(ctx, mat, mat->storage, x, x_len, y, y_len, 0);
}

// out += lhs * rhs with ndarray-view operands.  rowmaj: out rows are the unit of work
// (prod.rs:189-214); colmaj: one SpMV per rhs column (prod.rs:274-298).  Views are
// packed to contiguous C-order (rowmaj) / F-order (colmaj) on the device.
static int dense_host(sprs_b200_ctx* ctx, const sprs_b200_csmat* lhs, int want_storage,
                      bool rowmaj, const double* rhs, uint64_t rhs_rows, uint64_t rhs_cols,
                      int64_t rhs_rs, int64_t rhs_cs, double* out, uint64_t out_rows,
                      uint64_t out_cols, int64_t out_rs, int64_t out_cs) {
    if (!ctx || !lhs) return SPRS_B200_ERR_ARGUMENT;
    // assert order of the reference: prod.rs:198-201 / 283-286
    if (lhs->cols != rhs_rows || lhs->rows != out_rows || rhs_cols != out_cols)
        SPRS_FAIL(ctx, SPRS_B200_ERR_DIMENSION, "Dimension mismatch");
    if (lhs->storage != want_storage) SPRS_FAIL(ctx, SPRS_B200_ERR_STORAGE, "Storage mismatch");
    const uint64_t k = rhs_cols;
    if (out_rows == 0 || k == 0) return SPRS_B200_OK;
    if (!rhs || !out) return SPRS_B200_ERR_ARGUMENT;
    SPRS_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    const sprs_b200_csmat* csr = nullptr;
    SPRS_TRY(csmat_csr_view(ctx, lhs, &csr));
    // Pack views on the host into the pinned staging buffer in the kernel's layout:
    // row-major (rowmaj) or column-major (colmaj).  O(size) copies, no arithmetic.
    const size_t nb = (size_t)rhs_rows * k, nc = (size_t)out_rows * k;
    void* hs = nullptr;
    SPRS_TRY(ctx_stage(ctx, (nb + nc) * sizeof(double), &hs));
    double* hb = (double*)hs;
    double* hc = hb + nb;
    if (rowmaj) {
        for (uint64_t r = 0; r < rhs_rows; ++r)
            for (uint64_t c = 0; c < k; ++c)
                hb[r * k + c] = rhs[(int64_t)r * rhs_rs + (int64_t)c * rhs_cs];
        for (uint64_t r = 0; r < out_rows; ++r)
            for (uint64_t c = 0; c < k; ++c)
                hc[r * k + c] = out[(int64_t)r * out_rs + (int64_t)c * out_cs];
    } else {
        for (uint64_t c = 0; c < k; ++c)
            for (uint64_t r = 0; r < rhs_rows; ++r)
                hb[c * rhs_rows + r] = rhs[(int64_t)r * rhs_rs + (int64_t)c * rhs_cs];
        for (uint64_t c = 0; c < k; ++c)
            for (uint64_t r = 0; r < out_rows; ++r)
                hc[c * out_rows + r] = out[(int64_t)r * out_rs + (int64_t)c * out_cs];
    }
    void *d_b = nullptr, *d_c = nullptr;
    SPRS_TRY(ctx_scratch(ctx, 1, nb * sizeof(double), &d_b));
    SPRS_TRY(ctx_scratch(ctx, 2, nc * sizeof(double), &d_c));
    SPRS_CUDA(ctx, cudaMemcpyAsync(d_b, hb, nb * sizeof(double), cudaMemcpyHostToDevice, s));
    SPRS_CUDA(ctx, cudaMemcpyAsync(d_c, hc, nc * sizeof(double), cudaMemcpyHostToDevice, s));
    if (rowmaj)
        SPRS_TRY(spmm_rowmaj_launch(ctx, csr, (const double*)d_b, k, k, (double*)d_c, k, 1, s));
    else
        for (uint64_t c = 0; c < k; ++c)
            SPRS_TRY(spmv_launch(ctx, csr, (const double*)d_b + c * rhs_rows,
                                 (double*)d_c + c * out_rows, 1, s));
    SPRS_CUDA(ctx, cudaMemcpyAsync(hc, d_c, nc * sizeof(double), cudaMemcpyDeviceToHost, s));
    SPRS_CUDA(ctx, cudaStreamSynchronize(s));
    if (rowmaj) {
        for (uint64_t r = 0; r < out_rows; ++r)
            for (uint64_t c = 0; c < k; ++c)
                out[(int64_t)r * out_rs + (int64_t)c * out_cs] = hc[r * k + c];
    } else {
        for (uint64_t c = 0; c < k; ++c)
            for (uint64_t r = 0; r < out_rows; ++r)
                out[(int64_t)r * out_rs + (int64_t)c * out_cs] = hc[c * out_rows + r];
    }
    return SPRS_B200_OK;
}

int sprs_b200_csr_mulacc_dense_rowmaj(sprs_b200_ctx* ctx, const sprs_b200_csmat* lhs,
                                      const double* rhs, uint64_t rhs_rows, uint64_t rhs_cols,
                                      int64_t rhs_rs, int64_t rhs_cs, double* out,
                                      uint64_t out_rows, uint64_t out_cols, int64_t out_rs,
                                      int64_t out_cs) {
    return dense_host(ctx, lhs, SPRS_B200_CSR, true, rhs, rhs_rows, rhs_cols, rhs_rs, rhs_cs,
                      out, out_rows, out_cols, out_rs, out_cs);
}
int sprs_b200_csr_mulacc_dense_colmaj(sprs_b200_ctx* ctx, const sprs_b200_csmat* lhs,
                                      const double* rhs, uint64_t rhs_rows, uint64_t rhs_cols,
                                      int64_t rhs_rs, int64_t rhs_cs, double* out,
                                      uint64_t out_rows, uint64_t out_cols, int64_t out_rs,
                                      int64_t out_cs) {
    return dense_host(ctx, lhs, SPRS_B200_CSR, false, rhs, rhs_rows, rhs_cols, rhs_rs, rhs_cs,
                      out, out_rows, out_cols, out_rs, out_cs);
}
int sprs_b200_csc_mulacc_dense_rowmaj(sprs_b200_ctx* ctx, const sprs_b200_csmat* lhs,
                                      const double* rhs, uint64_t rhs_rows, uint64_t rhs_cols,
                                      int64_t rhs_rs, int64_t rhs_cs, double* out,
                                      uint64_t out_rows, uint64_t out_cols, int64_t out_rs,
                                      int64_t out_cs) {
    return dense_host(ctx, lhs, SPRS_B200_CSC, true, rhs, rhs_rows, rhs_cols, rhs_rs, rhs_cs,
                      out, out_rows, out_cols, out_rs, out_cs);
}
int sprs_b200_csc_mulacc_dense_colmaj(sprs_b200_ctx* ctx, const sprs_b200_csmat* lhs,
                                      const double* rhs, uint64_t rhs_rows, uint64_t rhs_cols,
                                      int64_t rhs_rs, int64_t rhs_cs, double* out,
                                      uint64_t out_rows, uint64_t out_cols, int64_t out_rs,
                                      int64_t out_cs) {
    return dense_host(ctx, lhs, SPRS_B200_CSC, false, rhs, rhs_rows, rhs_cols, rhs_rs, rhs_cs,
                      out, out_rows, out_cols, out_rs, out_cs);
}

}  // extern "C"

// ---- scoped ownership and mirrors built on the device (declared in common.cuh)
int mem_alloc(sprs_b200_ctx* ctx, MemKind kind, size_t bytes, cudaStream_t s, const char* what,
              void** p) {
    const cudaError_t e = kind == MemKind::device   ? cudaMalloc(p, bytes)
                          : kind == MemKind::stream ? cudaMallocAsync(p, bytes, s)
                                                    : cudaMallocHost(p, bytes);
    if (e == cudaSuccess) return SPRS_B200_OK;
    cudaGetLastError();  // (the failed allocation leaves its error behind: reported here)
    *p = nullptr;
    static const char* const calls[] = {"cudaMalloc", "cudaMallocAsync", "cudaMallocHost"};
    SPRS_FAIL(ctx, SPRS_B200_ERR_CUDA, "%s: %s of %zu bytes failed: %s", what, calls[(int)kind],
              bytes, cudaGetErrorString(e));
}

void mem_free(MemKind kind, void* p, cudaStream_t s) {
    if (kind == MemKind::device)
        cudaFree(p);
    else if (kind == MemKind::stream)
        cudaFreeAsync(p, s);
    else
        cudaFreeHost(p);
}

int indptr_bytes_for(uint64_t nnz) {
    static const bool force64 = [] {
        const char* v = getenv("SPRS_B200_FORCE_INDPTR64");
        return v && atoi(v) != 0;
    }();
    return (nnz >= 0xffffffffull || force64) ? 8 : 4;
}

sprs_b200_csmat csmat_init(sprs_b200_ctx* ctx, int storage, uint64_t rows, uint64_t cols,
                           uint64_t nnz, int indptr_bytes, Arrays arrays) {
    sprs_b200_csmat m;
    m.ctx = ctx;
    m.storage = storage;
    m.rows = rows;
    m.cols = cols;
    m.outer = storage == SPRS_B200_CSR ? rows : cols;
    m.inner = storage == SPRS_B200_CSR ? cols : rows;
    m.nnz = nnz;
    m.indptr_bytes = indptr_bytes;
    m.owns = arrays != Arrays::borrowed;
    m.pooled = arrays == Arrays::pooled;
    return m;
}

CsmatPtr new_result(sprs_b200_ctx* ctx, int storage, uint64_t rows, uint64_t cols, uint64_t nnz,
                    int indptr_bytes, Arrays arrays) {
    return CsmatPtr(new sprs_b200_csmat(
        csmat_init(ctx, storage, rows, cols, nnz, indptr_bytes, arrays)));
}

int alloc_result(sprs_b200_ctx* ctx, sprs_b200_csmat* m, cudaStream_t s, const char* what) {
    const MemKind kind = m->pooled ? MemKind::stream : MemKind::device;
    SPRS_TRY(mem_alloc(ctx, kind, (m->outer + 1) * (size_t)m->indptr_bytes + 16, s, what,
                       &m->d_indptr));
    SPRS_TRY(mem_alloc(ctx, kind, m->nnz * 4 + 16, s, what, (void**)&m->d_indices));
    SPRS_TRY(mem_alloc(ctx, kind, m->nnz * 8 + 16, s, what, (void**)&m->d_data));
    return SPRS_B200_OK;
}

// CSR view of a mirror for the product kernels: the mirror itself, or (CSC) its cached
// device conversion -- same sums in the same order (ascending column per output element).
int csmat_csr_view(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, const sprs_b200_csmat** out) {
    if (m->storage == SPRS_B200_CSR) {
        *out = m;
        return SPRS_B200_OK;
    }
    if (!m->csr_cache) {
        sprs_b200_csmat* t = nullptr;
        SPRS_TRY(sprs_b200_csmat_to_other_storage(ctx, m, &t));
        m->csr_cache = t;
    }
    *out = m->csr_cache;
    return SPRS_B200_OK;
}

int finish_result(sprs_b200_ctx* ctx, CsmatPtr& m, cudaStream_t s, const char* what, bool hot_set,
                  sprs_b200_csmat** out) {
    SPRS_TRY(spmv_prepare(ctx, m.get(), s, hot_set));
    if (cudaStreamSynchronize(s) != cudaSuccess || cudaGetLastError() != cudaSuccess)
        SPRS_FAIL(ctx, SPRS_B200_ERR_CUDA, "%s: kernel failed", what);
    *out = m.release();
    return SPRS_B200_OK;
}
