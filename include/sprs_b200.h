/* sprs_b200.h -- C ABI of the H100-native sprs product path.
 *
 * This is the drop-in boundary: exactly what a Rust `sprs-b200-sys` crate would
 * bind (INTEGRATION.md shows the extern "C" block and the safe wrapper).  It
 * follows the reference's own FFI conventions:
 *   - raw-pointer CSR, plain scalars, explicit sizes, zero-based ("proper")
 *     indptr expected from callers that slice -- the in-tree precedent is
 *     `prod_nnz(a_rows,a_cols,b_cols,a_indptr*,a_indices*,a_data*,...)`
 *     sprs-benches/src/eigen.cpp:5-29, declared sprs-benches/src/main.rs:27-42,
 *     called with proper_indptr()/as_ptr() at main.rs:55-80;
 *   - caller-owned host buffers borrowed for the call (sprs_suitesparse_camd/
 *     src/lib.rs:39-51), library-owned opaque handles released by an explicit
 *     *_free called from Rust `Drop` (the UMFPACK pattern,
 *     suitesparse_umfpack_sys/src/umfpack_free_numeric.rs:3-6);
 *   - `int` status returns, 0 = ok; the Rust side maps non-zero to
 *     LinalgError::ThirdPartyError(code, msg) (sprs/src/errors.rs:70) and keeps
 *     the reference's panics ("Dimension mismatch", "Storage mismatch") for
 *     contract violations (prod.rs:114-118, 198-201, 283-286; smmp.rs:207).
 *
 * Scalars are f64 (BASELINE).  Host index arrays may be 4 or 8 bytes wide
 * (u32/i32 or u64/usize/i64/isize -- signed types are valid because sprs
 * structure checks guarantee non-negative values, sparse.rs:326-332); the
 * device mirror always stores u32 indices and u32 (or u64 when nnz >= 2^32)
 * indptr.  No call routes through a CPU implementation: if the device or the
 * kernels are unavailable every entry point fails with SPRS_B200_ERR_CUDA.
 */
#ifndef SPRS_B200_H
#define SPRS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct sprs_b200_ctx sprs_b200_ctx;       /* one device + stream + scratch          */
typedef struct sprs_b200_csmat sprs_b200_csmat;   /* device mirror of a CsMatBase           */
typedef struct sprs_b200_spgemm sprs_b200_spgemm; /* state between symbolic and numeric     */

/* sprs::CompressedStorage (sprs/src/sparse.rs:31-38) */
enum { SPRS_B200_CSR = 0, SPRS_B200_CSC = 1 };

/* status codes */
enum {
    SPRS_B200_OK = 0,
    SPRS_B200_ERR_DIMENSION = 1,   /* "Dimension mismatch"  (prod.rs:114-116)            */
    SPRS_B200_ERR_STORAGE = 2,     /* "Storage mismatch"    (prod.rs:118)                */
    SPRS_B200_ERR_CUDA = 3,        /* CUDA runtime / launch failure; see last_error      */
    SPRS_B200_ERR_NCCL = 4,
    SPRS_B200_ERR_INDEX_RANGE = 5, /* "Index type is not large enough" (csmat.rs:1794)   */
    SPRS_B200_ERR_ARGUMENT = 6,    /* null pointer, bad width, bad handle                */
    SPRS_B200_ERR_STRUCTURE = 7,   /* indptr not monotone / index out of bounds          */
    SPRS_B200_ERR_UNSUPPORTED = 8,
    SPRS_B200_ERR_COMM = 9,        /* multi-GPU rendezvous / barrier failure; see last_error */
    SPRS_B200_ERR_SINGULAR = 10    /* LinalgError::SingularMatrix (errors.rs:59-69); see
                                      sprs_b200_trisolve_singular                           */
};

int sprs_b200_version(void);

/* ---- context -------------------------------------------------------------- */
int sprs_b200_ctx_create(int device, sprs_b200_ctx** out);
int sprs_b200_ctx_destroy(sprs_b200_ctx* ctx);
/* message of the last failing call on this ctx (or of a failed ctx_create when ctx==NULL) */
const char* sprs_b200_last_error(const sprs_b200_ctx* ctx);
int sprs_b200_ctx_device(const sprs_b200_ctx* ctx);
int sprs_b200_ctx_sm_count(const sprs_b200_ctx* ctx);
int sprs_b200_ctx_synchronize(sprs_b200_ctx* ctx);

/* ---- device mirror of CsMatBase{storage, nrows, ncols, indptr, indices, data}
 *      (sprs/src/sparse.rs:94-109).  `indptr` has outer+1 entries and may be
 *      non-zero-based (row-sliced view, indptr.rs:122-124): it is rebased on
 *      upload, as proper_indptr() does (csmat.rs:919-921).  Widths in bytes.   */
int sprs_b200_csmat_upload(sprs_b200_ctx* ctx, int storage, uint64_t rows, uint64_t cols,
                           const void* indptr, int indptr_bytes, const void* indices,
                           int index_bytes, const double* data, sprs_b200_csmat** out);
/* Adopt device-resident arrays (u32, zero-based, 16-byte aligned) without copying; the
 * caller keeps ownership and must keep them alive.  Used by generators / benchmarks.
 * The arrays must be COMPLETE when the call is made (it reads them on the ctx's own stream:
 * synchronise the stream that produced them first).  upload / from_device adopt the structure
 * as given, like CsMatBase::new_unchecked: out-of-range indices are the caller's contract
 * (the host mirrors check it, sparse.rs:300-369; sprs_b200_csmat_check_structure does so on the
 * device).  One product at a time per mirror: a mirror carries the SpMV's per-tile carry
 * scratch, so two SpMVs of the SAME mirror must not be in flight on different streams.     */
int sprs_b200_csmat_from_device(sprs_b200_ctx* ctx, int storage, uint64_t rows, uint64_t cols,
                                uint64_t nnz, const uint32_t* d_indptr,
                                const uint32_t* d_indices, const double* d_data,
                                sprs_b200_csmat** out);
int sprs_b200_csmat_free(sprs_b200_csmat* m);
int sprs_b200_csmat_storage(const sprs_b200_csmat* m);
uint64_t sprs_b200_csmat_rows(const sprs_b200_csmat* m);
uint64_t sprs_b200_csmat_cols(const sprs_b200_csmat* m);
uint64_t sprs_b200_csmat_nnz(const sprs_b200_csmat* m);
/* copy the mirror back to caller-allocated host arrays (outer+1, nnz, nnz entries) */
int sprs_b200_csmat_download(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, void* indptr,
                             int indptr_bytes, void* indices, int index_bytes, double* data);
/* raw device pointers of the mirror (u32 indices; indptr u32 unless nnz >= 2^32) */
int sprs_b200_csmat_device_arrays(const sprs_b200_csmat* m, const void** d_indptr,
                                  int* indptr_bytes, const uint32_t** d_indices,
                                  const double** d_data);
/* TriMatBase::to_csr (sprs/src/sparse/triplet_iter.rs:127-224): COO triplets in any order,
 * duplicates allowed -> CSR mirror with ascending unique columns per row, duplicate entries
 * SUMMED (in insertion order).  Host arrays (index width 4 or 8) or device u32 arrays.
 * A triplet outside rows x cols returns ERR_STRUCTURE (the reference asserts in add_triplet). */
int sprs_b200_csmat_from_triplets(sprs_b200_ctx* ctx, uint64_t rows, uint64_t cols, uint64_t n,
                                  const void* row_inds, const void* col_inds, int index_bytes,
                                  const double* data, sprs_b200_csmat** out);
int sprs_b200_csmat_from_triplets_dev(sprs_b200_ctx* ctx, uint64_t rows, uint64_t cols,
                                      uint64_t n, const uint32_t* d_row, const uint32_t* d_col,
                                      const double* d_val, sprs_b200_csmat** out);
/* check_compressed_structure (sprs/src/sparse.rs:300-369) on the device: counts outer
 * dims with a decreasing indptr, an out-of-range index or non-ascending indices. */
int sprs_b200_csmat_check_structure(sprs_b200_ctx* ctx, const sprs_b200_csmat* m,
                                    uint64_t* n_violations);
/* CsMatBase::to_other_storage / raw::convert_mat_storage (csmat.rs:1405-1426,1782-1829):
 * a new mirror with the other storage order, indices ascending per outer dim. */
int sprs_b200_csmat_to_other_storage(sprs_b200_ctx* ctx, const sprs_b200_csmat* m,
                                     sprs_b200_csmat** out);

/* ---- sparse (+, -, Hadamard) sparse and sparse * scalar, device-resident result --------
 * The host-buffer form needs no symbol of its own: read csmat_nnz of the result, allocate,
 * and csmat_download it.                                                                    */
enum { SPRS_B200_BINOP_ADD = 0, SPRS_B200_BINOP_SUB = 1, SPRS_B200_BINOP_MUL = 2 };
/* csmat_binop (binop.rs:178-271): new mirror C, storage of lhs; entries whose result is 0.0 dropped.
 * Same storage required (else STORAGE; the host mirrors convert rhs for Add/Sub), same shape
 * (else DIMENSION, checked first), op outside the enum -> ARGUMENT.  Blocking, ctx stream;
 * operands adopted with from_device must be complete when called.                          */
int sprs_b200_csmat_binop(sprs_b200_ctx* ctx, const sprs_b200_csmat* lhs,
                          const sprs_b200_csmat* rhs, int op, sprs_b200_csmat** out);
/* &A * s (binop.rs:132-163 -> CsMatBase::map): same structure, data[k]*s, zeros kept */
int sprs_b200_csmat_scale(sprs_b200_ctx* ctx, const sprs_b200_csmat* m, double s,
                          sprs_b200_csmat** out);

/* ---- sparse x dense vector, HOST buffers (copies are part of the call) --------
 * prod::mul_acc_mat_vec_csr(mat, in_vec, res_vec)  prod.rs:103-127 : y += A x
 * prod::mul_acc_mat_vec_csc                        prod.rs:74-99
 * Errors: DIMENSION if x_len != cols or y_len != rows, STORAGE if wrong storage. */
int sprs_b200_mul_acc_mat_vec_csr(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat,
                                  const double* in_vec, uint64_t in_len, double* res_vec,
                                  uint64_t res_len);
int sprs_b200_mul_acc_mat_vec_csc(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat,
                                  const double* in_vec, uint64_t in_len, double* res_vec,
                                  uint64_t res_len);
/* `&A * &x` (csmat.rs:2119-2160): y = A x into a caller-allocated zero-initialised-
 * or-not buffer (y is overwritten; saves uploading the zeros the operator allocates). */
int sprs_b200_mul_mat_vec(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat, const double* x,
                          uint64_t x_len, double* y, uint64_t y_len);

/* prod::csr_mul_csvec(lhs, rhs) (prod.rs:162-184): what `&A * &v` runs for a CSR matrix and a
 * sparse vector (vec.rs:1104-1131; the README example, BASELINE config 1).  res[i] is the
 * reference's sorted-merge dot of row i with v (CsVecBase::dot_acc, vec.rs:846-881): only
 * entries present in BOTH patterns are multiplied, summed sequentially in ascending column
 * order -- bit-identical to the reference, non-finite values included.  `res` is a dense host
 * array of `rows` doubles (0.0 where no entries meet); the caller builds the CsVec by dropping
 * exact zeros (prod.rs:178-180) and handles the dim == 0 early return (prod.rs:170-173).
 * v_indices: ascending, unique, < dim (the CsVec invariant), 4 or 8 bytes wide.
 * Errors: DIMENSION if dim != cols or res_len != rows, STORAGE if the mirror is not CSR,
 * STRUCTURE for an index >= dim.                                                        */
int sprs_b200_csr_mul_csvec(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat, uint64_t dim,
                            uint64_t v_nnz, const void* v_indices, int index_bytes,
                            const double* v_data, double* res, uint64_t res_len);
/* The same dot products, each sum starting from res[i] instead of 0.0: res[i] is read, then
 * overwritten.  CsVecBase::dot_dense (vec.rs:894-904) sums with `Iterator::sum`, whose f64
 * fold starts from -0.0, so its mirrors pass res = {-0.0}.                               */
int sprs_b200_csr_mul_csvec_acc(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat, uint64_t dim,
                                uint64_t v_nnz, const void* v_indices, int index_bytes,
                                const double* v_data, double* res, uint64_t res_len);

/* ---- sparse x dense matrix, HOST buffers; rhs/out are ndarray views, strides in
 * ELEMENTS (may be negative/any, like ArrayView).  out += lhs * rhs.
 * prod::csr_mulacc_dense_rowmaj prod.rs:189-214 ; csr_mulacc_dense_colmaj :274-298
 * prod::csc_mulacc_dense_rowmaj prod.rs:219-241 ; csc_mulacc_dense_colmaj :246-269  */
int sprs_b200_csr_mulacc_dense_rowmaj(sprs_b200_ctx* ctx, const sprs_b200_csmat* lhs,
                                      const double* rhs, uint64_t rhs_rows, uint64_t rhs_cols,
                                      int64_t rhs_rs, int64_t rhs_cs, double* out,
                                      uint64_t out_rows, uint64_t out_cols, int64_t out_rs,
                                      int64_t out_cs);
int sprs_b200_csr_mulacc_dense_colmaj(sprs_b200_ctx* ctx, const sprs_b200_csmat* lhs,
                                      const double* rhs, uint64_t rhs_rows, uint64_t rhs_cols,
                                      int64_t rhs_rs, int64_t rhs_cs, double* out,
                                      uint64_t out_rows, uint64_t out_cols, int64_t out_rs,
                                      int64_t out_cs);
int sprs_b200_csc_mulacc_dense_rowmaj(sprs_b200_ctx* ctx, const sprs_b200_csmat* lhs,
                                      const double* rhs, uint64_t rhs_rows, uint64_t rhs_cols,
                                      int64_t rhs_rs, int64_t rhs_cs, double* out,
                                      uint64_t out_rows, uint64_t out_cols, int64_t out_rs,
                                      int64_t out_cs);
int sprs_b200_csc_mulacc_dense_colmaj(sprs_b200_ctx* ctx, const sprs_b200_csmat* lhs,
                                      const double* rhs, uint64_t rhs_rows, uint64_t rhs_cols,
                                      int64_t rhs_rs, int64_t rhs_cs, double* out,
                                      uint64_t out_rows, uint64_t out_cols, int64_t out_rs,
                                      int64_t out_cs);

/* ---- device-resident entry points (x, y, B, C already in HBM; `stream` is a
 * cudaStream_t passed as void*; NULL is CUDA's legacy default stream, as usual).
 * Asynchronous: they return after enqueueing.  accumulate != 0 : y += A x ; == 0 : y = A x.
 * The matrix must be CSR (convert a CSC mirror with csmat_to_other_storage).     */
int sprs_b200_spmv_dev(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat, const double* d_x,
                       double* d_y, int accumulate, void* stream);
/* C(rows x k) (+)= A * B(cols x k); B, C row-major with leading dimensions ldb, ldc
 * (csr_mulacc_dense_rowmaj on contiguous C-order operands, csmat.rs:2010-2018).  */
int sprs_b200_spmm_rowmaj_dev(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat, const double* d_b,
                              uint64_t ldb, uint64_t k, double* d_c, uint64_t ldc,
                              int accumulate, void* stream);
/* number of kernel launches the library has issued on this ctx (all entry points) */
uint64_t sprs_b200_launch_count(const sprs_b200_ctx* ctx);

/* ---- multi-GPU, one process per GPU (the reference has no multi-device code; the shard
 * primitive is slice_outer, slicing.rs:65-89): each rank holds a contiguous row block as
 * its own mirror, x is replicated, y (n entries) lives in a peer-mappable buffer per rank.
 * peer_alloc returns the buffer and its 64-byte CUDA IPC handle; the caller ships handles to
 * the other ranks (any transport), which map them with peer_open.
 * spmv_allgather_dev: y[row_offset .. row_offset+rows) = A_local x, stored by the kernel
 * into ALL n_targets buffers (d_y_bufs[0] must be this rank's own buffer, the others the
 * peer mappings): the all-gather of y is fused into the SpMV.  The caller orders the next
 * consumer of y after a cross-rank barrier on the same stream.                        */
int sprs_b200_peer_alloc(sprs_b200_ctx* ctx, uint64_t bytes, void** d_ptr,
                         unsigned char ipc_handle[64]);
int sprs_b200_peer_open(sprs_b200_ctx* ctx, const unsigned char ipc_handle[64], void** d_ptr);
int sprs_b200_peer_close(sprs_b200_ctx* ctx, void* d_ptr);
int sprs_b200_peer_free(sprs_b200_ctx* ctx, void* d_ptr);
int sprs_b200_copy_dev(sprs_b200_ctx* ctx, void* dst, const void* src, uint64_t bytes,
                       void* stream);
/* host <-> device copies for callers that own no CUDA runtime of their own (a Rust host
 * filling a symmetric buffer): enqueued on `stream`, which is synchronised before returning */
int sprs_b200_copy_to_device(sprs_b200_ctx* ctx, void* d_dst, const void* h_src, uint64_t bytes,
                             void* stream);
int sprs_b200_copy_to_host(sprs_b200_ctx* ctx, void* h_dst, const void* d_src, uint64_t bytes,
                           void* stream);
/* all-gather "put": copy y[row_offset .. row_offset+rows) of this rank's buffer into the same
 * position of n_peers (0..8) peer buffers with one kernel (coalesced 16-byte stores over
 * NVLink).  Every peer buffer must be non-null and have the same address modulo 16 as
 * d_y_own (any two cudaMalloc / symm_alloc buffers do), else ERR_ARGUMENT and nothing is
 * launched.  The same rule holds for d_y_bufs[1..) against d_y_bufs[0] in
 * spmv_chunked_push_dev.                                                                  */
int sprs_b200_peer_push_dev(sprs_b200_ctx* ctx, const double* d_y_own, uint64_t row_offset,
                            uint64_t rows, int n_peers, double* const* d_y_peers, void* stream);
int sprs_b200_spmv_allgather_dev(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat,
                                 const double* d_x, uint64_t row_offset, int n_targets,
                                 double* const* d_y_bufs, int accumulate, void* stream);
/* The same all-gather pipelined by plain stream ordering: the tile stream of the block is
 * launched in `n_chunks` chunks of decreasing size (0 = default 4, at most 8); behind each
 * chunk's event a side stream of the ctx copies the rows that chunk completed (carries
 * applied) into d_y_bufs[1..) with a put kernel while the next chunk computes; `stream` is
 * joined with the side stream before the call returns control to it.  Bit-identical to
 * sprs_b200_spmv_dev.  Safe under tools that serialise kernels.                          */
int sprs_b200_spmv_chunked_push_dev(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat,
                                    const double* d_x, uint64_t row_offset, int n_targets,
                                    double* const* d_y_bufs, int accumulate, int n_chunks,
                                    void* stream);

/* ---- multi-GPU communicator (SURVEY 8b "comm_init / spmv_rowpart", 8e): the ranks of ONE
 * node -- one process per GPU (the torchrun layout) or threads of one process -- meet through
 * a 64-byte id that rank 0 creates and the caller ships to the other ranks by any transport
 * (the way an ncclUniqueId travels: MPI, a file, an environment variable, torch.distributed).
 * No torch, no NCCL underneath: a POSIX shared-memory segment carries the host barrier and the
 * handle exchange; device buffers are shared through CUDA IPC, or through CUDA VMM handles
 * bound to an NVSwitch multicast object when every rank's device supports one.
 * All calls below except _rank/_world/_ptr are COLLECTIVE: every rank makes them in the same
 * order.  A rank that fails marks the communicator failed; the others return ERR_COMM instead
 * of waiting for it.                                                                       */
#define SPRS_B200_MAX_RANKS 8
typedef struct sprs_b200_comm sprs_b200_comm;
typedef struct sprs_b200_symm sprs_b200_symm;     /* one buffer per rank, mapped on every rank */
int sprs_b200_comm_unique_id(char id[64]);
int sprs_b200_comm_init_rank(sprs_b200_ctx* ctx, const char id[64], int rank, int world,
                             sprs_b200_comm** out);
int sprs_b200_comm_free(sprs_b200_comm* comm);
int sprs_b200_comm_rank(const sprs_b200_comm* comm);
int sprs_b200_comm_world(const sprs_b200_comm* comm);
/* 1 when symm_alloc(want_multicast) will bind an NVSwitch multicast address (every device
 * supports it, one process and one device per rank; SPRS_B200_COMM_MULTICAST=0 disables it) */
int sprs_b200_comm_multicast_supported(const sprs_b200_comm* comm);
/* all-gather of one small host record per rank (bytes <= 512): all = world * bytes */
int sprs_b200_comm_allgather_host(sprs_b200_comm* comm, const void* mine, uint64_t bytes,
                                  void* all);
int sprs_b200_comm_barrier_host(sprs_b200_comm* comm);
/* stream-ordered device barrier (one tiny kernel exchanging epoch flags in peer memory): what
 * every rank enqueued on its stream before its barrier -- e.g. the stores of its y rows into
 * the other ranks' buffers -- has completed when the barrier completes on any rank.        */
int sprs_b200_comm_barrier_dev(sprs_b200_comm* comm, void* stream);
/* synchronises `stream`; ERR_COMM if a device barrier gave up waiting for a peer */
int sprs_b200_comm_check(sprs_b200_comm* comm, void* stream);
/* `bytes` of zero-initialised device memory on every rank, every rank's buffer mapped into
 * every rank; with want_multicast (and support) also one multicast address whose stores the
 * switch replicates into all of them.                                                       */
int sprs_b200_symm_alloc(sprs_b200_comm* comm, uint64_t bytes, int want_multicast,
                         sprs_b200_symm** out);
int sprs_b200_symm_free(sprs_b200_symm* buf);
void* sprs_b200_symm_ptr(const sprs_b200_symm* buf, int rank);
void* sprs_b200_symm_multicast_ptr(const sprs_b200_symm* buf); /* NULL when not bound */
uint64_t sprs_b200_symm_bytes(const sprs_b200_symm* buf);
/* slice_outer cut points (slicing.rs:65-89): bounds[0..nparts], bounds[g] = first row whose
 * cost prefix nnz + row_cost*rows reaches g/nparts of the total (row_cost in non-zero
 * equivalents; 0 balances non-zeros only).  Host arrays, indptr width 4 or 8.             */
int sprs_b200_partition_rows(const void* indptr, int indptr_bytes, uint64_t rows, int nparts,
                             double row_cost, uint64_t* bounds);
/* How the rows of y reach the other ranks in spmv_rowpart: FUSED = the SpMV kernel delivers the
 * finished rows itself -- to ONE multicast address when y is multicast-bound (a store per row;
 * the row leaves the GPU once and the switch replicates it), otherwise to world-1 peer mappings
 * (the rows of a warp tile staged in shared memory, one TMA bulk store per peer and tile);
 * PUSH = plain SpMV, then one put kernel copying the rank's slice (coalesced 16-byte stores).
 * AUTO = the measured default (DESIGN.md 5).                                              */
enum { SPRS_B200_EXCHANGE_AUTO = 0, SPRS_B200_EXCHANGE_FUSED = 1, SPRS_B200_EXCHANGE_PUSH = 2,
       /* OR-ed into `exchange`: leave the closing device barrier to the caller (who then calls
        * sprs_b200_comm_barrier_dev on the same stream before y is read anywhere) */
       SPRS_B200_EXCHANGE_NO_BARRIER = 0x100 };
/* Row-partitioned y = A x (device-resident): this rank's CSR row block `mat` (rows
 * row_offset .. row_offset + mat.rows of A, slice_outer + proper_indptr), x replicated
 * (d_x: cols doubles on this device), y a symmetric buffer of n doubles.  Enqueues on
 * `stream`: SpMV of the block, the all-gather of the slice into EVERY rank's y, the device
 * barrier.  When that work has completed on a rank, its y holds the whole product.  A caller
 * that reads y and calls again must use two y buffers in turn (a fast rank stores rows of
 * product k+1 into a peer that may still read product k).                                  */
int sprs_b200_spmv_rowpart(sprs_b200_comm* comm, const sprs_b200_csmat* mat, const double* d_x,
                           sprs_b200_symm* y, uint64_t row_offset, int exchange, void* stream);
/* `&A * &x` on a row-partitioned matrix with HOST vectors, each rank touching only its own
 * slices: x_slice = x[col_offset .. col_offset+col_count) is uploaded into the symmetric x
 * buffer (cols doubles) and all-gathered over NVLink, the local block multiplied, y_slice
 * (this rank's mat.rows rows) downloaded.  Blocking; the union of the ranks' column slices
 * must cover 0..cols.                                                                       */
int sprs_b200_mul_mat_vec_rowpart(sprs_b200_comm* comm, const sprs_b200_csmat* mat,
                                  sprs_b200_symm* x, const double* x_slice, uint64_t col_offset,
                                  uint64_t col_count, double* y_slice, uint64_t y_len);

/* ---- sparse x sparse: smmp::mul_csr_csr (smmp.rs:196-237), two calls so the
 * CALLER allocates the output Vecs, like symbolic -> numeric (smmp.rs:81,151).
 * symbolic: pattern of C = A*B; returns a plan and nnz(C).
 * numeric : fills caller arrays: indptr (A.rows+1), indices (nnzC, ascending per
 *           row, structural zeros kept -- smmp.rs:109-129), data (nnzC).
 * Both operands must be CSR with A.cols == B.rows (else DIMENSION / STORAGE).
 * The plan BORROWS both operand mirrors: keep them alive until spgemm_free.         */
int sprs_b200_spgemm_symbolic(sprs_b200_ctx* ctx, const sprs_b200_csmat* a,
                              const sprs_b200_csmat* b, sprs_b200_spgemm** plan,
                              uint64_t* nnz_c);
int sprs_b200_spgemm_numeric(sprs_b200_ctx* ctx, sprs_b200_spgemm* plan, void* c_indptr,
                             int indptr_bytes, void* c_indices, int index_bytes,
                             double* c_data);
/* same, leaving C on the device as a new mirror (plan may then be freed) */
int sprs_b200_spgemm_numeric_dev(sprs_b200_ctx* ctx, sprs_b200_spgemm* plan,
                                 sprs_b200_csmat** c);
/* work counters of a plan: n_prod = sum_i sum_{k in A_i} nnz(B_k) */
uint64_t sprs_b200_spgemm_nprod(const sprs_b200_spgemm* plan);
int sprs_b200_spgemm_free(sprs_b200_spgemm* plan);

/* ---- BiCGSTAB with device-resident vectors (SURVEY.md 8f rank 3) ---------------
 * Replaces sprs::linalg::bicgstab::BiCGSTAB<f64> (linalg/bicgstab.rs:95-300): `new`
 * (:120-146) computes r = b - A x0, rhat = p = r, err = |r|, rho = err^2; `step`
 * (:198-234), `soft_restart` (:177-184), `hard_restart` (:186-196) and `solve`
 * (:151-175) follow the reference operation by operation (unfused multiply/add; dot
 * products summed in a fixed order, so repeatable, but not the reference's strictly
 * sequential order: values agree to rounding).  x, r, rhat, p, b stay in HBM across
 * iterations; a step moves three 16-byte scalar pairs to the host.
 * The matrix may be CSR or CSC (both sum A*v in ascending column order) and must be
 * square with n rows (else DIMENSION, the reference's "Dimension mismatch" panic).  The
 * solver BORROWS the matrix mirror: keep it alive until bicgstab_free.  x0 and b are
 * copied (host pointers for _new, device pointers for _new_dev).  _new_dev copies them on
 * the ctx's own stream and takes no stream argument, so the device arrays must be COMPLETE
 * when the call is made: synchronise the stream that produced them first.              */
typedef struct sprs_b200_bicgstab sprs_b200_bicgstab;
enum {
    SPRS_B200_BICGSTAB_X = 0,    /* x()    latest solution            (bicgstab.rs:272) */
    SPRS_B200_BICGSTAB_R = 1,    /* r()    latest residual            (:282)            */
    SPRS_B200_BICGSTAB_RHAT = 2, /* rhat() reference direction        (:290)            */
    SPRS_B200_BICGSTAB_P = 3,    /* p()    step direction             (:295)            */
    SPRS_B200_BICGSTAB_B = 4     /* b()    the objective vector       (:277)            */
};
int sprs_b200_bicgstab_new(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat, const double* x0,
                           const double* b, uint64_t n, sprs_b200_bicgstab** out);
int sprs_b200_bicgstab_new_dev(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat,
                               const double* d_x0, const double* d_b, uint64_t n,
                               sprs_b200_bicgstab** out);
/* Operator form: y = A x is delegated to `matvec` (called with device pointers to n doubles
 * each and the stream the solver works on; it must ENQUEUE y = A x on that stream and return
 * 0).  This is how the solver runs on a row-partitioned matrix: the callback is the
 * distributed SpMV + all-gather of y (sprs_b200/dist.py), every rank keeps full-length
 * vectors and computes the same dot products in the same order, so all ranks take the same
 * steps and restarts without exchanging a scalar.  x0 / b: host pointers, or device pointers
 * when device_pointers != 0.                                                              */
typedef int (*sprs_b200_matvec_fn)(void* user, const double* d_x, double* d_y, void* stream);
int sprs_b200_bicgstab_new_op(sprs_b200_ctx* ctx, uint64_t n, sprs_b200_matvec_fn matvec,
                              void* user, const double* x0, const double* b,
                              int device_pointers, sprs_b200_bicgstab** out);
int sprs_b200_bicgstab_free(sprs_b200_bicgstab* s);
/* one iteration; *err_out (optional) = the running error estimate |r| */
int sprs_b200_bicgstab_step(sprs_b200_bicgstab* s, double* err_out);
int sprs_b200_bicgstab_soft_restart(sprs_b200_bicgstab* s);
int sprs_b200_bicgstab_hard_restart(sprs_b200_bicgstab* s);
/* up to max_iter steps; *converged = 1 (Ok) when the TRUE error |b - A x| < tol was
 * confirmed by a hard restart, 0 (Err) when the iteration limit was reached.          */
int sprs_b200_bicgstab_solve(sprs_b200_bicgstab* s, double tol, uint64_t max_iter,
                             int* converged);
int sprs_b200_bicgstab_set_restart_threshold(sprs_b200_bicgstab* s, double thresh);
/* counts = {iteration_count, soft_restart_count, hard_restart_count};
 * scalars = {err, rho, soft_restart_threshold}; either may be NULL                    */
int sprs_b200_bicgstab_stats(const sprs_b200_bicgstab* s, uint64_t counts[3],
                             double scalars[3]);
/* copy vector `which` (enum above) to a host array of len == n */
int sprs_b200_bicgstab_get(const sprs_b200_bicgstab* s, int which, double* out, uint64_t len);
/* borrowed device pointer to vector `which` (valid until bicgstab_free) */
int sprs_b200_bicgstab_get_dev(const sprs_b200_bicgstab* s, int which, const double** d_out);

/* ---- sparse triangular solves with a dense right-hand side (sprs::linalg::trisolve,
 * linalg/trisolve.rs): lsolve_csr_dense_rhs (:30-73), usolve_csr_dense_rhs (:219-262),
 * lsolve_csc_dense_rhs (:85-149), usolve_csc_dense_rhs (:161-210).  Entries of the other
 * triangle are ignored.  Every row is x_r = b_r, x_r = x_r - a_rc * x_c over its terms in the
 * reference's order (ascending column; descending for usolve_csc), then x_r / diag, each
 * operation rounded on its own: the result is bit-identical to the reference.
 * A plan is built once per matrix and triangle: it finds every row's diagonal and the first
 * singular row or column in processing order (diagonal missing or == 0; -0.0 counts as zero,
 * NaN does not).  The plan BORROWS the mirror and READS ITS VALUES when it is built: the
 * mirror must be kept alive and unchanged until trisolve_free.  A CSC plan owns a device
 * transpose of the mirror.                                                                  */
typedef struct sprs_b200_trisolve sprs_b200_trisolve;
enum { SPRS_B200_TRI_LOWER = 0, SPRS_B200_TRI_UPPER = 1 };
/* the reason of a SingularMatrix, chosen from (storage, triangle) as the reference does:
 * IS_ZERO "diagonal element is 0" (lsolve_csr), NUMERIC "diagonal element is a numeric 0"
 * (usolve_csr; CSC forms with a stored 0), STRUCTURAL "diagonal element is a structural 0"
 * (CSC forms without a stored diagonal)                                                      */
enum {
    SPRS_B200_SINGULAR_IS_ZERO = 0,
    SPRS_B200_SINGULAR_NUMERIC = 1,
    SPRS_B200_SINGULAR_STRUCTURAL = 2
};
/* ERR_DIMENSION if the matrix is not square, ERR_ARGUMENT for a bad triangle.  Blocking. */
int sprs_b200_trisolve_plan(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat, int tri,
                            sprs_b200_trisolve** out);
/* 1 and (index, reason) when a solve with this plan returns ERR_SINGULAR, else 0 */
int sprs_b200_trisolve_singular(const sprs_b200_trisolve* plan, uint64_t* index, int* reason);
/* rhs (host, len doubles) solved in place; blocking.  ERR_DIMENSION if len != n.  A singular
 * plan returns ERR_SINGULAR after leaving rhs as the reference does: rows processed before the
 * singular index solved, the others untouched (CSR) or holding b_r minus the terms of the
 * columns processed before it (CSC).  Waits between rows are bounded by progress: ERR_CUDA
 * (x incomplete) only if no row of the whole solve moved for ~9 s of GPU clock -- a bug report,
 * never a valid input, however long a single wait lasts.  The plan stays usable after it.    */
int sprs_b200_trisolve_solve(sprs_b200_trisolve* plan, double* rhs, uint64_t len);
/* the same on a device vector of n doubles, enqueued on `stream` (asynchronous, like
 * spmv_dev); returns ERR_SINGULAR (after enqueueing the same work) when the plan is singular.
 * One stream at a time per plan.  A breach of the wait bound in a solve_dev is reported
 * (ERR_CUDA, once) by the next solve or solve_dev of the plan, before it enqueues anything.  */
int sprs_b200_trisolve_solve_dev(sprs_b200_trisolve* plan, double* d_rhs, void* stream);
/* waits for the last solve enqueued with the plan (on its stream), then frees it */
int sprs_b200_trisolve_free(sprs_b200_trisolve* plan);

/* ---- measurement aid (bench.py roofline.gather_ceiling; not a product path): the SpMV's
 * memory behaviour on THIS matrix with the row logic removed -- the same (index, value) stream
 * and the same x gathers, one plain sum per lane, no rows, no y (csrc/diag.cu).  Any SpMV that
 * gathers x through L1/L2 does at least this work: nnz_covered / ms_per_pass is the ceiling
 * the product kernel is held against.  Blocking; `iters` timed passes after two warm-ups.   */
int sprs_b200_diag_gather_ceiling(sprs_b200_ctx* ctx, const sprs_b200_csmat* mat,
                                  const double* d_x, int iters, double* ms_per_pass,
                                  uint64_t* nnz_covered);

/* ---- synthetic inputs, generated in HBM (SURVEY.md 8d; sprs-rand/src/lib.rs:24-81
 * gives the uniform distribution; R-MAT is this repo's definition).  Each writes
 * `count` 64-bit keys (row<<32 | col) for candidate edges [first, first+count);
 * rejected candidates (index >= n) get key UINT64_MAX.  Sorting/dedup is the
 * caller's job (bench plumbing).                                                  */
int sprs_b200_gen_rmat_keys(sprs_b200_ctx* ctx, uint64_t seed, int scale, uint64_t n_rows,
                            uint64_t n_cols, double a, double b, double c, uint64_t first,
                            uint64_t count, uint64_t* d_keys, void* stream);
int sprs_b200_gen_uniform_keys(sprs_b200_ctx* ctx, uint64_t seed, uint64_t n_rows,
                               uint64_t n_cols, uint64_t first, uint64_t count,
                               uint64_t* d_keys, void* stream);
/* N(0,1) value per key (hash of key and seed): partition independent */
int sprs_b200_gen_normal_from_keys(sprs_b200_ctx* ctx, uint64_t seed, const uint64_t* d_keys,
                                   uint64_t count, double* d_out, void* stream);
/* split sorted unique keys into u32 row / col arrays (row optional) */
int sprs_b200_gen_split_keys(sprs_b200_ctx* ctx, const uint64_t* d_keys, uint64_t count,
                             uint32_t* d_rows, uint32_t* d_cols, void* stream);
/* 64-bit mix of each key (for thinning to an exact nnz) */
int sprs_b200_gen_hash_keys(sprs_b200_ctx* ctx, uint64_t seed, const uint64_t* d_keys,
                            uint64_t count, uint64_t* d_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SPRS_B200_H */
