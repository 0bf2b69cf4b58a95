//! Raw declarations of include/sprs_b200.h.  Conventions follow the in-tree FFI
//! precedent `prod_nnz` (sprs-benches/src/main.rs:27-42): plain scalars, raw pointers,
//! zero-based indptr, caller-owned host buffers; opaque handles freed explicitly
//! (suitesparse_umfpack_sys/src/umfpack_free_numeric.rs:3-6).
#![allow(non_camel_case_types)]
use std::os::raw::{c_char, c_double, c_int, c_void};

#[repr(C)] pub struct sprs_b200_ctx { _private: [u8; 0] }
#[repr(C)] pub struct sprs_b200_csmat { _private: [u8; 0] }
#[repr(C)] pub struct sprs_b200_spgemm { _private: [u8; 0] }
#[repr(C)] pub struct sprs_b200_comm { _private: [u8; 0] }
#[repr(C)] pub struct sprs_b200_symm { _private: [u8; 0] }
#[repr(C)] pub struct sprs_b200_bicgstab { _private: [u8; 0] }
#[repr(C)] pub struct sprs_b200_trisolve { _private: [u8; 0] }

pub const SPRS_B200_CSR: c_int = 0;
pub const SPRS_B200_CSC: c_int = 1;
pub const SPRS_B200_BINOP_ADD: c_int = 0;
pub const SPRS_B200_BINOP_SUB: c_int = 1;
pub const SPRS_B200_BINOP_MUL: c_int = 2;
pub const SPRS_B200_OK: c_int = 0;
pub const SPRS_B200_ERR_DIMENSION: c_int = 1;
pub const SPRS_B200_ERR_STORAGE: c_int = 2;
pub const SPRS_B200_ERR_CUDA: c_int = 3;
pub const SPRS_B200_ERR_NCCL: c_int = 4;
pub const SPRS_B200_ERR_INDEX_RANGE: c_int = 5;
pub const SPRS_B200_ERR_ARGUMENT: c_int = 6;
pub const SPRS_B200_ERR_STRUCTURE: c_int = 7;
pub const SPRS_B200_ERR_UNSUPPORTED: c_int = 8;
pub const SPRS_B200_ERR_SINGULAR: c_int = 10;
pub const SPRS_B200_TRI_LOWER: c_int = 0;
pub const SPRS_B200_TRI_UPPER: c_int = 1;
pub const SPRS_B200_SINGULAR_IS_ZERO: c_int = 0;
pub const SPRS_B200_SINGULAR_NUMERIC: c_int = 1;
pub const SPRS_B200_SINGULAR_STRUCTURAL: c_int = 2;
pub const SPRS_B200_BICGSTAB_X: c_int = 0;
pub const SPRS_B200_BICGSTAB_R: c_int = 1;
pub const SPRS_B200_BICGSTAB_RHAT: c_int = 2;
pub const SPRS_B200_BICGSTAB_P: c_int = 3;
pub const SPRS_B200_BICGSTAB_B: c_int = 4;

/// y = A x callback of the operator-form solver: device pointers to n doubles, a cudaStream_t.
pub type sprs_b200_matvec_fn = Option<unsafe extern "C" fn(
    user: *mut c_void, d_x: *const c_double, d_y: *mut c_double, stream: *mut c_void) -> c_int>;

extern "C" {
    pub fn sprs_b200_version() -> c_int;
    pub fn sprs_b200_ctx_create(device: c_int, out: *mut *mut sprs_b200_ctx) -> c_int;
    pub fn sprs_b200_ctx_destroy(ctx: *mut sprs_b200_ctx) -> c_int;
    pub fn sprs_b200_last_error(ctx: *const sprs_b200_ctx) -> *const c_char;
    pub fn sprs_b200_csmat_upload(
        ctx: *mut sprs_b200_ctx, storage: c_int, rows: u64, cols: u64,
        indptr: *const c_void, indptr_bytes: c_int,
        indices: *const c_void, index_bytes: c_int,
        data: *const c_double, out: *mut *mut sprs_b200_csmat) -> c_int;
    pub fn sprs_b200_csmat_free(m: *mut sprs_b200_csmat) -> c_int;
    pub fn sprs_b200_csmat_nnz(m: *const sprs_b200_csmat) -> u64;
    pub fn sprs_b200_csmat_download(
        ctx: *mut sprs_b200_ctx, m: *const sprs_b200_csmat, indptr: *mut c_void,
        indptr_bytes: c_int, indices: *mut c_void, index_bytes: c_int, data: *mut c_double) -> c_int;
    pub fn sprs_b200_csmat_to_other_storage(
        ctx: *mut sprs_b200_ctx, m: *const sprs_b200_csmat, out: *mut *mut sprs_b200_csmat) -> c_int;
    pub fn sprs_b200_csmat_binop(
        ctx: *mut sprs_b200_ctx, lhs: *const sprs_b200_csmat, rhs: *const sprs_b200_csmat,
        op: c_int, out: *mut *mut sprs_b200_csmat) -> c_int;
    pub fn sprs_b200_csmat_scale(
        ctx: *mut sprs_b200_ctx, m: *const sprs_b200_csmat, s: c_double,
        out: *mut *mut sprs_b200_csmat) -> c_int;
    pub fn sprs_b200_mul_acc_mat_vec_csr(
        ctx: *mut sprs_b200_ctx, mat: *const sprs_b200_csmat, in_vec: *const c_double, in_len: u64,
        res_vec: *mut c_double, res_len: u64) -> c_int;
    pub fn sprs_b200_mul_acc_mat_vec_csc(
        ctx: *mut sprs_b200_ctx, mat: *const sprs_b200_csmat, in_vec: *const c_double, in_len: u64,
        res_vec: *mut c_double, res_len: u64) -> c_int;
    pub fn sprs_b200_mul_mat_vec(
        ctx: *mut sprs_b200_ctx, mat: *const sprs_b200_csmat, x: *const c_double, x_len: u64,
        y: *mut c_double, y_len: u64) -> c_int;
    pub fn sprs_b200_csr_mul_csvec(
        ctx: *mut sprs_b200_ctx, mat: *const sprs_b200_csmat, dim: u64, v_nnz: u64,
        v_indices: *const c_void, index_bytes: c_int, v_data: *const c_double,
        res: *mut c_double, res_len: u64) -> c_int;
    pub fn sprs_b200_csr_mul_csvec_acc(
        ctx: *mut sprs_b200_ctx, mat: *const sprs_b200_csmat, dim: u64, v_nnz: u64,
        v_indices: *const c_void, index_bytes: c_int, v_data: *const c_double,
        res: *mut c_double, res_len: u64) -> c_int;
    pub fn sprs_b200_csr_mulacc_dense_rowmaj(
        ctx: *mut sprs_b200_ctx, lhs: *const sprs_b200_csmat, rhs: *const c_double,
        rhs_rows: u64, rhs_cols: u64, rhs_rs: i64, rhs_cs: i64, out: *mut c_double,
        out_rows: u64, out_cols: u64, out_rs: i64, out_cs: i64) -> c_int;
    pub fn sprs_b200_csr_mulacc_dense_colmaj(
        ctx: *mut sprs_b200_ctx, lhs: *const sprs_b200_csmat, rhs: *const c_double,
        rhs_rows: u64, rhs_cols: u64, rhs_rs: i64, rhs_cs: i64, out: *mut c_double,
        out_rows: u64, out_cols: u64, out_rs: i64, out_cs: i64) -> c_int;
    pub fn sprs_b200_csc_mulacc_dense_rowmaj(
        ctx: *mut sprs_b200_ctx, lhs: *const sprs_b200_csmat, rhs: *const c_double,
        rhs_rows: u64, rhs_cols: u64, rhs_rs: i64, rhs_cs: i64, out: *mut c_double,
        out_rows: u64, out_cols: u64, out_rs: i64, out_cs: i64) -> c_int;
    pub fn sprs_b200_csc_mulacc_dense_colmaj(
        ctx: *mut sprs_b200_ctx, lhs: *const sprs_b200_csmat, rhs: *const c_double,
        rhs_rows: u64, rhs_cols: u64, rhs_rs: i64, rhs_cs: i64, out: *mut c_double,
        out_rows: u64, out_cols: u64, out_rs: i64, out_cs: i64) -> c_int;
    pub fn sprs_b200_spgemm_symbolic(
        ctx: *mut sprs_b200_ctx, a: *const sprs_b200_csmat, b: *const sprs_b200_csmat,
        plan: *mut *mut sprs_b200_spgemm, nnz_c: *mut u64) -> c_int;
    pub fn sprs_b200_spgemm_numeric(
        ctx: *mut sprs_b200_ctx, plan: *mut sprs_b200_spgemm, c_indptr: *mut c_void,
        indptr_bytes: c_int, c_indices: *mut c_void, index_bytes: c_int, c_data: *mut c_double) -> c_int;
    pub fn sprs_b200_spgemm_free(plan: *mut sprs_b200_spgemm) -> c_int;
    // linalg::bicgstab::BiCGSTAB<f64> with device-resident vectors (bicgstab.rs:95-300)
    pub fn sprs_b200_bicgstab_new(
        ctx: *mut sprs_b200_ctx, mat: *const sprs_b200_csmat, x0: *const c_double,
        b: *const c_double, n: u64, out: *mut *mut sprs_b200_bicgstab) -> c_int;
    pub fn sprs_b200_bicgstab_new_op(
        ctx: *mut sprs_b200_ctx, n: u64, matvec: sprs_b200_matvec_fn, user: *mut c_void,
        x0: *const c_double, b: *const c_double, device_pointers: c_int,
        out: *mut *mut sprs_b200_bicgstab) -> c_int;
    pub fn sprs_b200_bicgstab_free(s: *mut sprs_b200_bicgstab) -> c_int;
    // linalg::trisolve dense-rhs solves (trisolve.rs:30-262); the plan borrows the mirror
    pub fn sprs_b200_trisolve_plan(
        ctx: *mut sprs_b200_ctx, mat: *const sprs_b200_csmat, tri: c_int,
        out: *mut *mut sprs_b200_trisolve) -> c_int;
    pub fn sprs_b200_trisolve_singular(
        plan: *const sprs_b200_trisolve, index: *mut u64, reason: *mut c_int) -> c_int;
    pub fn sprs_b200_trisolve_solve(plan: *mut sprs_b200_trisolve, rhs: *mut c_double, len: u64) -> c_int;
    pub fn sprs_b200_trisolve_solve_dev(
        plan: *mut sprs_b200_trisolve, d_rhs: *mut c_double, stream: *mut c_void) -> c_int;
    pub fn sprs_b200_trisolve_free(plan: *mut sprs_b200_trisolve) -> c_int;
    pub fn sprs_b200_bicgstab_step(s: *mut sprs_b200_bicgstab, err_out: *mut c_double) -> c_int;
    pub fn sprs_b200_bicgstab_soft_restart(s: *mut sprs_b200_bicgstab) -> c_int;
    pub fn sprs_b200_bicgstab_hard_restart(s: *mut sprs_b200_bicgstab) -> c_int;
    pub fn sprs_b200_bicgstab_solve(
        s: *mut sprs_b200_bicgstab, tol: c_double, max_iter: u64, converged: *mut c_int) -> c_int;
    pub fn sprs_b200_bicgstab_set_restart_threshold(s: *mut sprs_b200_bicgstab, thresh: c_double) -> c_int;
    pub fn sprs_b200_bicgstab_stats(
        s: *const sprs_b200_bicgstab, counts: *mut u64, scalars: *mut c_double) -> c_int;
    pub fn sprs_b200_bicgstab_get(
        s: *const sprs_b200_bicgstab, which: c_int, out: *mut c_double, len: u64) -> c_int;
    // ---- the rest of include/sprs_b200.h: device-resident entry points, the device COO->CSR,
    // multi-GPU plumbing (one process per GPU) and the synthetic-input generators
    pub fn sprs_b200_ctx_device(ctx: *const sprs_b200_ctx) -> c_int;
    pub fn sprs_b200_ctx_sm_count(ctx: *const sprs_b200_ctx) -> c_int;
    pub fn sprs_b200_ctx_synchronize(ctx: *mut sprs_b200_ctx) -> c_int;
    pub fn sprs_b200_csmat_from_device(
        ctx: *mut sprs_b200_ctx, storage: c_int, rows: u64, cols: u64, nnz: u64,
        d_indptr: *const u32, d_indices: *const u32, d_data: *const c_double,
        out: *mut *mut sprs_b200_csmat) -> c_int;
    pub fn sprs_b200_csmat_storage(m: *const sprs_b200_csmat) -> c_int;
    pub fn sprs_b200_csmat_rows(m: *const sprs_b200_csmat) -> u64;
    pub fn sprs_b200_csmat_cols(m: *const sprs_b200_csmat) -> u64;
    pub fn sprs_b200_csmat_device_arrays(
        m: *const sprs_b200_csmat, d_indptr: *mut *const c_void, indptr_bytes: *mut c_int,
        d_indices: *mut *const u32, d_data: *mut *const c_double) -> c_int;
    pub fn sprs_b200_csmat_from_triplets(
        ctx: *mut sprs_b200_ctx, rows: u64, cols: u64, n: u64, row_inds: *const c_void,
        col_inds: *const c_void, index_bytes: c_int, data: *const c_double,
        out: *mut *mut sprs_b200_csmat) -> c_int;
    pub fn sprs_b200_csmat_from_triplets_dev(
        ctx: *mut sprs_b200_ctx, rows: u64, cols: u64, n: u64, d_row: *const u32,
        d_col: *const u32, d_val: *const c_double, out: *mut *mut sprs_b200_csmat) -> c_int;
    pub fn sprs_b200_csmat_check_structure(
        ctx: *mut sprs_b200_ctx, m: *const sprs_b200_csmat, n_violations: *mut u64) -> c_int;
    pub fn sprs_b200_spmv_dev(
        ctx: *mut sprs_b200_ctx, mat: *const sprs_b200_csmat, d_x: *const c_double,
        d_y: *mut c_double, accumulate: c_int, stream: *mut c_void) -> c_int;
    pub fn sprs_b200_spmm_rowmaj_dev(
        ctx: *mut sprs_b200_ctx, mat: *const sprs_b200_csmat, d_b: *const c_double, ldb: u64,
        k: u64, d_c: *mut c_double, ldc: u64, accumulate: c_int, stream: *mut c_void) -> c_int;
    pub fn sprs_b200_launch_count(ctx: *const sprs_b200_ctx) -> u64;
    pub fn sprs_b200_peer_alloc(
        ctx: *mut sprs_b200_ctx, bytes: u64, d_ptr: *mut *mut c_void, ipc_handle: *mut u8) -> c_int;
    pub fn sprs_b200_peer_open(
        ctx: *mut sprs_b200_ctx, ipc_handle: *const u8, d_ptr: *mut *mut c_void) -> c_int;
    pub fn sprs_b200_peer_close(ctx: *mut sprs_b200_ctx, d_ptr: *mut c_void) -> c_int;
    pub fn sprs_b200_peer_free(ctx: *mut sprs_b200_ctx, d_ptr: *mut c_void) -> c_int;
    pub fn sprs_b200_copy_dev(
        ctx: *mut sprs_b200_ctx, dst: *mut c_void, src: *const c_void, bytes: u64,
        stream: *mut c_void) -> c_int;
    pub fn sprs_b200_peer_push_dev(
        ctx: *mut sprs_b200_ctx, d_y_own: *const c_double, row_offset: u64, rows: u64,
        n_peers: c_int, d_y_peers: *const *mut c_double, stream: *mut c_void) -> c_int;
    pub fn sprs_b200_spmv_allgather_dev(
        ctx: *mut sprs_b200_ctx, mat: *const sprs_b200_csmat, d_x: *const c_double,
        row_offset: u64, n_targets: c_int, d_y_bufs: *const *mut c_double, accumulate: c_int,
        stream: *mut c_void) -> c_int;
    pub fn sprs_b200_copy_to_device(
        ctx: *mut sprs_b200_ctx, d_dst: *mut c_void, h_src: *const c_void, bytes: u64,
        stream: *mut c_void) -> c_int;
    pub fn sprs_b200_copy_to_host(
        ctx: *mut sprs_b200_ctx, h_dst: *mut c_void, d_src: *const c_void, bytes: u64,
        stream: *mut c_void) -> c_int;
    // ---- multi-GPU communicator (one node; ranks = processes or threads; include/sprs_b200.h)
    pub fn sprs_b200_comm_unique_id(id: *mut c_char) -> c_int;
    pub fn sprs_b200_comm_init_rank(
        ctx: *mut sprs_b200_ctx, id: *const c_char, rank: c_int, world: c_int,
        out: *mut *mut sprs_b200_comm) -> c_int;
    pub fn sprs_b200_comm_free(comm: *mut sprs_b200_comm) -> c_int;
    pub fn sprs_b200_comm_rank(comm: *const sprs_b200_comm) -> c_int;
    pub fn sprs_b200_comm_world(comm: *const sprs_b200_comm) -> c_int;
    pub fn sprs_b200_comm_multicast_supported(comm: *const sprs_b200_comm) -> c_int;
    pub fn sprs_b200_comm_allgather_host(
        comm: *mut sprs_b200_comm, mine: *const c_void, bytes: u64, all: *mut c_void) -> c_int;
    pub fn sprs_b200_comm_barrier_host(comm: *mut sprs_b200_comm) -> c_int;
    pub fn sprs_b200_comm_barrier_dev(comm: *mut sprs_b200_comm, stream: *mut c_void) -> c_int;
    pub fn sprs_b200_comm_check(comm: *mut sprs_b200_comm, stream: *mut c_void) -> c_int;
    pub fn sprs_b200_symm_alloc(
        comm: *mut sprs_b200_comm, bytes: u64, want_multicast: c_int,
        out: *mut *mut sprs_b200_symm) -> c_int;
    pub fn sprs_b200_symm_free(buf: *mut sprs_b200_symm) -> c_int;
    pub fn sprs_b200_symm_ptr(buf: *const sprs_b200_symm, rank: c_int) -> *mut c_void;
    pub fn sprs_b200_symm_multicast_ptr(buf: *const sprs_b200_symm) -> *mut c_void;
    pub fn sprs_b200_symm_bytes(buf: *const sprs_b200_symm) -> u64;
    pub fn sprs_b200_partition_rows(
        indptr: *const c_void, indptr_bytes: c_int, rows: u64, nparts: c_int, row_cost: c_double,
        bounds: *mut u64) -> c_int;
    pub fn sprs_b200_spmv_rowpart(
        comm: *mut sprs_b200_comm, mat: *const sprs_b200_csmat, d_x: *const c_double,
        y: *mut sprs_b200_symm, row_offset: u64, exchange: c_int, stream: *mut c_void) -> c_int;
    pub fn sprs_b200_mul_mat_vec_rowpart(
        comm: *mut sprs_b200_comm, mat: *const sprs_b200_csmat, x: *mut sprs_b200_symm,
        x_slice: *const c_double, col_offset: u64, col_count: u64, y_slice: *mut c_double,
        y_len: u64) -> c_int;
    pub fn sprs_b200_diag_gather_ceiling(
        ctx: *mut sprs_b200_ctx, mat: *const sprs_b200_csmat, d_x: *const c_double, iters: c_int,
        ms_per_pass: *mut c_double, nnz_covered: *mut u64) -> c_int;
    pub fn sprs_b200_spmv_chunked_push_dev(
        ctx: *mut sprs_b200_ctx, mat: *const sprs_b200_csmat, d_x: *const c_double,
        row_offset: u64, n_targets: c_int, d_y_bufs: *const *mut c_double, accumulate: c_int,
        n_chunks: c_int, stream: *mut c_void) -> c_int;
    pub fn sprs_b200_spgemm_numeric_dev(
        ctx: *mut sprs_b200_ctx, plan: *mut sprs_b200_spgemm, c: *mut *mut sprs_b200_csmat) -> c_int;
    pub fn sprs_b200_spgemm_nprod(plan: *const sprs_b200_spgemm) -> u64;
    pub fn sprs_b200_bicgstab_new_dev(
        ctx: *mut sprs_b200_ctx, mat: *const sprs_b200_csmat, d_x0: *const c_double,
        d_b: *const c_double, n: u64, out: *mut *mut sprs_b200_bicgstab) -> c_int;
    pub fn sprs_b200_bicgstab_get_dev(
        s: *const sprs_b200_bicgstab, which: c_int, d_out: *mut *const c_double) -> c_int;
    pub fn sprs_b200_gen_rmat_keys(
        ctx: *mut sprs_b200_ctx, seed: u64, scale: c_int, n_rows: u64, n_cols: u64, a: c_double,
        b: c_double, c: c_double, first: u64, count: u64, d_keys: *mut u64, stream: *mut c_void) -> c_int;
    pub fn sprs_b200_gen_uniform_keys(
        ctx: *mut sprs_b200_ctx, seed: u64, n_rows: u64, n_cols: u64, first: u64, count: u64,
        d_keys: *mut u64, stream: *mut c_void) -> c_int;
    pub fn sprs_b200_gen_normal_from_keys(
        ctx: *mut sprs_b200_ctx, seed: u64, d_keys: *const u64, count: u64, d_out: *mut c_double,
        stream: *mut c_void) -> c_int;
    pub fn sprs_b200_gen_split_keys(
        ctx: *mut sprs_b200_ctx, d_keys: *const u64, count: u64, d_rows: *mut u32,
        d_cols: *mut u32, stream: *mut c_void) -> c_int;
    pub fn sprs_b200_gen_hash_keys(
        ctx: *mut sprs_b200_ctx, seed: u64, d_keys: *const u64, count: u64, d_out: *mut u64,
        stream: *mut c_void) -> c_int;
}
