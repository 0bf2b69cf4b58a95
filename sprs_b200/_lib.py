"""ctypes binding of libsprs_b200.so -- the same C ABI (include/sprs_b200.h) a Rust
`sprs-b200-sys` crate binds.  Loading fails loudly when the library is missing:
there is no CPU fallback anywhere in this package."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsprs_b200.so")

OK, ERR_DIMENSION, ERR_STORAGE, ERR_CUDA, ERR_NCCL, ERR_INDEX_RANGE, ERR_ARGUMENT, \
    ERR_STRUCTURE, ERR_UNSUPPORTED = range(9)
CSR, CSC = 0, 1
BINOP_ADD, BINOP_SUB, BINOP_MUL = 0, 1, 2
ERR_SINGULAR = 10
TRI_LOWER, TRI_UPPER = 0, 1
SINGULAR_IS_ZERO, SINGULAR_NUMERIC, SINGULAR_STRUCTURAL = 0, 1, 2

_vp, _u64, _i64, _int, _dp = C.c_void_p, C.c_uint64, C.c_int64, C.c_int, C.c_void_p
_dense_sig = [_vp, _vp, _dp, _u64, _u64, _i64, _i64, _dp, _u64, _u64, _i64, _i64]

# sprs_b200_matvec_fn: int (*)(void* user, const double* d_x, double* d_y, void* stream)
MATVEC_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p)

# name -> (restype, argtypes); one entry per symbol declared in include/sprs_b200.h
PROTOTYPES = {
    "sprs_b200_version": (_int, []),
    "sprs_b200_ctx_create": (_int, [_int, C.POINTER(_vp)]),
    "sprs_b200_ctx_destroy": (_int, [_vp]),
    "sprs_b200_last_error": (C.c_char_p, [_vp]),
    "sprs_b200_ctx_device": (_int, [_vp]),
    "sprs_b200_ctx_sm_count": (_int, [_vp]),
    "sprs_b200_ctx_synchronize": (_int, [_vp]),
    "sprs_b200_csmat_upload": (_int, [_vp, _int, _u64, _u64, _vp, _int, _vp, _int, _dp,
                                      C.POINTER(_vp)]),
    "sprs_b200_csmat_from_device": (_int, [_vp, _int, _u64, _u64, _u64, _vp, _vp, _vp,
                                           C.POINTER(_vp)]),
    "sprs_b200_csmat_free": (_int, [_vp]),
    "sprs_b200_csmat_storage": (_int, [_vp]),
    "sprs_b200_csmat_rows": (_u64, [_vp]),
    "sprs_b200_csmat_cols": (_u64, [_vp]),
    "sprs_b200_csmat_nnz": (_u64, [_vp]),
    "sprs_b200_csmat_download": (_int, [_vp, _vp, _vp, _int, _vp, _int, _dp]),
    "sprs_b200_csmat_device_arrays": (_int, [_vp, C.POINTER(_vp), C.POINTER(_int),
                                             C.POINTER(_vp), C.POINTER(_vp)]),
    "sprs_b200_csmat_from_triplets": (_int, [_vp, _u64, _u64, _u64, _vp, _vp, _int, _dp,
                                             C.POINTER(_vp)]),
    "sprs_b200_csmat_from_triplets_dev": (_int, [_vp, _u64, _u64, _u64, _vp, _vp, _vp,
                                                 C.POINTER(_vp)]),
    "sprs_b200_csmat_check_structure": (_int, [_vp, _vp, C.POINTER(_u64)]),
    "sprs_b200_csmat_to_other_storage": (_int, [_vp, _vp, C.POINTER(_vp)]),
    "sprs_b200_csmat_binop": (_int, [_vp, _vp, _vp, _int, C.POINTER(_vp)]),
    "sprs_b200_csmat_scale": (_int, [_vp, _vp, C.c_double, C.POINTER(_vp)]),
    "sprs_b200_mul_acc_mat_vec_csr": (_int, [_vp, _vp, _dp, _u64, _dp, _u64]),
    "sprs_b200_mul_acc_mat_vec_csc": (_int, [_vp, _vp, _dp, _u64, _dp, _u64]),
    "sprs_b200_mul_mat_vec": (_int, [_vp, _vp, _dp, _u64, _dp, _u64]),
    "sprs_b200_csr_mul_csvec": (_int, [_vp, _vp, _u64, _u64, _vp, _int, _dp, _dp, _u64]),
    "sprs_b200_csr_mul_csvec_acc": (_int, [_vp, _vp, _u64, _u64, _vp, _int, _dp, _dp, _u64]),
    "sprs_b200_csr_mulacc_dense_rowmaj": (_int, _dense_sig),
    "sprs_b200_csr_mulacc_dense_colmaj": (_int, _dense_sig),
    "sprs_b200_csc_mulacc_dense_rowmaj": (_int, _dense_sig),
    "sprs_b200_csc_mulacc_dense_colmaj": (_int, _dense_sig),
    "sprs_b200_spmv_dev": (_int, [_vp, _vp, _dp, _dp, _int, _vp]),
    "sprs_b200_spmm_rowmaj_dev": (_int, [_vp, _vp, _dp, _u64, _u64, _dp, _u64, _int, _vp]),
    "sprs_b200_launch_count": (_u64, [_vp]),
    "sprs_b200_peer_alloc": (_int, [_vp, _u64, C.POINTER(_vp), C.c_char_p]),
    "sprs_b200_peer_open": (_int, [_vp, C.c_char_p, C.POINTER(_vp)]),
    "sprs_b200_peer_close": (_int, [_vp, _vp]),
    "sprs_b200_peer_free": (_int, [_vp, _vp]),
    "sprs_b200_copy_dev": (_int, [_vp, _vp, _vp, _u64, _vp]),
    "sprs_b200_copy_to_device": (_int, [_vp, _vp, _vp, _u64, _vp]),
    "sprs_b200_copy_to_host": (_int, [_vp, _vp, _vp, _u64, _vp]),
    "sprs_b200_comm_unique_id": (_int, [C.c_char_p]),
    "sprs_b200_comm_init_rank": (_int, [_vp, C.c_char_p, _int, _int, C.POINTER(_vp)]),
    "sprs_b200_comm_free": (_int, [_vp]),
    "sprs_b200_comm_rank": (_int, [_vp]),
    "sprs_b200_comm_world": (_int, [_vp]),
    "sprs_b200_comm_multicast_supported": (_int, [_vp]),
    "sprs_b200_comm_allgather_host": (_int, [_vp, _vp, _u64, _vp]),
    "sprs_b200_comm_barrier_host": (_int, [_vp]),
    "sprs_b200_comm_barrier_dev": (_int, [_vp, _vp]),
    "sprs_b200_comm_check": (_int, [_vp, _vp]),
    "sprs_b200_symm_alloc": (_int, [_vp, _u64, _int, C.POINTER(_vp)]),
    "sprs_b200_symm_free": (_int, [_vp]),
    "sprs_b200_symm_ptr": (_vp, [_vp, _int]),
    "sprs_b200_symm_multicast_ptr": (_vp, [_vp]),
    "sprs_b200_symm_bytes": (_u64, [_vp]),
    "sprs_b200_partition_rows": (_int, [_vp, _int, _u64, _int, C.c_double, _vp]),
    "sprs_b200_spmv_rowpart": (_int, [_vp, _vp, _dp, _vp, _u64, _int, _vp]),
    "sprs_b200_mul_mat_vec_rowpart": (_int, [_vp, _vp, _vp, _dp, _u64, _u64, _dp, _u64]),
    "sprs_b200_peer_push_dev": (_int, [_vp, _vp, _u64, _u64, _int, C.POINTER(_vp), _vp]),
    "sprs_b200_spmv_allgather_dev": (_int, [_vp, _vp, _dp, _u64, _int, C.POINTER(_vp), _int, _vp]),
    "sprs_b200_spmv_chunked_push_dev": (_int, [_vp, _vp, _dp, _u64, _int, C.POINTER(_vp), _int,
                                               _int, _vp]),
    "sprs_b200_spgemm_symbolic": (_int, [_vp, _vp, _vp, C.POINTER(_vp), C.POINTER(_u64)]),
    "sprs_b200_spgemm_numeric": (_int, [_vp, _vp, _vp, _int, _vp, _int, _dp]),
    "sprs_b200_spgemm_numeric_dev": (_int, [_vp, _vp, C.POINTER(_vp)]),
    "sprs_b200_spgemm_nprod": (_u64, [_vp]),
    "sprs_b200_spgemm_free": (_int, [_vp]),
    "sprs_b200_bicgstab_new": (_int, [_vp, _vp, _dp, _dp, _u64, C.POINTER(_vp)]),
    "sprs_b200_bicgstab_new_dev": (_int, [_vp, _vp, _dp, _dp, _u64, C.POINTER(_vp)]),
    "sprs_b200_bicgstab_new_op": (_int, [_vp, _u64, MATVEC_FN, _vp, _dp, _dp, _int,
                                         C.POINTER(_vp)]),
    "sprs_b200_bicgstab_free": (_int, [_vp]),
    "sprs_b200_bicgstab_step": (_int, [_vp, C.POINTER(C.c_double)]),
    "sprs_b200_bicgstab_soft_restart": (_int, [_vp]),
    "sprs_b200_bicgstab_hard_restart": (_int, [_vp]),
    "sprs_b200_bicgstab_solve": (_int, [_vp, C.c_double, _u64, C.POINTER(_int)]),
    "sprs_b200_bicgstab_set_restart_threshold": (_int, [_vp, C.c_double]),
    "sprs_b200_bicgstab_stats": (_int, [_vp, C.POINTER(_u64), C.POINTER(C.c_double)]),
    "sprs_b200_bicgstab_get": (_int, [_vp, _int, _dp, _u64]),
    "sprs_b200_bicgstab_get_dev": (_int, [_vp, _int, C.POINTER(_vp)]),
    "sprs_b200_trisolve_plan": (_int, [_vp, _vp, _int, C.POINTER(_vp)]),
    "sprs_b200_trisolve_singular": (_int, [_vp, C.POINTER(_u64), C.POINTER(_int)]),
    "sprs_b200_trisolve_solve": (_int, [_vp, _dp, _u64]),
    "sprs_b200_trisolve_solve_dev": (_int, [_vp, _dp, _vp]),
    "sprs_b200_trisolve_free": (_int, [_vp]),
    "sprs_b200_diag_gather_ceiling": (_int, [_vp, _vp, _dp, _int, C.POINTER(C.c_double),
                                             C.POINTER(_u64)]),
    "sprs_b200_gen_rmat_keys": (_int, [_vp, _u64, _int, _u64, _u64, C.c_double, C.c_double,
                                       C.c_double, _u64, _u64, _vp, _vp]),
    "sprs_b200_gen_uniform_keys": (_int, [_vp, _u64, _u64, _u64, _u64, _u64, _vp, _vp]),
    "sprs_b200_gen_normal_from_keys": (_int, [_vp, _u64, _vp, _u64, _vp, _vp]),
    "sprs_b200_gen_split_keys": (_int, [_vp, _vp, _u64, _vp, _vp, _vp]),
    "sprs_b200_gen_hash_keys": (_int, [_vp, _u64, _vp, _u64, _vp, _vp]),
}

_NOT_EMULATED = ("sprs_b200_comm_", "sprs_b200_symm_", "sprs_b200_partition_rows",
                 "sprs_b200_spmv_rowpart", "sprs_b200_mul_mat_vec_rowpart", "sprs_b200_diag_",
                 # the binops are in a separate emulated build (tests/emu_binop.py)
                 "sprs_b200_csmat_binop", "sprs_b200_csmat_scale",
                 # so are the triangular solves (tests/emu_trisolve.py)
                 "sprs_b200_trisolve_")
_lib = None


def load():
    """Load libsprs_b200.so and attach prototypes.  Raises (never falls back)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "libsprs_b200.so is not built (%s): run `python -c 'import __graft_entry__ as g; "
            "g.build()'` or `make -C sprs_b200/csrc`.  sprs_b200 has no CPU fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    # the CPU emulator build of tests/emu (test infrastructure) has no multi-rank layer
    emulated = os.path.basename(LIB_PATH).startswith("libsprs_b200_emu")
    for name, (res, args) in PROTOTYPES.items():
        if emulated and name.startswith(_NOT_EMULATED) and not hasattr(lib, name):
            continue
        fn = getattr(lib, name)  # AttributeError if the ABI lost a symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib
