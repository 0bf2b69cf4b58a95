"""Synthetic sparse inputs built in HBM (bench / test plumbing, not the product path).

torch is used here only for device memory and for sort / unique / searchsorted while
assembling CSR from candidate keys; the keys and values come from the counter-based
kernels in csrc/gen.cu so that every rank regenerates identical matrices.

  rand_csr(...)   sprs-rand's distribution (sprs-rand/src/lib.rs:24-81): nnz =
                  ceil(density * rows * cols) exactly, a uniform random row per non-zero,
                  distinct uniform columns per row, values N(0,1) (lib.rs:85-88).  Uniform
                  cells are drawn, duplicates dropped, and more drawn until at least the
                  target are distinct, then thinned by hash to the target; ValueError when
                  the target exceeds rows * cols (the reference asserts density <= 1).
  rmat_csr(...)   this repo's R-MAT definition (the reference has none, SURVEY F8):
                  Graph500 (a,b,c,d) = (0.57,0.19,0.19,0.05), scale = ceil(log2 n),
                  candidates with an index >= n rejected, duplicates dropped, then
                  thinned uniformly to the target nnz (exactly when at most 2^27 keys are
                  distinct, to within sampling noise of it otherwise); ValueError when
                  six oversampling passes leave fewer distinct keys than the target.

tests/gen_model.py restates all of it on the host; tests/test_gpu_gen_bits.py compares the two
bit for bit and pins the benchmark matrices by digest.
"""
import ctypes as C
import math

import numpy as np
import torch

from . import _lib
from .sparse import DeviceCsMat

SENTINEL = -1  # UINT64_MAX read as int64


def _device(ctx):
    return torch.device("cuda", ctx.device)


def _stream_ptr():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _sync():
    torch.cuda.current_stream().synchronize()


def _dptr(t):
    return C.c_void_p(t.data_ptr())


class DeviceCsr:
    """CSR matrix resident in HBM as torch tensors (int32 storage of u32 values) plus
    its sprs_b200 mirror (adopted without copying)."""

    def __init__(self, ctx, rows, cols, indptr, indices, data):
        self.ctx, self.rows, self.cols = ctx, rows, cols
        self.indptr, self.indices, self.data = indptr, indices, data
        self.nnz = int(indices.numel())
        # the arrays were produced on torch's current stream; the library builds the mirror's
        # SpMV partition on ITS stream: make them ready first (sprs_b200.h: from_device adopts
        # arrays that must be complete when the call is made)
        if indptr.is_cuda:
            _sync()
        h = C.c_void_p()
        ctx.check(ctx.lib.sprs_b200_csmat_from_device(
            ctx.h, _lib.CSR, rows, cols, self.nnz, _dptr(indptr), _dptr(indices), _dptr(data),
            C.byref(h)))
        self.mirror = DeviceCsMat(ctx, h, keepalive=(indptr, indices, data))

    def slice_rows(self, r0, r1):
        """slice_outer(r0..r1) + proper_indptr (slicing.rs:65-89, csmat.rs:919-921)."""
        s, e = u32(self.indptr[r0]), u32(self.indptr[r1])  # int32 storage of u32 values
        ip = (self.indptr[r0:r1 + 1] - self.indptr[r0]).contiguous()  # wraps to the right u32
        return DeviceCsr(self.ctx, r1 - r0, self.cols, ip, self.indices[s:e].clone(),
                         self.data[s:e].clone())

    def to_host(self):
        return (self.indptr.cpu().numpy().view(np.uint32), self.indices.cpu().numpy().view(np.uint32),
                self.data.cpu().numpy())


def u32(t):
    """Python int of one element of an int32 tensor that stores a u32 value (nnz < 2^32)."""
    v = int(t.item())
    return v & 0xFFFFFFFF if t.dtype == torch.int32 else v


def _keys_to_csr(ctx, keys, rows, cols, seed):
    """sorted unique int64 keys (row<<32|col) -> DeviceCsr."""
    dev = keys.device
    n = keys.numel()
    bounds = torch.arange(rows + 1, device=dev, dtype=torch.int64) << 32
    indptr = torch.searchsorted(keys, bounds).to(torch.int32)
    del bounds
    indices = torch.empty(n, device=dev, dtype=torch.int32)
    data = torch.empty(n, device=dev, dtype=torch.float64)
    lib = ctx.lib
    if n:
        ctx.check(lib.sprs_b200_gen_split_keys(ctx.h, _dptr(keys), n, None, _dptr(indices),
                                               _stream_ptr()))
        ctx.check(lib.sprs_b200_gen_normal_from_keys(ctx.h, seed ^ 0xDA7A, _dptr(keys), n,
                                                     _dptr(data), _stream_ptr()))
    _sync()
    if dev.type == "cuda":
        # the sorts above leave several times the matrix in torch's cache (tens of GB for the
        # 1e9-nnz R-MAT); the library allocates outside that cache (cudaMalloc, its
        # stream-ordered pool), so on an 80 GB H100 it is handed back before the matrix is used
        torch.cuda.empty_cache()
    return DeviceCsr(ctx, rows, cols, indptr, indices, data)


def _thin(ctx, keys, target, seed, exact):
    """Drop (uniformly, by key hash) down to `target` keys; exact=True hits it exactly."""
    n = keys.numel()
    if n <= target:
        return keys
    h = torch.empty(n, device=keys.device, dtype=torch.int64)
    ctx.check(ctx.lib.sprs_b200_gen_hash_keys(ctx.h, seed ^ 0x7417, _dptr(keys), n, _dptr(h),
                                              _stream_ptr()))
    if exact:
        thr = torch.kthvalue(h, target).values  # keep the `target` smallest hashes
        keep = h <= thr
    else:
        keep = h < int((target / n) * (1 << 63))
    del h
    return keys[keep]


def _collect(ctx, gen, n_candidates, chunk=1 << 27):
    """Generate candidates in chunks, drop rejected, return sorted unique keys."""
    parts = []
    first = 0
    dev = _device(ctx)
    while first < n_candidates:
        cnt = min(chunk, n_candidates - first)
        k = torch.empty(cnt, device=dev, dtype=torch.int64)
        gen(first, cnt, k)
        k = k[k != SENTINEL]
        k = torch.unique(k)  # sorted unique within the chunk keeps the final sort smaller
        parts.append(k)
        first += cnt
    keys = torch.cat(parts) if len(parts) > 1 else parts[0]
    del parts
    if keys.numel():
        keys = torch.unique(keys)
    return keys


def rand_csr(ctx, rows, cols, nnz_per_row, seed=0x5EED0002):
    """sprs-rand semantics; exact nnz = ceil(density*rows*cols) (lib.rs:37-38)."""
    target = int(math.ceil(nnz_per_row * rows))
    if target > rows * cols:
        raise ValueError("rand_csr: %d non-zeros do not fit %d x %d" % (target, rows, cols))
    over = target + max(4096, target // 512)

    def gen(first, cnt, out):
        ctx.check(ctx.lib.sprs_b200_gen_uniform_keys(ctx.h, seed, rows, cols, first, cnt,
                                                     _dptr(out), _stream_ptr()))
    keys = _collect(ctx, gen, over)
    while keys.numel() < target:  # dense targets: duplicates ate the slack of the first pass
        over = int(over * 1.5)
        keys = _collect(ctx, gen, over)
    keys = _thin(ctx, keys, target, seed, exact=True)
    return _keys_to_csr(ctx, keys, rows, cols, seed)


def rmat_csr(ctx, n, nnz_per_row, seed=0x5EED0005, abc=(0.57, 0.19, 0.19), oversample=None):
    """R-MAT n x n with ~nnz_per_row*n non-zeros (see module docstring)."""
    scale = max(1, int(math.ceil(math.log2(n))))
    target = int(nnz_per_row * n)
    a, b, c = abc

    def gen(first, cnt, out):
        ctx.check(ctx.lib.sprs_b200_gen_rmat_keys(ctx.h, seed, scale, n, n, a, b, c, first, cnt,
                                                  _dptr(out), _stream_ptr()))
    factor = oversample or 1.6
    for _ in range(6):
        keys = _collect(ctx, gen, int(target * factor))
        if keys.numel() >= target:
            break
        factor *= 1.5
    else:
        raise ValueError("rmat_csr: %d distinct keys of the %d asked for after six passes"
                         % (keys.numel(), target))
    keys = _thin(ctx, keys, target, seed, exact=keys.numel() <= (1 << 27))
    return _keys_to_csr(ctx, keys, n, n, seed)


def make_matrix(ctx, gen, n, nnz_per_row, seed):
    """Square n x n bench matrix: gen = "rmat" | "rand"."""
    if gen == "rmat":
        return rmat_csr(ctx, n, nnz_per_row, seed=seed)
    return rand_csr(ctx, n, n, nnz_per_row, seed=seed)


def triangular(ctx, a, lower=True):
    """The strict lower (or upper) triangle of a square DeviceCsr `a` (a rand_csr / rmat_csr
    key set) plus a diagonal d_r = 1 + sum |off-diagonal of row r|, as a new DeviceCsr: the
    inputs of the triangular solves (csrc/trisolve.cu).  The dominant diagonal keeps x bounded.
    Each row's sum is the difference of two entries of one float64 prefix sum of |a_rc| over the
    whole triangle (torch.cumsum), so d_r equals 1 + sum |row| only to within the prefix sum's
    rounding -- far inside the dominance the solves need."""
    n = a.rows
    dev = a.indices.device
    ip = a.indptr.to(torch.int64) & 0xFFFFFFFF  # int32 storage of u32 values
    rows = torch.repeat_interleave(torch.arange(n, device=dev, dtype=torch.int32), ip[1:] - ip[:-1])
    keep = a.indices < rows if lower else a.indices > rows  # n < 2^31: u32 values fit int32
    kr = rows[keep]
    del rows
    kc, kv = a.indices[keep], a.data[keep]
    del keep
    m = kc.numel()
    cnt = torch.bincount(kr, minlength=n)
    kip = torch.zeros(n + 1, device=dev, dtype=torch.int64)
    torch.cumsum(cnt, 0, out=kip[1:])
    cs = torch.zeros(m + 1, device=dev, dtype=torch.float64)
    torch.cumsum(kv.abs(), 0, out=cs[1:])
    diag = 1.0 + (cs[kip[1:]] - cs[kip[:-1]])
    del cs
    nip = kip + torch.arange(n + 1, device=dev, dtype=torch.int64)  # one diagonal per row
    rank = torch.arange(m, device=dev, dtype=torch.int64) - kip[kr.to(torch.int64)]
    pos = nip[kr.to(torch.int64)] + rank + (0 if lower else 1)
    del rank, kr
    indices = torch.empty(m + n, device=dev, dtype=torch.int32)
    data = torch.empty(m + n, device=dev, dtype=torch.float64)
    indices[pos] = kc
    data[pos] = kv
    del pos, kc, kv
    dpos = nip[1:] - 1 if lower else nip[:-1]
    indices[dpos] = torch.arange(n, device=dev, dtype=torch.int32)
    data[dpos] = diag
    _sync()
    return DeviceCsr(ctx, n, n, nip.to(torch.int32), indices, data)


def trisolve_dev(ctx, plan, x):
    """Enqueue plan's solve of the device vector x (torch, float64, in place) on torch's current
    stream; returns the SingularMatrix it raised, or None."""
    from .sparse import SingularMatrix
    try:
        s = _stream_ptr()
        plan.solve_dev(x.data_ptr(), s.value if s else None)
    except SingularMatrix as e:
        return e
    return None


def normal_vector(ctx, n, seed=0x5EED1002):
    x = torch.empty(n, device=_device(ctx), dtype=torch.float64)
    ctx.check(ctx.lib.sprs_b200_gen_normal_from_keys(ctx.h, seed, None, n, _dptr(x),
                                                     _stream_ptr()))
    return x


def spmv(ctx, a, x, y, accumulate=False):
    """y (+)= A x on torch's current stream; a is a DeviceCsr or DeviceCsMat."""
    m = a.mirror if isinstance(a, DeviceCsr) else a
    ctx.check(ctx.lib.sprs_b200_spmv_dev(ctx.h, m.h, _dptr(x), _dptr(y), int(accumulate),
                                         _stream_ptr()))
    return y


def spmm_rowmaj(ctx, a, b, c, accumulate=False):
    """C (+)= A B, B and C row-major torch tensors."""
    m = a.mirror if isinstance(a, DeviceCsr) else a
    k = b.shape[1]
    ctx.check(ctx.lib.sprs_b200_spmm_rowmaj_dev(ctx.h, m.h, _dptr(b), b.stride(0), k, _dptr(c),
                                                c.stride(0), int(accumulate), _stream_ptr()))
    return c


class _DevArray:
    """Zero-copy torch view of a raw device allocation (__cuda_array_interface__)."""

    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr,
                                         "data": (ptr, False), "version": 2}


def spgemm(ctx, a, b):
    """C = A B on the device (smmp::mul_csr_csr: symbolic, then numeric into a new mirror).
    Returns (mirror, indptr, indices, data): the DeviceCsMat that owns C and zero-copy torch
    views of its arrays (int32 storage of u32 values; int64 indptr when nnz(C) >= 2^32),
    valid while the mirror is alive -- what RowPartitionedSpGEMM's local_spgemm returns."""
    ma = a.mirror if isinstance(a, DeviceCsr) else a
    mb = b.mirror if isinstance(b, DeviceCsr) else b
    lib = ctx.lib
    if _device(ctx).type == "cuda":
        _sync()  # operands produced on torch's stream; symbolic / numeric run on the ctx stream
    plan, nnz_c, cm = C.c_void_p(), C.c_uint64(), C.c_void_p()
    ctx.check(lib.sprs_b200_spgemm_symbolic(ctx.h, ma.h, mb.h, C.byref(plan), C.byref(nnz_c)))
    try:
        ctx.check(lib.sprs_b200_spgemm_numeric_dev(ctx.h, plan, C.byref(cm)))
    finally:
        lib.sprs_b200_spgemm_free(plan)
    return _with_views(ctx, DeviceCsMat(ctx, cm))


def _with_views(ctx, mirror):
    """(mirror, indptr, indices, data): zero-copy torch views of a result mirror's arrays."""
    d_ip, d_ind, d_dat, ipb = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_int()
    ctx.check(ctx.lib.sprs_b200_csmat_device_arrays(mirror.h, C.byref(d_ip), C.byref(ipb),
                                                    C.byref(d_ind), C.byref(d_dat)))
    dev = _device(ctx)
    outer = mirror.rows if mirror.storage == "CSR" else mirror.cols
    nnz = mirror.nnz
    indptr = torch.as_tensor(_DevArray(d_ip.value, outer + 1, "<i4" if ipb.value == 4 else "<i8"),
                             device=dev)
    if nnz:
        indices = torch.as_tensor(_DevArray(d_ind.value, nnz, "<i4"), device=dev)
        data = torch.as_tensor(_DevArray(d_dat.value, nnz, "<f8"), device=dev)
    else:
        indices = torch.empty(0, dtype=torch.int32, device=dev)
        data = torch.empty(0, dtype=torch.float64, device=dev)
    return mirror, indptr, indices, data


_BINOP_OPS = {"add": _lib.BINOP_ADD, "sub": _lib.BINOP_SUB, "mul": _lib.BINOP_MUL}


def binop(ctx, a, b, op):
    """C = A + B ("add"), A - B ("sub") or A .* B ("mul") on the device (csmat_binop,
    binop.rs:178-271; same storage and shape).  Returns (mirror, indptr, indices, data) like
    spgemm: the DeviceCsMat that owns C and zero-copy torch views of its arrays."""
    ma = a.mirror if isinstance(a, DeviceCsr) else a
    mb = b.mirror if isinstance(b, DeviceCsr) else b
    if _device(ctx).type == "cuda":
        _sync()  # operands produced on torch's stream; the binop runs on the ctx stream
    cm = C.c_void_p()
    ctx.check(ctx.lib.sprs_b200_csmat_binop(ctx.h, ma.h, mb.h, _BINOP_OPS[op], C.byref(cm)))
    return _with_views(ctx, DeviceCsMat(ctx, cm))


def scale(ctx, a, s):
    """C = A * s on the device (CsMatBase::map: same structure, zeros kept); returns
    (mirror, indptr, indices, data) like binop."""
    ma = a.mirror if isinstance(a, DeviceCsr) else a
    if _device(ctx).type == "cuda":
        _sync()
    cm = C.c_void_p()
    ctx.check(ctx.lib.sprs_b200_csmat_scale(ctx.h, ma.h, float(s), C.byref(cm)))
    return _with_views(ctx, DeviceCsMat(ctx, cm))


def bmat(ctx, blocks):
    """sprs::bmat on the device (csrc/construct.cu): blocks is a list of rows of DeviceCsr,
    DeviceCsMat or None.  Returns (mirror, indptr, indices, data) of the CSR result like binop."""
    from .construct import bmat_dev
    if _device(ctx).type == "cuda":
        _sync()  # blocks produced on torch's stream; the construction runs on the ctx stream
    mirrors = [[b.mirror if isinstance(b, DeviceCsr) else b for b in row] for row in blocks]
    return _with_views(ctx, bmat_dev(ctx, mirrors))


def kron(ctx, a, b):
    """sprs::kronecker_product on the device (csrc/construct.cu), in a's storage; returns
    (mirror, indptr, indices, data) like binop."""
    from .construct import kron_dev
    ma = a.mirror if isinstance(a, DeviceCsr) else a
    mb = b.mirror if isinstance(b, DeviceCsr) else b
    if _device(ctx).type == "cuda":
        _sync()
    return _with_views(ctx, kron_dev(ctx, ma, mb))


# ---- the dense boundary on torch tensors (the dense section of csrc/transpose.cu)
def _strides(t):
    """element strides of a 2-D float64 tensor as the library takes them (all zero for a tensor
    with a zero-length axis, as ndarray has them)"""
    if t.dim() != 2 or t.dtype != torch.float64:
        raise TypeError("a 2-D float64 tensor is required")
    return (0, 0) if 0 in t.shape else (t.stride(0), t.stride(1))


def to_dense(ctx, a, out=None):
    """CsMat::to_dense (csmat.rs:1127-1134) on the device: a C-order tensor (out, if given, must
    have unit column stride) holding A's values as bits and +0.0 elsewhere; torch's stream."""
    m = a.mirror if isinstance(a, DeviceCsr) else a
    if out is None:
        out = torch.empty((m.rows, m.cols), dtype=torch.float64, device=_device(ctx))
    if out.shape != (m.rows, m.cols) or (out.numel() and out.stride(1) != 1):
        raise ValueError("out must be a (rows, cols) tensor with unit column stride")
    ld = out.stride(0) if out.numel() else m.cols
    ctx.check(ctx.lib.sprs_b200_csmat_to_dense_dev(ctx.h, m.h, _dptr(out), ld, _stream_ptr()))
    return out


def assign_to_dense(ctx, out, a):
    """assign_to_dense (to_dense.rs:12-30) into a 2-D float64 tensor view: A's values as bits,
    every other element untouched; torch's stream."""
    m = a.mirror if isinstance(a, DeviceCsr) else a
    rs, cs = _strides(out)
    ctx.check(ctx.lib.sprs_b200_assign_to_dense_dev(ctx.h, m.h, _dptr(out), out.shape[0],
                                                    out.shape[1], rs, cs, _stream_ptr()))
    return out


def from_dense(ctx, d, epsilon, storage="CSR"):
    """csr_from_dense / csc_from_dense (csmat.rs:502-549) of a 2-D float64 tensor view.  Returns
    (mirror, indptr, indices, data) like binop: the DeviceCsMat that owns the result and
    zero-copy torch views of its arrays."""
    rs, cs = _strides(d)
    if _device(ctx).type == "cuda":
        _sync()  # d produced on torch's stream; the passes run on the ctx stream
    cm = C.c_void_p()
    ctx.check(ctx.lib.sprs_b200_csmat_from_dense_dev(
        ctx.h, _lib.CSR if storage == "CSR" else _lib.CSC, d.shape[0], d.shape[1], _dptr(d), rs, cs,
        float(epsilon), C.byref(cm)))
    return _with_views(ctx, DeviceCsMat(ctx, cm))


def binop_dense(ctx, a, d, op="add", alpha=1.0, beta=1.0, out=None):
    """csmat_binop_dense_raw (binop.rs:384-433) on the device: out = alpha*A + beta*D ("add") or
    alpha*A*D ("mul"), A's storage matching the fastest axis of D and out.  out=None allocates it
    as add_dense_mat_same_ordering does (C order when D's fastest axis is Axis(1), F order
    otherwise); out may be d itself.  torch's stream."""
    m = a.mirror if isinstance(a, DeviceCsr) else a
    rrs, rcs = _strides(d)
    if out is None:
        out = torch.empty(d.shape, dtype=torch.float64, device=_device(ctx))
        if rcs > rrs:  # Axis(0) fastest: F order
            out = torch.empty((d.shape[1], d.shape[0]), dtype=torch.float64, device=_device(ctx)).t()
    ors, ocs = _strides(out)
    ctx.check(ctx.lib.sprs_b200_csmat_binop_dense_dev(
        ctx.h, m.h, _BINOP_OPS[op], float(alpha), float(beta), _dptr(d), d.shape[0], d.shape[1], rrs,
        rcs, _dptr(out), out.shape[0], out.shape[1], ors, ocs, _stream_ptr()))
    return out
