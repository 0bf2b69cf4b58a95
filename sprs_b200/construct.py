"""Sparse matrix construction on the device: the sprs crate's `bmat`, `vstack`, `hstack`
(sprs/src/sparse/construct.rs) and `kronecker_product` (sprs/src/sparse/kronecker.rs).

  vstack(mats)               always CSR: the CSR forms of mats, outer vectors appended in order
  hstack(mats)               always CSC: the same with the CSC forms, so that
                             hstack(ms) == vstack([m.transpose_view() for m in ms]).transpose_view()
  bmat(blocks)               always CSR: a None is zero((max rows of its block row, max cols of its
                             block column)); each block row is hstack-ed, the rows vstack-ed
  kronecker_product(a, b)    in a's storage (b converted first when the storages differ)

Results are bit-identical to the reference: stacking copies every value (NaN payloads and -0.0
included), the Kronecker product is one IEEE multiply per output entry and drops nothing.  The
work runs in libsprs_b200.so (csrc/construct.cu); the result keeps its device mirror attached,
so it goes straight into the next device operation.

The reference's panics come in its order, as SprsPanic with its messages: "Empty stacking list",
then "Dimension mismatch" (bmat: the block rows differ in length), "Empty bmat row", "Empty bmat
col", then "Dimension mismatch" from the stacking; kronecker_product raises the reference's
`Option::unwrap()` panic when a produced index does not fit the index dtype.

Differences from the reference on the device:
  * A result dimension >= 2^32 raises SprsPanic (ERR_INDEX_RANGE: device mirrors index with u32)
    even with 64-bit index dtypes, where `usize` would allow it.
  * The result's index dtypes are those of the first block (bmat, stacks) or of `a` (kron): Rust
    makes every operand share them.
"""
import ctypes as C

import numpy as np

from .sparse import CSC, CSR, CsMat, DeviceCsMat, SprsPanic

UNWRAP_NONE = "called `Option::unwrap()` on a `None` value"


def _result(ctx, dev, storage, shape, like):
    """The CsMat of a device result with like's index dtypes and its mirror attached."""
    ip, ind, dat = dev.download(like.indices.dtype, like.indptr.dtype)
    out = object.__new__(CsMat)
    out.storage, out.shape = storage, (int(shape[0]), int(shape[1]))
    out.indptr, out.indices, out.data = ip, ind, dat
    out._ctx, out._dev = like._ctx, dev
    return out


def bmat_dev(ctx, blocks):
    """sprs_b200_csmat_bmat on device mirrors: blocks is a list of rows of DeviceCsMat or None
    (rows of one length).  Returns the CSR result's DeviceCsMat."""
    nbr = len(blocks)
    nbc = len(blocks[0]) if nbr else 0
    flat = (C.c_void_p * max(nbr * nbc, 1))(*[b.h if b is not None else None
                                               for row in blocks for b in row])
    out = C.c_void_p()
    ctx.check(ctx.lib.sprs_b200_csmat_bmat(ctx.h, nbr, nbc, flat, C.byref(out)))
    return DeviceCsMat(ctx, out)


def transpose_view_dev(ctx, dev):
    """A DeviceCsMat of the same device arrays in the other storage (keeps dev alive)."""
    out = C.c_void_p()
    ctx.check(ctx.lib.sprs_b200_csmat_transpose_view(ctx.h, dev.h, C.byref(out)))
    return DeviceCsMat(ctx, out, keepalive=dev)


def kron_dev(ctx, a, b):
    """sprs_b200_csmat_kron on device mirrors; returns the result's DeviceCsMat."""
    out = C.c_void_p()
    ctx.check(ctx.lib.sprs_b200_csmat_kron(ctx.h, a.h, b.h, C.byref(out)))
    return DeviceCsMat(ctx, out)


def _check_grid(blocks):
    """construct.rs bmat's asserts, in its order."""
    if len(blocks) == 0:
        raise SprsPanic("Empty stacking list")
    ncols = len(blocks[0])
    if ncols == 0:
        raise SprsPanic("Empty stacking list")
    if any(len(row) != ncols for row in blocks):
        raise SprsPanic("Dimension mismatch")
    if any(all(b is None for b in row) for row in blocks):
        raise SprsPanic("Empty bmat row")
    if any(all(row[j] is None for row in blocks) for j in range(ncols)):
        raise SprsPanic("Empty bmat col")


def _stack_shape(blocks):
    rows = sum(max(b.rows() for b in row if b is not None) for row in blocks)
    row0 = blocks[0]
    widths = [max(r[j].cols() for r in blocks if r[j] is not None) for j in range(len(row0))]
    cols = sum(b.cols() if b is not None else w for b, w in zip(row0, widths))
    return rows, cols


def bmat(blocks):
    """sprs::bmat (construct.rs): a CSR matrix from a grid of CsMat blocks or None."""
    blocks = [list(row) for row in blocks]
    _check_grid(blocks)
    first = next(b for row in blocks for b in row if b is not None)
    ctx = first.context()
    dev = bmat_dev(ctx, [[b.device() if b is not None else None for b in row] for row in blocks])
    return _result(ctx, dev, CSR, _stack_shape(blocks), first)


def vstack(mats):
    """sprs::vstack (construct.rs): the CSR forms of mats stacked vertically; always CSR."""
    mats = list(mats)
    if not mats:
        raise SprsPanic("Empty stacking list")
    ctx = mats[0].context()
    dev = bmat_dev(ctx, [[m.device()] for m in mats])
    return _result(ctx, dev, CSR, (sum(m.rows() for m in mats), mats[0].cols()), mats[0])


def hstack(mats):
    """sprs::hstack (construct.rs): the CSC forms of mats stacked horizontally; always CSC.
    On the device: the transpose view of the vstack of the blocks' transpose views."""
    mats = list(mats)
    if not mats:
        raise SprsPanic("Empty stacking list")
    ctx = mats[0].context()
    views = [transpose_view_dev(ctx, m.device()) for m in mats]
    dev = transpose_view_dev(ctx, bmat_dev(ctx, [[v] for v in views]))
    return _result(ctx, dev, CSC, (mats[0].rows(), sum(m.cols() for m in mats)), mats[0])


def _max_inner_index(m, storage):
    """The largest inner index of m's `storage` form (m has non-zeros)."""
    nnz = m.nnz()
    if m.storage == storage:
        return int(m.indices[:nnz].max())
    lens = np.diff(m.indptr.astype(np.int64))
    return int(np.flatnonzero(lens)[-1])  # the other storage's inner index is m's outer one


def kronecker_product(a, b):
    """sprs::kronecker_product (kronecker.rs): in a's storage, b converted when they differ."""
    if a.nnz() and b.nnz():
        inner_b = b.inner_dims() if b.storage == a.storage else b.outer_dims()
        top = _max_inner_index(a, a.storage) * inner_b + _max_inner_index(b, a.storage)
        if top > np.iinfo(a.indices.dtype).max:
            raise SprsPanic(UNWRAP_NONE)
    ctx = a.context()
    dev = kron_dev(ctx, a.device(), b.device())
    return _result(ctx, dev, a.storage, (a.rows() * b.rows(), a.cols() * b.cols()), a)
