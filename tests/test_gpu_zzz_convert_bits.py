"""Storage conversion, triplet assembly and the CSC / dense-view product routes BIT FOR BIT with
real-valued data.

Everything downstream of these routes -- CSC operands of the SpMV, the SpMM and SpGEMM, the
binop's storage conversion, MatrixMarket input -- inherits their bits, and integer data cannot
see an order: every partial sum is exact there.  Values here are N(0,1), and N(0,1) * 2^k (k
uniform in [-20, 20] per entry), where almost any re-association changes a bit.

- `to_other_storage` (csrc/transpose.cu, csmat.rs:1782-1829) moves values without arithmetic:
  every array equals `O.convert_mat_storage`, the values compared as uint64 (NaN payloads,
  -0.0, subnormals and +-Inf included), at the radix sort's pass seams (inner dimension 1, 2,
  256, 257, 65536, 65537, 2^24 + 1: 1 to 4 passes of 8 bits), at nnz 4095 / 4096 / 4097 (the
  4096-item sort block), and with one inner index holding several blocks' worth of entries.
- `from_triplets` sums the members of a duplicate run in INSERTION order, from the first
  member's value.  The reference sorts with `sort_unstable_by_key` (triplet_iter.rs:144-150), so
  its order is unspecified for runs of three or more terms; for those runs the check is against
  this project's contract, insertion order, which is also the oracle's `std::stable_sort`
  (sprs_oracle.cpp).  Two-term runs match the reference in any order.  The runs straddle the
  radix sort's warp (512 items) and block (4096 items) boundaries in both of its sorts (by
  column, then by row), at pass-count parities that take both ping-pong buffer orders.  NaN
  results of additions are compared by class (the GPU returns the canonical NaN, x86 propagates
  a payload), everything else by bits.
- CSC dense products run the CSR kernels on the cached device conversion: `csc_mulacc_dense_
  rowmaj` (k >= 8) adds each output element's terms in ascending column order, like prod.rs:
  219-241, so it equals the oracle bit for bit.  The k < 8 route is one SpMV per column, which is
  checked against the host model of the SpMV's order (tests/spmv_model.py) and against the oracle
  on the rows the model says are summed in storage order.
- Sparse-vector dots against a sequential host loop that restates each reference function.

Every test that claims an order first shows, with the oracle alone, that another order of the
same terms changes at least 15 % of its entries of three or more terms, and asserts the seams
it claims (pass counts, straddles, row lengths)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import exact
import spmv_model as M
from test_gpu_exact import _csr_from_lens

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RS_WCHUNK, RS_CHUNK = 512, 4096    # transpose.cu: contiguous items per warp / per sort block
BIG = 1e308
MIN_SHARE = 0.15


@pytest.fixture(scope="module")
def sp():
    import sprs_b200
    sprs_b200.Context.default()  # raises without a GPU / without the .so: no fallback
    return sprs_b200


@pytest.fixture(scope="module")
def O():
    from oracle import oracle
    return oracle


# ---------------------------------------------------------------- values
def bits_for(r):
    """transpose.cu bits_for: key bits of a dimension of size r."""
    bits = 1
    while bits < 32 and (1 << bits) < r:
        bits += 1
    return bits


def passes(r):
    return (bits_for(r) + 7) // 8


def real_values(rng, n):
    return rng.standard_normal(n) * np.exp2(rng.integers(-20, 21, n))


def u64(x):
    return np.ascontiguousarray(x, dtype=np.float64).view(np.uint64)


NAN_PAYLOADS = np.array([0x7FF8000000000001, 0xFFF80000DEADBEEF, 0x7FF0000000000123],
                        dtype=np.uint64).view(np.float64)
RAW_EDGES = np.concatenate([NAN_PAYLOADS, [-0.0, 5e-324, -2.5e-310, np.inf, -np.inf]])


def plant_raw(rng, d):
    """Values that must travel as raw bits: NaN payloads (one a signalling NaN), -0.0,
    subnormals, +-Inf, at random positions."""
    d = d.copy()
    if len(d) >= len(RAW_EDGES):
        d[rng.choice(len(d), len(RAW_EDGES), replace=False)] = RAW_EDGES
    return d


# ---------------------------------------------------------------- 1a: to_other_storage
def convert_case(rng, name):
    """(outer, inner, indptr, indices, data) of one §1a shape, before values are planted."""
    if name.startswith("inner="):
        inner = int(name[6:])
        outer = 14_000 if inner <= 2 else 3000
        lens = np.minimum(rng.integers(0, 8, outer), inner)
        if inner == 1:
            lens = (rng.random(outer) < 0.95).astype(np.int64)  # ~13 300 entries on inner index 0
    elif name.startswith("nnz="):
        nnz, outer, inner = int(name[4:]), 700, 5000
        lens = np.bincount(rng.integers(0, outer, nnz), minlength=outer)
    elif name == "hub":  # inner index 7 in every outer: > 3 sort blocks of entries
        outer, inner = 14_000, 5000
        lens = rng.integers(1, 4, outer)
        ip, ind = _csr_from_lens(rng, lens - 1, inner - 1)
        ind = ind.astype(np.int64)
        ind[ind >= 7] += 1
        rows = np.repeat(np.arange(outer), lens - 1)
        all_rows = np.concatenate([rows, np.arange(outer)])
        all_ind = np.concatenate([ind, np.full(outer, 7)])
        o = np.lexsort((all_ind, all_rows))
        ip = np.zeros(outer + 1, dtype=np.int64)
        np.cumsum(lens, out=ip[1:])
        return outer, inner, ip.astype(np.uint32), all_ind[o].astype(np.uint32)
    elif name == "empty_outer":
        return 0, 300, np.zeros(1, np.uint32), np.zeros(0, np.uint32)
    elif name == "empty_inner":
        return 40, 0, np.zeros(41, np.uint32), np.zeros(0, np.uint32)
    elif name == "no_nonzeros":
        return 40, 70, np.zeros(41, np.uint32), np.zeros(0, np.uint32)
    else:
        raise ValueError(name)
    ip, ind = _csr_from_lens(rng, lens, inner)
    return outer, inner, ip, ind


CONVERT_CASES = ["inner=1", "inner=2", "inner=256", "inner=257", "inner=65536", "inner=65537",
                 "inner=%d" % ((1 << 24) + 1), "nnz=4095", "nnz=4096", "nnz=4097", "hub",
                 "empty_outer", "empty_inner", "no_nonzeros"]


def convert_seams(outer, inner, ip, ind):
    """What a §1a case reaches: radix passes, sort blocks, and the most entries of one inner
    index in sort blocks."""
    nnz = int(ip[-1]) - int(ip[0])
    top = int(np.bincount(ind.astype(np.int64), minlength=1).max()) if nnz else 0
    return {"passes": passes(inner), "nnz": nnz, "blocks": -(-nnz // RS_CHUNK),
            "hub_blocks": top / RS_CHUNK}


def _check_convert(got, want, what):
    exact.assert_csr_bits((got[0], got[1], np.zeros(len(got[2]))),
                          (want[0], want[1], np.zeros(len(want[2]))), what + ": structure")
    g, w = u64(got[2]), u64(want[2])
    assert np.array_equal(g, w), "%s: %d values differ in their bits" % (what, int((g != w).sum()))


@pytest.mark.parametrize("idx", [np.uint32, np.uint64])
@pytest.mark.parametrize("name", CONVERT_CASES)
def test_to_other_storage_bits(sp, O, name, idx):
    """CSR -> CSC -> CSR: every array equals the oracle's, values as raw bits; the round trip
    is the identity."""
    rng = np.random.default_rng(CONVERT_CASES.index(name) + 11)
    outer, inner, ip, ind = convert_case(rng, name)
    seams = convert_seams(outer, inner, ip, ind)
    if name.startswith("inner="):
        assert seams["passes"] == {1: 1, 2: 1, 256: 1, 257: 2, 65536: 2, 65537: 3}.get(inner, 4)
        assert seams["blocks"] >= 3
    if name.startswith("nnz="):
        assert seams["nnz"] == int(name[4:])
    if name in ("hub", "inner=1"):
        assert seams["hub_blocks"] > 3
    d = plant_raw(rng, real_values(rng, len(ind)))
    ip, ind = ip.astype(idx), ind.astype(idx)
    a = sp.CsMat.new((outer, inner), ip, ind, d)
    t = a.to_other_storage()
    assert t.is_csc() and t.indices.dtype == idx
    want = O.convert_mat_storage(outer, inner, ip, ind, d)
    _check_convert((t.indptr, t.indices, t.data), want, "%s %s CSR -> CSC" % (name, idx.__name__))
    back = t.to_other_storage()
    assert back.is_csr()
    _check_convert((back.indptr, back.indices, back.data), (ip, ind, d), name + " round trip")


def test_to_other_storage_csc_to_csr_bits(sp, O):
    """CSC -> CSR of a CSC matrix with a hub row, against convert_mat_storage(cols, rows)."""
    rng = np.random.default_rng(21)
    outer, inner, ip, ind = convert_case(rng, "hub")  # outer = columns of the CSC matrix
    d = plant_raw(rng, real_values(rng, len(ind)))
    a = sp.CsMat.new_csc((inner, outer), ip, ind, d)
    t = a.to_other_storage()
    assert t.is_csr()
    _check_convert((t.indptr, t.indices, t.data), O.convert_mat_storage(outer, inner, ip, ind, d),
                   "CSC -> CSR")


def test_to_other_storage_slice_outer_bits(sp, O):
    """A slice_outer view, whose indptr does not start at 0 (the upload rebases it)."""
    rng = np.random.default_rng(22)
    outer, inner, ip, ind = convert_case(rng, "inner=65537")
    d = plant_raw(rng, real_values(rng, len(ind)))
    a = sp.CsMat.new((outer, inner), ip, ind, d)
    v = a.slice_outer(517, 2900)
    assert int(v.indptr[0]) > 0
    t = v.to_other_storage()
    s, e = int(ip[517]), int(ip[2900])
    want = O.convert_mat_storage(2900 - 517, inner, ip[517:2901] - ip[517], ind[s:e], d[s:e])
    _check_convert((t.indptr, t.indices, t.data), want, "slice_outer(517, 2900)")


# ---------------------------------------------------------------- 1b: from_triplets
def triplet_case(rng, rows, cols, n_runs=300, n_hot=4, n_other=12_000):
    """COO whose duplicate runs (3 to 50 members) sit in a few hot columns, their members
    scattered over the whole insertion order: in the column sort they straddle warp and block
    boundaries of the input, and in the row sort -- whose input is the column order, where a hot
    column's entries form one long bucket -- they straddle them again.  Plus pairs and
    singles everywhere.  Returns (rows, cols, r, c, runs) with runs = [(row, col)] of >= 3."""
    hot = rng.choice(cols, min(n_hot, cols), replace=False)
    cells = set()
    run_cells = []
    while len(run_cells) < n_runs:
        cell = (int(rng.integers(0, rows)), int(hot[rng.integers(0, len(hot))]))
        if cell not in cells:
            cells.add(cell)
            run_cells.append(cell)
    r, c = [], []
    for cell in run_cells:
        n = int(rng.integers(3, 51))
        r += [cell[0]] * n
        c += [cell[1]] * n
    # other entries: singles and pairs, a third of them in the hot columns
    oc = np.where(rng.random(n_other) < 0.33, hot[rng.integers(0, len(hot), n_other)],
                  rng.integers(0, cols, n_other))
    orow = rng.integers(0, rows, n_other)
    keep = np.array([(int(a), int(b)) not in cells for a, b in zip(orow, oc)], dtype=bool)
    orow, oc = orow[keep], oc[keep]
    pairs = rng.random(len(orow)) < 0.2
    r = np.concatenate([r, orow, orow[pairs]]).astype(np.int64)
    c = np.concatenate([c, oc, oc[pairs]]).astype(np.int64)
    perm = rng.permutation(len(r))
    return r[perm], c[perm], run_cells


def run_members(r, c, rows, cols):
    """Per cell with >= 3 triplets: the insertion positions of its members (ascending)."""
    key = r * cols + c
    order = np.argsort(key, kind="stable")
    k = key[order]
    heads = np.flatnonzero(np.r_[True, k[1:] != k[:-1]])
    lens = np.diff(np.r_[heads, len(k)])
    return [order[h:h + n] for h, n in zip(heads, lens) if n >= 3]


def triplet_seams(r, c, rows, cols):
    """Runs of >= 3 members whose members straddle a warp / block boundary of the column sort's
    input (insertion positions) and of the row sort's input (positions in column order)."""
    in_col_sort = np.empty(len(c), dtype=np.int64)
    in_col_sort[np.argsort(c, kind="stable")] = np.arange(len(c))
    out = {"passes": (passes(rows), passes(cols)), "runs": 0}
    for name, pos in (("col", None), ("row", in_col_sort)):
        for w, bound in (("warp", RS_WCHUNK), ("block", RS_CHUNK)):
            out["%s_%s" % (name, w)] = 0
    for m in run_members(r, c, rows, cols):
        out["runs"] += 1
        for name, pos in (("col", m), ("row", in_col_sort[m])):
            for w, bound in (("warp", RS_WCHUNK), ("block", RS_CHUNK)):
                if pos.min() // bound != pos.max() // bound:
                    out["%s_%s" % (name, w)] += 1
    return out


def triplet_values(rng, n):
    return real_values(rng, n)


def plant_triplet_edges(rng, rows, cols, r, c, v):
    """Appends cells with edge runs (each at a fresh cell, scattered through the order):
    a lone -0.0; x, -x (cancels to +0.0, kept); -0.0 three times (stays -0.0); 1e308, 1e308,
    -1e308 (+Inf in insertion order) and 1e308, -1e308, 1e308 (1e308); a NaN member; +Inf with
    -Inf (NaN); +Inf with finite members (+Inf).  Returns the new arrays and the edge cells."""
    taken = set(zip(r.tolist(), c.tolist()))
    x = float(v[0])
    groups = [[-0.0], [x, -x], [x, -x, -0.0], [-0.0, -0.0, -0.0], [BIG, BIG, -BIG],
              [BIG, -BIG, BIG], [1.5, np.nan, -2.0, 3.0], [np.inf, 2.0, -np.inf],
              [np.inf, 1.0, 2.0, -7.0]]
    cells = []
    while len(cells) < len(groups):
        cell = (int(rng.integers(0, rows)), int(rng.integers(0, cols)))
        if cell not in taken:
            taken.add(cell)
            cells.append(cell)
    er = np.concatenate([[cl[0]] * len(g) for cl, g in zip(cells, groups)]).astype(np.int64)
    ec = np.concatenate([[cl[1]] * len(g) for cl, g in zip(cells, groups)]).astype(np.int64)
    ev = np.concatenate(groups)
    # members of each edge group keep their relative order, spread through the array
    n = len(r) + len(er)
    slots = np.sort(rng.choice(n, len(er), replace=False))
    is_edge = np.zeros(n, dtype=bool)
    is_edge[slots] = True
    R, Cc, V = np.empty(n, np.int64), np.empty(n, np.int64), np.empty(n)
    R[is_edge], Cc[is_edge], V[is_edge] = er, ec, ev
    R[~is_edge], Cc[~is_edge], V[~is_edge] = r, c, v
    return R, Cc, V, cells


def _csr_lookup(want, cell):
    ip, ind, d = want
    s, e = int(ip[cell[0]]), int(ip[cell[0] + 1])
    k = s + int(np.searchsorted(ind[s:e].astype(np.int64), cell[1]))
    assert k < e and int(ind[k]) == cell[1]
    return d[k]


def triplet_sensitivity(O, rng, shape, r, c, v):
    """Share of the >= 3-term entries whose bits change when the oracle sums the same triplets
    in another insertion order."""
    want = O.triplets_to_csr(shape, r, c, v, np.uint32)
    perm = rng.permutation(len(r))
    other = O.triplets_to_csr(shape, r[perm], c[perm], v[perm], np.uint32)
    assert np.array_equal(want[0], other[0]) and np.array_equal(want[1], other[1])
    ones = O.triplets_to_csr(shape, r, c, np.ones(len(r)), np.uint32)[2]
    three = ones >= 3
    return three.sum(), float((u64(want[2][three]) != u64(other[2][three])).mean())


TRIPLET_SHAPES = {(1, 1): (200, 250), (1, 2): (230, 3000), (2, 1): (3000, 200),
                  (2, 3): (3000, 70_000), (3, 4): (70_000, (1 << 24) + 1)}


def _from_triplets_dev(sp, shape, r, c, v):
    import torch
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    dev = G._device(ctx)
    tr = torch.from_numpy(r.astype(np.uint32).view(np.int32)).to(dev)
    tc = torch.from_numpy(c.astype(np.uint32).view(np.int32)).to(dev)
    tv = torch.from_numpy(np.ascontiguousarray(v)).to(dev)
    G._sync()
    h = C.c_void_p()
    ctx.check(ctx.lib.sprs_b200_csmat_from_triplets_dev(ctx.h, shape[0], shape[1], len(r),
                                                        G._dptr(tr), G._dptr(tc), G._dptr(tv),
                                                        C.byref(h)))
    return sp.DeviceCsMat(ctx, h).download()


@pytest.mark.parametrize("pc", list(TRIPLET_SHAPES))
def test_from_triplets_duplicate_order_bits(sp, O, pc):
    """Duplicate runs of 3 to 50 real-valued members, summed in insertion order, at (row, col)
    radix pass counts `pc`; through the host and the device-array entry points."""
    shape = TRIPLET_SHAPES[pc]
    rng = np.random.default_rng(pc[0] * 10 + pc[1])
    r, c, _ = triplet_case(rng, *shape)
    seams = triplet_seams(r, c, *shape)
    assert seams["passes"] == pc
    for k in ("col_warp", "col_block", "row_warp", "row_block"):
        assert seams[k] >= 20, "%s: only %d runs straddle (%s)" % (k, seams[k], seams)
    v = triplet_values(rng, len(r))
    n3, share = triplet_sensitivity(O, rng, shape, r, c, v)
    assert n3 >= 300 and share >= MIN_SHARE, (n3, share)
    R, Cc, V, cells = plant_triplet_edges(rng, *shape, r, c, v)
    want = O.triplets_to_csr(shape, R, Cc, V, np.uint64)
    ev = [_csr_lookup(want, cl) for cl in cells]
    expect = [-0.0, 0.0, 0.0, -0.0, np.inf, BIG, np.nan, np.nan, np.inf]
    exact.assert_same_class(ev, expect, "oracle edge cells")
    for what in ("host", "dev"):
        if what == "host":
            m = sp.CsMat.from_triplets(shape, R, Cc, V)
            got = (m.indptr, m.indices, m.data)
        else:
            got = _from_triplets_dev(sp, shape, R, Cc, V)
        exact.assert_csr_bits((got[0], got[1], np.zeros(len(got[2]))),
                              (want[0], want[1], np.zeros(len(want[2]))), what + ": structure")
        exact.assert_same_class(got[2], want[2], "from_triplets %s %s" % (what, pc))


def test_from_triplets_single_negative_zero_bits(sp, O):
    """One -0.0 triplet stays -0.0 (the run's sum starts from its first value, not +0.0)."""
    for entry in ("host", "dev"):
        r, c, v = np.array([3]), np.array([5]), np.array([-0.0])
        if entry == "host":
            m = sp.CsMat.from_triplets((4, 9), r, c, v)
            got = (m.indptr, m.indices, m.data)
        else:
            got = _from_triplets_dev(sp, (4, 9), r, c, v)
        exact.assert_csr_bits(got, O.triplets_to_csr((4, 9), r, c, v), entry)
        assert np.signbit(got[2][0])


# ---------------------------------------------------------------- 1c: product routes
def product_operand(rng, rows, cols, long_rows=6):
    """CSR arrays with short rows, empty rows and `long_rows` rows of 120-260 non-zeros."""
    lens = rng.integers(0, 9, rows)
    lens[rng.random(rows) < 0.1] = 0
    lens[rng.choice(rows, long_rows, replace=False)] = rng.integers(120, 261, long_rows)
    ip, ind = _csr_from_lens(rng, np.minimum(lens, cols), cols)
    d = real_values(rng, len(ind))
    d[rng.choice(len(d), 5, replace=False)] = -0.0
    return ip, ind, d


def csc_of(O, rows, cols, csr):
    """The CSC arrays of a CSR matrix (convert_mat_storage)."""
    return O.convert_mat_storage(rows, cols, *csr)


def column_permuted(O, rng, rows, cols, csr):
    """The same matrix with its columns permuted: A P (CSR) and P^T's row permutation, so that
    A P times P^T B has the same terms as A B, summed in another order."""
    perm = rng.permutation(cols)
    ip, ind, d = csr
    rr = np.repeat(np.arange(rows), np.diff(ip.astype(np.int64)))
    nk = perm[ind.astype(np.int64)]
    o = np.lexsort((nk, rr))
    return (ip, nk[o].astype(np.uint32), d[o]), np.argsort(perm)


def assert_product_sensitivity(O, rng, rows, cols, csr, b, c0):
    """A P times P^T B changes >= 15 % of the output elements of >= 3 terms (c0 and >= 2
    products)."""
    want = O.csr_mulacc_dense_rowmaj(*csr, b, c0.copy())
    ap, inv = column_permuted(O, rng, rows, cols, csr)
    other = O.csr_mulacc_dense_rowmaj(*ap, np.ascontiguousarray(b[inv]), c0.copy())
    three = np.diff(csr[0].astype(np.int64)) >= 2
    assert three.sum() >= 20
    share = float((u64(want[three]) != u64(other[three])).mean())
    assert share >= MIN_SHARE, share
    assert np.diff(csr[0].astype(np.int64)).max() > 100


@pytest.mark.parametrize("k", [8, 33, 64, 66, 129])
def test_csc_mulacc_dense_rowmaj_bits(sp, O, k):
    """csc_mulacc_dense_rowmaj into a non-zero out, and `A_csc * B` from zero: the SpMM on the
    cached CSR conversion, bit for bit against prod.rs:219-241."""
    rng = np.random.default_rng(300 + k)
    rows, cols = 600, 900
    csr = product_operand(rng, rows, cols)
    csc = csc_of(O, rows, cols, csr)
    b = real_values(rng, cols * k).reshape(cols, k)
    c0 = real_values(rng, rows * k).reshape(rows, k)
    assert_product_sensitivity(O, rng, rows, cols, csr, b, c0)
    A = sp.CsMat.new_csc((rows, cols), *csc)
    got = c0.copy()
    sp.prod.csc_mulacc_dense_rowmaj(A, b, got)
    exact.assert_bits(got, O.csc_mulacc_dense_rowmaj(*csc, b, c0.copy()), "csc rowmaj k=%d" % k)
    prod = A * b
    assert prod.flags.c_contiguous
    exact.assert_bits(prod, O.csc_mulacc_dense_rowmaj(*csc, b, np.zeros((rows, k))),
                      "A_csc * B k=%d" % k)


def model_colmaj(csr, b, c0):
    """One SpMV per rhs column in the SpMV's order (tests/spmv_model.py)."""
    return np.stack([M.spmv(*csr, b[:, j], y0=c0[:, j]) for j in range(b.shape[1])], axis=1)


def check_colmaj(O, csr, b, c0, got, oracle_out, what):
    """got == the model bit for bit, and == the oracle on the rows summed in storage order."""
    exact.assert_bits(got, model_colmaj(csr, np.ascontiguousarray(b), np.ascontiguousarray(c0)), what)
    rows_so = M.storage_order_rows(csr[0])
    assert rows_so.sum() >= 50, what + ": too few rows summed in storage order"
    exact.assert_bits(got[rows_so], oracle_out[rows_so], what + ": storage-order rows vs oracle")


@pytest.mark.parametrize("k", [1, 3, 7])
def test_csc_mulacc_dense_colmaj_bits(sp, O, k):
    """csc_mulacc_dense_colmaj and `A_csc * B` (k < 8, F-order result): one SpMV per column on
    the CSR conversion."""
    rng = np.random.default_rng(320 + k)
    rows, cols = 600, 900
    csr = product_operand(rng, rows, cols)
    csc = csc_of(O, rows, cols, csr)
    b = real_values(rng, cols * k).reshape(cols, k)
    c0 = np.asfortranarray(real_values(rng, rows * k).reshape(rows, k))
    # the oracle's CSC order (column by column) differs from the CSR row order on the long rows
    A = sp.CsMat.new_csc((rows, cols), *csc)
    got = c0.copy(order="F")
    sp.prod.csc_mulacc_dense_colmaj(A, b, got)
    check_colmaj(O, csr, b, c0, got, O.csc_mulacc_dense_colmaj(*csc, b, c0.copy(order="F")),
                 "csc colmaj k=%d" % k)
    prod = A * b
    assert prod.flags.f_contiguous and not prod.flags.c_contiguous or k == 1
    check_colmaj(O, csr, b, np.zeros((rows, k)), prod,
                 O.csc_mulacc_dense_colmaj(*csc, b, np.zeros((rows, k), order="F")), "A_csc * B k=%d" % k)


@pytest.mark.parametrize("storage", ["csr", "csc"])
@pytest.mark.parametrize("k", [3, 40])
def test_dense_times_sparse_bits(sp, O, storage, k):
    """`D @ A` = (A^T . D^T)^T (csmat.rs:2050-2099): the product of the transposed operands by
    the route of its width, F-order like `reversed_axes`."""
    rng = np.random.default_rng(340 + k + (storage == "csc"))
    rows, cols = 500, 700  # A is rows x cols, D is k x rows
    csr = product_operand(rng, rows, cols)
    D = real_values(rng, k * rows).reshape(k, rows)
    if storage == "csr":
        A = sp.CsMat.new((rows, cols), *csr)
        t_arrays = csr      # A^T is CSC with A's arrays
    else:
        csc = csc_of(O, rows, cols, csr)
        A = sp.CsMat.new_csc((rows, cols), *csc)
        t_arrays = csc      # A^T is CSR with A's CSC arrays
    got = D @ A
    # reversed_axes of the inner product: C-order (k >= 8) becomes F-order, F-order C-order
    assert got.shape == (k, cols) and (got.flags.f_contiguous if k >= 8 else got.flags.c_contiguous)
    zero = np.zeros((cols, k))
    if storage == "csr":   # A^T (cols x rows) CSC
        if k >= 8:
            want = O.csc_mulacc_dense_rowmaj(*t_arrays, D.T, zero)
            exact.assert_bits(got.T, want, "D @ A_csr k=%d" % k)
        else:
            t_csr = O.convert_mat_storage(rows, cols, *csr)   # CSR of A^T
            check_colmaj(O, t_csr, D.T, zero, got.T,
                         O.csc_mulacc_dense_colmaj(*t_arrays, D.T, zero.copy(order="F")),
                         "D @ A_csr k=%d" % k)
    else:                  # A^T (cols x rows) CSR = the CSC arrays of A
        if k >= 8:
            want = O.csr_mulacc_dense_rowmaj(*t_arrays, D.T, zero)
            exact.assert_bits(got.T, want, "D @ A_csc k=%d" % k)
        else:
            check_colmaj(O, t_arrays, D.T, zero, got.T,
                         O.csr_mulacc_dense_colmaj(*t_arrays, D.T, zero.copy(order="F")),
                         "D @ A_csc k=%d" % k)


def rhs_views(rng, cols, k):
    """Strided rhs views (name, view) of shape (cols, k)."""
    base = real_values(rng, cols * k).reshape(cols, k)
    big = real_values(rng, (2 * cols + 1) * (3 * k + 2)).reshape(2 * cols + 1, 3 * k + 2)
    return [("transposed", real_values(rng, k * cols).reshape(k, cols).T),
            ("F-order", np.asfortranarray(base)),
            ("step-sliced", big[1::2, 2::3][:cols, :k]), ("rows reversed", base[::-1]),
            ("columns reversed", base[:, ::-1]),
            ("broadcast", np.broadcast_to(real_values(rng, k), (cols, k)))]


@pytest.mark.parametrize("route", ["csr_mulacc_dense_rowmaj", "csc_mulacc_dense_rowmaj",
                                   "csr_mulacc_dense_colmaj", "csc_mulacc_dense_colmaj"])
def test_dense_views_bits(sp, O, route):
    """prod.*_mulacc_dense_* on strided rhs views (transposed, F-order, step-sliced, negative
    strides, zero stride) into an `out` window of a sentinel-filled array: the result equals
    the same product on contiguous copies, and nothing outside the window changes."""
    rng = np.random.default_rng(360 + len(route) + route.startswith("csc"))
    rows, cols = 300, 400
    k = 12 if "rowmaj" in route else 5
    csr = product_operand(rng, rows, cols, long_rows=3)
    arrays = csr if route.startswith("csr") else csc_of(O, rows, cols, csr)
    A = (sp.CsMat.new if route.startswith("csr") else sp.CsMat.new_csc)((rows, cols), *arrays)
    sentinel = -7.25
    assert_product_sensitivity(O, rng, rows, cols, csr, real_values(rng, cols * k).reshape(cols, k),
                               real_values(rng, rows * k).reshape(rows, k))
    for name, b in rhs_views(rng, cols, k):
        for out_kind in ("window", "window reversed"):
            host = np.full((2 * rows + 3, 3 * k + 2), sentinel)
            out = host[1::2, 2::3][:rows, :k]
            if out_kind == "window reversed":
                out = out[::-1, ::-1]
            c0 = real_values(rng, rows * k).reshape(rows, k)
            out[...] = c0
            getattr(sp.prod, route)(A, b, out)
            what = "%s, rhs %s, out %s" % (route, name, out_kind)
            bc = np.ascontiguousarray(b)
            if "rowmaj" in route:
                want = getattr(O, route)(*arrays, bc, c0.copy())
                exact.assert_bits(out, want, what)
            else:
                check_colmaj(O, csr, bc, c0, out, getattr(O, route)(*arrays, bc, c0.copy(order="F")),
                             what)
            mask = np.ones(host.shape, dtype=bool)
            mask[1::2, 2::3][:rows, :k] = False
            assert np.all(host[mask] == sentinel), what + ": elements outside the window changed"


def test_csc_csr_cache_reuse_bits(sp, O):
    """One CSC mirror through mul_acc_mat_vec_csc, csc_mulacc_dense_rowmaj, then the SpMV again:
    the cached CSR conversion is built once and gives the same bits each time."""
    rng = np.random.default_rng(380)
    rows, cols = 600, 900
    csr = product_operand(rng, rows, cols)
    csc = csc_of(O, rows, cols, csr)
    A = sp.CsMat.new_csc((rows, cols), *csc)
    x = real_values(rng, cols)
    y0 = real_values(rng, rows)
    b = real_values(rng, cols * 16).reshape(cols, 16)
    c0 = real_values(rng, rows * 16).reshape(rows, 16)
    want_y = M.spmv(*csr, x, y0=y0)
    ys, launches = [], []
    ctx = A.context()
    for step in range(2):
        y = y0.copy()
        n0 = ctx.launches
        sp.prod.mul_acc_mat_vec_csc(A, x, y)
        launches.append(ctx.launches - n0)
        exact.assert_bits(y, want_y, "mul_acc_mat_vec_csc, call %d" % step)
        ys.append(y)
        out = c0.copy()
        sp.prod.csc_mulacc_dense_rowmaj(A, b, out)
        exact.assert_bits(out, O.csc_mulacc_dense_rowmaj(*csc, b, c0.copy()),
                          "csc_mulacc_dense_rowmaj, call %d" % step)
    assert launches[1] < launches[0], "the second SpMV converted again: %s" % launches
    rows_so = M.storage_order_rows(csr[0])
    exact.assert_bits(ys[0][rows_so], O.mul_acc_mat_vec_csc(*csc, x, y0.copy())[rows_so],
                      "SpMV storage-order rows vs oracle")


def test_csc_times_csvec_bits(sp, O):
    """`A_csc * v` = A * col_view(v) (vec.rs:1104-1131), the SpGEMM, against the oracle's
    col^T A^T."""
    rng = np.random.default_rng(390)
    rows, cols = 2000, 3000
    csr = product_operand(rng, rows, cols, long_rows=40)
    csc = csc_of(O, rows, cols, csr)
    A = sp.CsMat.new_csc((rows, cols), *csc)
    idx = np.sort(rng.choice(cols, 1500, replace=False))
    vd = real_values(rng, len(idx))
    vd[::37] = -0.0
    want = O.mul_csr_csr((1, cols), (np.array([0, len(idx)], dtype=np.uint32), idx.astype(np.uint32), vd),
                         (cols, rows), csc, threads=1)
    ones = O.mul_csr_csr((1, cols), (np.array([0, len(idx)], dtype=np.uint32), idx.astype(np.uint32),
                                     np.ones(len(idx))), (cols, rows),
                         (csc[0], csc[1], np.ones(len(csc[2]))), threads=1)[2]
    three = ones >= 3
    assert three.sum() >= 100
    # the same product with the inner dimension permuted: the terms in another order
    perm = rng.permutation(cols)
    inv = np.argsort(perm)
    o = np.argsort(perm[idx])
    b_ip = csc[0].astype(np.int64)
    lens = np.diff(b_ip)[inv]
    bp_ip = np.zeros(cols + 1, dtype=np.int64)
    np.cumsum(lens, out=bp_ip[1:])
    src = np.repeat(b_ip[:-1][inv] - bp_ip[:-1], lens) + np.arange(int(bp_ip[-1]))
    other = O.mul_csr_csr((1, cols), (np.array([0, len(idx)], dtype=np.uint32),
                                      np.sort(perm[idx]).astype(np.uint32), vd[o]),
                          (cols, rows), (bp_ip.astype(np.uint32), csc[1][src], csc[2][src]), threads=1)
    assert np.array_equal(other[1], want[1])
    assert (u64(other[2][three]) != u64(want[2][three])).mean() >= MIN_SHARE
    got = A * sp.CsVec(cols, idx, vd)
    exact.assert_bits(got.indices.astype(np.float64), want[1].astype(np.float64), "indices")
    exact.assert_bits(got.data, want[2], "A_csc * CsVec")


# ---------------------------------------------------------------- 1d: sparse-vector dots
def ref_dot_acc(i1, d1, i2, d2):
    """vec.rs:846-881 dot_acc: merge over both patterns, sum from +0.0."""
    s, p, q = 0.0, 0, 0
    while p < len(i1) and q < len(i2):
        if i1[p] == i2[q]:
            s = s + d1[p] * d2[q]
        if i1[p] <= i2[q]:
            p += 1
        else:
            q += 1
    return s


def ref_dot_dense_acc(i1, d1, dense):
    """dot with a dense rhs (dot_acc): sum from +0.0."""
    s = 0.0
    for i, v in zip(i1, d1):
        s = s + v * dense[i]
    return s


def ref_dot_dense(i1, d1, dense):
    """vec.rs:894-904 dot_dense: `Iterator::sum`, which folds from -0.0 in std's f64 Sum
    (rust-lang/rust#129321, in the reference's rust-version 1.88; pinned from the std source,
    not from a run)."""
    s = -0.0
    for i, v in zip(i1, d1):
        s = s + v * dense[i]
    return s


def ref_binary_search(i1, d1, i2, d2):
    """prod.rs:13-72: walk the vector with fewer entries, binary-search the other's tail."""
    swapped = len(i1) > len(i2)
    a_i, a_d, b_i, b_d = (i2, d2, i1, d1) if swapped else (i1, d1, i2, d2)
    s, lo = 0.0, 0
    for i, v in zip(a_i, a_d):
        j = lo + int(np.searchsorted(b_i[lo:], i))
        if j < len(b_i) and b_i[j] == i:
            s = s + ((b_d[j] * v) if swapped else (v * b_d[j]))
        lo = j
    return s


def _vec(rng, dim, n):
    idx = np.sort(rng.choice(dim, n, replace=False))
    return idx, real_values(rng, n)


def test_csvec_dots_bits(sp, O):
    """dot (sparse and dense rhs), dot_dense and csvec_dot_by_binary_search bit for bit against
    sequential loops that restate each reference function; empty and all-(-0.0) cases too."""
    rng = np.random.default_rng(400)
    dim = 5000
    i1, d1 = _vec(rng, dim, 1200)
    i2, d2 = _vec(rng, dim, 2500)
    d1[::29] = -0.0
    dense = real_values(rng, dim)
    dense[::31] = 0.0
    common = np.intersect1d(i1, i2)
    assert len(common) >= 300
    # sensitivity: the same common terms summed in reverse order
    terms = d1[np.isin(i1, common)] * d2[np.isin(i2, common)]
    fwd = ref_dot_acc(i1, d1, i2, d2)
    rev = 0.0
    for t in terms[::-1]:
        rev = rev + t
    assert u64(fwd) != u64(rev)
    v1, v2 = sp.CsVec(dim, i1, d1), sp.CsVec(dim, i2, d2)
    cases = [("dot sparse", v1.dot(v2), fwd),
             ("dot sparse, swapped", v2.dot(v1), ref_dot_acc(i2, d2, i1, d1)),
             ("dot dense", v1.dot(dense), ref_dot_dense_acc(i1, d1, dense)),
             ("dot_dense", v1.dot_dense(dense), ref_dot_dense(i1, d1, dense)),
             ("binary search", sp.prod.csvec_dot_by_binary_search(v1, v2), ref_binary_search(i1, d1, i2, d2)),
             ("binary search, swapped", sp.prod.csvec_dot_by_binary_search(v2, v1),
              ref_binary_search(i2, d2, i1, d1))]
    assert u64(cases[4][2]) == u64(O.csvec_dot_by_binary_search(i1, d1, i2, d2))
    # degenerate: empty, and every product -0.0 (negative values times +0.0)
    empty = sp.CsVec.empty(dim)
    neg_idx = np.sort(rng.choice(dim, 40, replace=False))
    neg = sp.CsVec(dim, neg_idx, -np.abs(real_values(rng, 40)))
    zeros = np.zeros(dim)
    zvec = sp.CsVec(dim, neg_idx, np.zeros(40))
    cases += [("dot_dense, empty", empty.dot_dense(dense), ref_dot_dense([], [], dense)),
              ("dot_dense, all -0.0", neg.dot_dense(zeros), ref_dot_dense(neg_idx, neg.data, zeros)),
              ("dot_dense, +0.0 terms", zvec.dot_dense(zeros), ref_dot_dense(neg_idx, zvec.data, zeros)),
              ("dot dense, empty", empty.dot(dense), ref_dot_dense_acc([], [], dense)),
              ("dot dense, all -0.0", neg.dot(zeros), ref_dot_dense_acc(neg_idx, neg.data, zeros)),
              ("dot sparse, all -0.0", neg.dot(zvec), ref_dot_acc(neg_idx, neg.data, neg_idx, zvec.data)),
              ("dot sparse, empty", empty.dot(v1), 0.0),
              ("binary search, empty", sp.prod.csvec_dot_by_binary_search(empty, v1), 0.0),
              ("binary search, all -0.0", sp.prod.csvec_dot_by_binary_search(neg, zvec),
               ref_binary_search(neg_idx, neg.data, neg_idx, zvec.data))]
    assert np.signbit(ref_dot_dense(neg_idx, neg.data, zeros)) and np.signbit(ref_dot_dense([], [], dense))
    for what, got, want in cases:
        exact.assert_bits(np.array([got]), np.array([want]), what)


# ---------------------------------------------------------------- 1f: full size
def _device_convert(sp, O, a, what):
    t = a.mirror.to_other_storage()
    got = t.download()
    hip, hind, hdat = a.to_host()
    want = O.convert_mat_storage(a.rows, a.cols, hip, hind, hdat)
    _check_convert(got, want, what)
    return hip, hind


def test_to_other_storage_rand_1m_full_size(sp, O):
    """BASELINE config 2 (1M x 1M, 32 non-zeros per row, N(0,1)): 3 radix passes."""
    from sprs_b200 import generate as G
    a = G.rand_csr(sp.Context.default(), 1_000_000, 1_000_000, 32, seed=0x5EED0002)
    assert passes(a.cols) == 3
    _device_convert(sp, O, a, "config 2")


def test_to_other_storage_rmat_500k_full_size(sp, O):
    """BASELINE config 4's A (500k R-MAT): its hub column holds over five sort blocks of
    entries (22 665 with this seed)."""
    from sprs_b200 import generate as G
    a = G.rmat_csr(sp.Context.default(), 500_000, 16, seed=0x5EED0004)
    _, hind = _device_convert(sp, O, a, "config 4 A")
    assert np.bincount(hind.astype(np.int64)).max() >= 5 * RS_CHUNK


def test_from_triplets_rand_1m_full_size(sp, O):
    """Config 2's triplets shuffled, with ~10 % of the cells repeated 3 to 8 times (real values,
    the copies scattered over the whole array), on the device against the oracle."""
    from sprs_b200 import generate as G
    a = G.rand_csr(sp.Context.default(), 1_000_000, 1_000_000, 32, seed=0x5EED0002)
    ip, ind, d = a.to_host()
    rng = np.random.default_rng(500)
    rows = np.repeat(np.arange(a.rows, dtype=np.int64), np.diff(ip.astype(np.int64)))
    cols = ind.astype(np.int64)
    rep = np.flatnonzero(rng.random(len(cols)) < 0.10)
    extra = rng.integers(2, 8, len(rep))  # 3 to 8 members in all
    src = np.repeat(rep, extra)
    r = np.concatenate([rows, rows[src]])
    c = np.concatenate([cols, cols[src]])
    v = np.concatenate([d, real_values(rng, len(src))])
    perm = rng.permutation(len(r))
    r, c, v = r[perm], c[perm], v[perm]
    shape = (a.rows, a.cols)
    want = O.triplets_to_csr(shape, r, c, v, np.uint32)
    got = _from_triplets_dev(sp, shape, r, c, v)
    exact.assert_csr_bits(got, want, "config 2 triplets")


# ---------------------------------------------------------------- 1g: 64-bit indptr
def test_convert_bits_indptr64_child_process():
    """This file's small cases again with SPRS_B200_FORCE_INDPTR64=1 (read once per process):
    gather_transposed_kernel<uint64_t> and the 64-bit SpMM / SpMV behind the CSC routes.  The
    CsVec case is left out: the SpGEMM takes 32-bit indptr operands only."""
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu",
                        os.path.abspath(__file__), "-k",
                        "not full_size and not child_process and not csc_times_csvec"],
                       capture_output=True, text=True, timeout=1500, cwd=ROOT,
                       env=dict(os.environ, SPRS_B200_FORCE_INDPTR64="1"))
    assert r.returncode == 0 and " passed" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
