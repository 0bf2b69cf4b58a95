"""The dense boundary on the device (the dense section of csrc/transpose.cu): to_dense,
assign_to_dense, csr_from_dense / csc_from_dense and the sparse (+) dense binops, against the CPU restatement of the reference's
loops (tests/dense_oracle.cpp) and its known answers (tests/golden/dense_fixtures.json).  Copies
compare bit for bit with NaN payloads; arithmetic results bit for bit with NaN by class.

The small tests also run on the emulated build of tests/emu (tests/test_emu_preflight.py);
`*_full_size`, `*_child_process` and `test_cpp*` ones need the H100."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import dense_oracle as DO
from conftest import ROOT, rand_csr

pytestmark = pytest.mark.gpu

SPECIALS = np.array([np.inf, -np.inf, np.nan, -np.nan, 0.0, -0.0, 5e-324, -5e-324, 2.2e-308,
                     1.5, -2.0, 1e308])
# a NaN with a payload, and one with the sign bit: copies must keep both
NAN_PAYLOAD = np.array([0x7FF0000000000ABC, 0xFFF8000000000123], dtype=np.uint64).view(np.float64)


@pytest.fixture(scope="module")
def sp():
    import sprs_b200
    sprs_b200._lib.load()
    return sprs_b200


@pytest.fixture(scope="module")
def kats():
    with open(os.path.join(ROOT, "tests", "golden", "dense_fixtures.json")) as f:
        return json.load(f)


def csmat(sp, m, idx=np.uint64):
    cls = sp.CsMat.new if m["storage"] == "CSR" else sp.CsMat.new_csc
    return cls(tuple(m["shape"]), np.array(m["indptr"], idx), np.array(m["indices"], idx),
               np.array(m["data"], np.float64))


def special_matrix(sp, rng, rows, cols, npr, frac=0.3, storage="CSR"):
    ip, ind, d = rand_csr(rng, rows, cols, npr)
    pool = np.concatenate([SPECIALS, NAN_PAYLOAD])
    d = np.where(rng.random(d.size) < frac, rng.choice(pool, d.size), d)
    a = sp.CsMat.new((rows, cols), ip, ind, d)
    return a if storage == "CSR" else a.to_other_storage()


def special_dense(rng, rows, cols, frac=0.2):
    d = rng.standard_normal((rows, cols))
    pool = np.concatenate([SPECIALS, NAN_PAYLOAD])
    m = rng.random((rows, cols)) < frac
    d[m] = rng.choice(pool, int(m.sum()))
    return d


def assert_from_dense(got, want):
    ip, ind, d = want
    assert np.array_equal(got.indptr.astype(np.uint64), ip)
    assert np.array_equal(got.indices.astype(np.uint64), ind)
    assert DO.same_bits(got.data, d)


def oracle_binop(m, op, alpha, beta, rhs, order):
    out = np.zeros(rhs.shape, order=order)
    DO.binop_dense(m, op, alpha, beta, rhs, out)
    return out


# ---- 1. the reference's known answers through the Python mirror
@pytest.mark.parametrize("idx", [np.uint32, np.uint64])
def test_dense_kats(sp, kats, idx):
    eye = np.array(kats["eye3_dense"])
    for key in ("eye3_csr", "eye3_csc"):                                     # to_dense.rs:56-72
        m = csmat(sp, kats[key], idx)
        d = np.zeros((3, 3))
        sp.assign_to_dense(d, m)
        assert np.array_equal(d, eye)
    assert np.array_equal(csmat(sp, kats["mat1"], idx).to_dense(), kats["to_dense_mat1"])
    assert np.array_equal(csmat(sp, kats["mat3"], idx).to_dense(), kats["to_dense_mat3"])
    assert sp.CsMat.csr_from_dense(eye, 0.0, idx) == csmat(sp, kats["eye3_csr"], idx)
    assert sp.CsMat.csc_from_dense(eye, 0.0, idx) == csmat(sp, kats["eye3_csc"], idx)
    fd = np.array(kats["from_dense_in"])
    got = sp.CsMat.csr_from_dense(fd, kats["from_dense_eps"], idx)
    assert got == csmat(sp, kats["csr_from_dense_out"], idx) and got.indices.dtype == idx
    assert sp.CsMat.csc_from_dense(fd, kats["from_dense_eps"], idx) == \
        csmat(sp, kats["csc_from_dense_out"], idx)
    # binop.rs:600-718
    a, b = csmat(sp, kats["mat1"], idx), np.array(kats["mat_dense1"])
    assert np.array_equal(sp.binop.add_dense_mat_same_ordering(a, b, 1.0, 1.0), kats["add_dense_out"])
    assert np.array_equal(a + b, kats["add_dense_out"])
    e = csmat(sp, kats["eye3_csr"], idx)
    assert np.array_equal(sp.binop.add_dense_mat_same_ordering(e, np.zeros((3, 3)), 1.0, 1.0), eye)
    assert np.array_equal(sp.binop.mul_dense_mat_same_ordering(e, np.ones((3, 3)), 1.0), eye)
    c = sp.binop.mul_dense_mat_same_ordering(e, np.ones((6, 6))[::2, ::2], 1.0)   # mul_dense_strided
    assert c.flags.c_contiguous and np.array_equal(c, eye)
    ec = csmat(sp, kats["eye3_csc"], idx)
    c = sp.binop.mul_dense_mat_same_ordering(ec, np.asfortranarray(np.ones((6, 6)))[::2, ::2], 1.0)
    assert c.T.flags.c_contiguous and np.array_equal(c, eye)
    # binop_standard_layouts / binop_strided_layouts: accepted without a panic
    z, zc = sp.CsMat.zero((3, 4)), sp.CsMat.zero((3, 4)).to_other_storage()
    sp.binop.csmat_binop_dense_raw_add(z, np.ones((3, 4)), 1.0, 1.0, np.ones((3, 4)))
    sp.binop.csmat_binop_dense_raw_add(zc, np.ones((3, 4), order="F"), 1.0, 1.0, np.zeros((3, 4), order="F"))
    sp.binop.csmat_binop_dense_raw_add(z, np.ones((3, 8))[:, ::2], 1.0, 1.0, np.zeros((3, 4)))
    sp.binop.csmat_binop_dense_raw_add(zc, np.ones((3, 8), order="F")[:, ::2], 1.0, 1.0,
                                       np.zeros((3, 4), order="F"))


# ---- 2. value classes, and the alpha / beta traps of the closures
@pytest.mark.parametrize("storage", ["CSR", "CSC"])
def test_dense_value_classes(sp, storage):
    rng = np.random.default_rng(17)
    a = special_matrix(sp, rng, 37, 53, 12, storage=storage)
    assert DO.same_bits(a.to_dense(), DO.to_dense(a))
    d = special_dense(rng, 37, 53)
    order = "C" if storage == "CSR" else "F"
    dv = np.asarray(d, order=order)
    for alpha in (1.0, -1.0, 0.0, -0.0, 0.5, np.inf, np.nan):
        for beta in (1.0, -1.0, 0.0, -0.0, 0.5, np.inf, np.nan):
            got = sp.binop.add_dense_mat_same_ordering(a, dv, alpha, beta)
            assert DO.same_values(got, oracle_binop(a, DO.ADD, alpha, beta, dv, order)), (alpha, beta)
        got = sp.binop.mul_dense_mat_same_ordering(a, dv, alpha)
        assert DO.same_values(got, oracle_binop(a, DO.MUL, alpha, 0.0, dv, order)), alpha
    # the literal consequences (binop.rs closures): -0.0 in D at a missing position
    e = sp.CsMat.new((1, 4), np.array([0, 1]), np.array([0]), np.array([2.0]))
    s = sp.binop.add_dense_mat_same_ordering(e, np.array([[1.0, -0.0, -3.0, np.inf]]), 1.0, 1.0)
    assert DO.same_bits(s, [[3.0, 0.0, -3.0, np.inf]])                     # -0.0 became +0.0
    m = sp.binop.mul_dense_mat_same_ordering(e, np.array([[1.0, -5.0, np.inf, np.nan]]), 1.0)
    assert DO.same_bits(m[:, :2], [[2.0, -0.0]]) and np.isnan(m[0, 2:]).all()
    p = sp.binop.add_dense_mat_same_ordering(e, np.ones((1, 4)), np.inf, 1.0)
    assert p[0, 0] == np.inf and np.isnan(p[0, 1:]).all()                   # inf * 0 poisons


def test_dense_copies_keep_bits(sp):
    """to_dense / assign / from_dense copy the stored bits: NaN payloads, -0.0, subnormals."""
    vals = np.concatenate([NAN_PAYLOAD, [-0.0, 5e-324, -np.inf]])
    a = sp.CsMat.new((2, 5), np.array([0, 3, 5]), np.array([0, 2, 4, 1, 3]), vals)
    d = a.to_dense()
    assert DO.same_bits(d, DO.to_dense(a))
    assert d.view(np.uint64)[0, 0] == 0x7FF0000000000ABC and d.view(np.uint64)[0, 2] == \
        0xFFF8000000000123 and d.view(np.uint64)[0, 4] == np.float64(-0.0).view(np.uint64)
    out = np.full((2, 5), 1.0)
    sp.assign_to_dense(out, a)
    assert DO.same_bits(out.ravel()[[0, 2, 4, 6, 8]], vals)
    f = sp.CsMat.csr_from_dense(d, 0.0)          # NaN and -0.0 are dropped, the rest kept as bits
    assert f.indptr.tolist() == [0, 0, 2] and f.indices.tolist() == [1, 3]
    assert DO.same_bits(f.data, vals[[3, 4]])


# ---- 3. epsilon classes
@pytest.mark.parametrize("eps", [-1.0, -0.0, 0.0, np.nan, np.inf, 5e-324, 0.5, 1.5])
def test_dense_from_dense_eps(sp, eps):
    rng = np.random.default_rng(5)
    d = special_dense(rng, 29, 41, frac=0.4)
    d[3, :5] = [0.5, -0.5, 1.5, -1.5, np.nextafter(0.5, 1)]   # |x| == eps is dropped
    for f, fo in ((sp.CsMat.csr_from_dense, DO.csr_from_dense),
                  (sp.CsMat.csc_from_dense, DO.csc_from_dense)):
        got = f(d, eps)
        assert_from_dense(got, fo(d, eps))
    kept = sp.CsMat.csr_from_dense(d, eps)
    e = eps if eps > 0 else 0.0
    assert kept.nnz() == int(np.count_nonzero(np.abs(d) > e))


# ---- 4. layouts, shapes and the panics
def views(d):
    f = np.asfortranarray(d)
    return {"C": d, "F": f, "cols::2": np.repeat(d, 2, axis=1)[:, ::2], "rows::-1": d[::-1].copy()[::-1],
            "rev": d[::-1], "revcols": d[:, ::-1], "T": np.ascontiguousarray(d.T).T,
            "Fslice": np.asfortranarray(np.repeat(d, 2, axis=0))[::2]}


def test_dense_layouts(sp):
    rng = np.random.default_rng(9)
    a = special_matrix(sp, rng, 23, 31, 8)
    ac = a.to_other_storage()
    d = special_dense(rng, 23, 31)
    bcast_row = np.broadcast_to(d[0], (23, 31))           # strides (0, 8): Axis(0) fastest
    bcast_col = np.broadcast_to(d[:, :1], (23, 31))       # strides (8, 0): Axis(1) fastest
    for name, v in dict(views(d), bcast_row=bcast_row, bcast_col=bcast_col).items():
        lay = sp.sparse.fastest_axis(v)
        order = "C" if lay == 1 else "F"
        m = a if lay == 1 else ac
        got = sp.binop.add_dense_mat_same_ordering(m, v, 0.5, -2.0)
        assert got.flags["C_CONTIGUOUS" if lay == 1 else "F_CONTIGUOUS"], name
        assert DO.same_values(got, oracle_binop(m, DO.ADD, 0.5, -2.0, v, order)), name
        assert DO.same_values(a + v, oracle_binop(m, DO.ADD, 1.0, 1.0, v, order)), name  # both branches
        assert DO.same_values(ac + v, oracle_binop(m, DO.ADD, 1.0, 1.0, v, order)), name
        for f, fo in ((sp.CsMat.csr_from_dense, DO.csr_from_dense),
                      (sp.CsMat.csc_from_dense, DO.csc_from_dense)):
            assert_from_dense(f(v, 0.1), fo(v, 0.1))
    # rhs and out in the other layout: "Storage mismatch"; the shapes are checked first
    with pytest.raises(sp.SprsPanic, match="Storage mismatch"):
        sp.binop.add_dense_mat_same_ordering(a, np.asfortranarray(d), 1.0, 1.0)
    with pytest.raises(sp.SprsPanic, match="Storage mismatch"):
        sp.binop.csmat_binop_dense_raw_add(a, d, 1.0, 1.0, np.zeros(d.shape, order="F"))
    with pytest.raises(sp.SprsPanic, match="Dimension mismatch"):
        sp.binop.csmat_binop_dense_raw_add(a, np.asfortranarray(d[:, :5]), 1.0, 1.0, np.zeros((23, 5), order="F"))
    with pytest.raises(sp.SprsPanic, match="Dimension mismatch"):
        sp.binop.csmat_binop_dense_raw_mul(a, d, 1.0, np.zeros((23, 30)))
    with pytest.raises(sp.SprsPanic, match="Dimension mismatch"):
        sp.assign_to_dense(np.zeros((31, 23)), a)
    with pytest.raises(sp.SprsPanic, match="Dimension mismatch"):
        a + d.T
    # the C ABI: dimension, then storage, then the op (the reference has no dense subtraction)
    import ctypes as C
    ctx = a.context()
    lib = ctx.lib
    out = np.zeros((23, 31))
    p = lambda x: x.ctypes.data_as(C.c_void_p)  # noqa
    call = lambda op, r, c, rs, cs: lib.sprs_b200_csmat_binop_dense(  # noqa
        ctx.h, a.device().h, op, 1.0, 1.0, p(d), r, c, rs, cs, p(out), 23, 31, 31, 1)
    assert call(sp._lib.BINOP_SUB, 23, 30, 1, 23) == sp._lib.ERR_DIMENSION
    assert call(sp._lib.BINOP_SUB, 23, 31, 1, 23) == sp._lib.ERR_STORAGE
    assert call(sp._lib.BINOP_SUB, 23, 31, 31, 1) == sp._lib.ERR_ARGUMENT
    assert call(7, 23, 31, 31, 1) == sp._lib.ERR_ARGUMENT
    assert lib.sprs_b200_csmat_to_dense(ctx.h, a.device().h, p(out), 30) == sp._lib.ERR_DIMENSION


@pytest.mark.parametrize("shape", [(0, 5), (5, 0), (0, 0), (1, 7), (7, 1), (1, 1)])
def test_dense_edge_shapes(sp, shape):
    """Empty arrays take ndarray's all-zero strides (Axis(1) fastest, C order) in both layouts;
    length-1 axes keep numpy's strides."""
    rows, cols = shape
    rng = np.random.default_rng(rows * 10 + cols)
    d = special_dense(rng, rows, cols, frac=0.5) if rows * cols else np.zeros(shape)
    a = sp.CsMat.csr_from_dense(d, 0.0)
    assert_from_dense(a, DO.csr_from_dense(d, 0.0))
    assert_from_dense(sp.CsMat.csc_from_dense(d, 0.0), DO.csc_from_dense(d, 0.0))
    assert DO.same_bits(a.to_dense(), DO.to_dense(a)) and a.to_dense().shape == shape
    ac = a.to_other_storage()
    assert DO.same_bits(ac.to_dense(), DO.to_dense(ac))
    for v in (d, np.asfortranarray(d)):
        got = a + v
        m = a if sp.sparse.fastest_axis(v) == 1 else ac
        assert DO.same_values(got, oracle_binop(m, DO.ADD, 1.0, 1.0, v, "C" if m is a else "F"))
    if rows * cols == 0:
        assert sp.sparse.fastest_axis(np.asfortranarray(d)) == 1
        with pytest.raises(sp.SprsPanic, match="Storage mismatch"):
            sp.binop.add_dense_mat_same_ordering(ac, np.asfortranarray(d), 1.0, 1.0)
        assert sp.binop.add_dense_mat_same_ordering(a, np.asfortranarray(d), 1.0, 1.0).shape == shape


# ---- 5. the tile seams of the kernels
def seam_matrix(sp, rng):
    """A 48 x 1024 CSR matrix (4 rows per DENSE_TILE) whose stored entries sit on every seam
    of the merge: rows ending at tile edges, tiles of empty rows only, full rows (window reloads
    inside a 32-position chunk), entries in the first and last slot of tiles, long rows."""
    rows, cols = 48, 1024
    dense = np.zeros((rows, cols))
    mask = np.zeros((rows, cols), bool)
    mask[0] = True                                         # a full row
    mask[1, ::3] = True
    mask[2, [0, 31, 32, 63, 1023]] = True
    mask[3, -1] = True                                     # the last slot of tile 0
    mask[4, 0] = True                                      # the first slot of tile 1
    # rows 8..15: two tiles of empty rows only
    for r in range(16, 40):
        mask[r, rng.choice(cols, int(rng.integers(0, 200)), replace=False)] = True
    mask[40:44] = True                                     # a whole tile of full rows
    mask[47, [0, 1023]] = True
    dense[mask] = rng.standard_normal(int(mask.sum()))
    kept = SPECIALS[~np.isnan(SPECIALS) & (SPECIALS != 0)]   # values from_dense keeps
    spec = mask & (rng.random(mask.shape) < 0.1)
    dense[spec] = rng.choice(kept, int(spec.sum()))
    return dense, mask


def test_dense_seams(sp):
    rng = np.random.default_rng(123)
    dense, mask = seam_matrix(sp, rng)
    rows, cols = dense.shape
    T = sp.DENSE_TILE
    pos = (np.arange(rows)[:, None] * cols + np.arange(cols)[None, :])[mask]
    row_end = (np.arange(1, rows + 1) * cols)
    seams = {
        "row ends at a tile edge": np.any(row_end % T == 0),
        "tile of empty rows only": any(not mask[r:r + T // cols].any() for r in range(0, rows, T // cols)),
        "entry in a tile's first slot": np.any((pos % T == 0) & (pos > 0)),
        "entry in a tile's last slot": np.any(pos % T == T - 1),
        "full row": mask.all(axis=1).any(),
        "window of 32 inside a chunk": np.any(mask.reshape(rows, -1, 32).all(axis=2)),
    }
    assert all(seams.values()), seams
    for storage, f, fo in (("CSR", sp.CsMat.csr_from_dense, DO.csr_from_dense),
                           ("CSC", sp.CsMat.csc_from_dense, DO.csc_from_dense)):
        a = f(dense, 0.0)
        assert_from_dense(a, fo(dense, 0.0))
        assert DO.same_bits(a.to_dense(), dense) and DO.same_bits(DO.to_dense(a), dense)
        d = special_dense(rng, rows, cols)
        d = d if storage == "CSR" else np.asfortranarray(d)
        order = "C" if storage == "CSR" else "F"
        assert DO.same_values(sp.binop.add_dense_mat_same_ordering(a, d, -1.5, 2.0),
                              oracle_binop(a, DO.ADD, -1.5, 2.0, d, order))
        assert DO.same_values(sp.binop.mul_dense_mat_same_ordering(a, d, 3.0),
                              oracle_binop(a, DO.MUL, 3.0, 0.0, d, order))


def test_dense_assign_untouched(sp):
    """assign_to_dense leaves a sentinel prefill wherever no entry exists (the scatter touches
    the stored positions only), across SCATTER_TILE seams and runs of empty rows."""
    rng = np.random.default_rng(77)
    dense, mask = seam_matrix(sp, rng)
    sentinel = np.array([0x7FF4000000000DEF], np.uint64).view(np.float64)[0]
    for a in (sp.CsMat.csr_from_dense(dense, 0.0), sp.CsMat.csc_from_dense(dense, 0.0)):
        assert a.nnz() > 3 * sp.SCATTER_TILE
        for out in (np.full(dense.shape, sentinel), np.full(dense.shape, sentinel, order="F"),
                    np.full((dense.shape[0], 2 * dense.shape[1]), sentinel)[:, ::2],
                    np.full(dense.shape, sentinel)[::-1, ::-1][::-1, ::-1],
                    np.full(dense.shape[::-1], sentinel).T[::-1][::-1]):
            sp.assign_to_dense(out, a)
            assert DO.same_bits(out[mask], dense[mask])
            assert (out[~mask].view(np.uint64) == 0x7FF4000000000DEF).all()


# ---- 6. the device forms on torch tensors
def test_dense_dev_forms(sp):
    import torch
    from sprs_b200 import generate as G
    rng = np.random.default_rng(31)
    a = special_matrix(sp, rng, 40, 70, 15)
    ac = a.to_other_storage()
    ctx = a.context()
    dev = G._device(ctx)
    want = DO.to_dense(a)
    for m in (a, ac):
        t = G.to_dense(ctx, m.device())
        G._sync()
        assert DO.same_bits(t.cpu().numpy(), want)
        wide = torch.full((40, 80), 3.0, dtype=torch.float64, device=dev)
        G.to_dense(ctx, m.device(), out=wide[:, 5:75])
        G._sync()
        w = wide.cpu().numpy()
        assert DO.same_bits(w[:, 5:75], want) and (w[:, :5] == 3.0).all() and (w[:, 75:] == 3.0).all()
        s = torch.full((70, 40), 9.0, dtype=torch.float64, device=dev).t()   # F-order view
        G.assign_to_dense(ctx, s, m.device())
        G._sync()
        ref = np.full((40, 70), 9.0)
        DO.assign_to_dense(ref, m)
        assert DO.same_bits(s.cpu().numpy(), ref)
    d = special_dense(rng, 40, 70)
    for m, dt, order in ((a, torch.from_numpy(d).to(dev), "C"),
                         (ac, torch.from_numpy(np.ascontiguousarray(d.T)).to(dev).t(), "F")):
        for op, code in (("add", DO.ADD), ("mul", DO.MUL)):
            got = G.binop_dense(ctx, m.device(), dt, op, 0.5, -3.0)
            G._sync()
            assert DO.same_values(got.cpu().numpy(), oracle_binop(m, code, 0.5, -3.0, d, order))
            assert (got.stride(1) == 1) == (order == "C")
        # in place: out is rhs (D <- alpha*A + beta*D)
        inplace = dt.clone()
        r = G.binop_dense(ctx, m.device(), inplace, "add", 2.0, 0.5, out=inplace)
        G._sync()
        assert r.data_ptr() == inplace.data_ptr()
        assert DO.same_values(inplace.cpu().numpy(), oracle_binop(m, DO.ADD, 2.0, 0.5, d, order))
    if dev.type != "cuda":
        return  # the zero-copy views of a result mirror need CUDA memory (the emulator has none)
    for storage in ("CSR", "CSC"):
        mirror, ip, ind, dat = G.from_dense(ctx, torch.from_numpy(d).to(dev), 0.25, storage)
        want = (DO.csr_from_dense if storage == "CSR" else DO.csc_from_dense)(d, 0.25)
        assert np.array_equal(ip.cpu().numpy().astype(np.int64).astype(np.uint64), want[0])
        assert np.array_equal(ind.cpu().numpy().view(np.uint32).astype(np.uint64), want[1])
        assert DO.same_bits(dat.cpu().numpy(), want[2]) and mirror.storage == storage


# ---- 7. index widths, round trips and composition
@pytest.mark.parametrize("idx", [np.uint32, np.uint64])
def test_dense_widths_round_trip(sp, idx):
    rng = np.random.default_rng(41)
    ip, ind, d = rand_csr(rng, 60, 90, 20)
    a = sp.CsMat.new((60, 90), ip.astype(idx), ind.astype(idx), d)   # no explicit zeros, no NaN
    b = sp.CsMat.csr_from_dense(a.to_dense(), 0.0, idx)
    assert b == a and b.indptr.dtype == idx and b.indices.dtype == idx
    c = sp.CsMat.csc_from_dense(a.to_dense(), 0.0, idx)
    assert c == a.to_other_storage() and c.to_other_storage() == a
    # from_dense results feed SpMV, the sparse binops and SpGEMM; a SpGEMM result densifies
    x = rng.integers(-4, 5, 90).astype(float)
    assert np.array_equal(b * x, a * x)
    if hasattr(a.context().lib, "sprs_b200_csmat_binop"):  # the main emulated build has no binops
        assert b + b == a + a
    p = b * b.transpose_view().to_other_storage()
    q = a * a.transpose_view().to_other_storage()
    assert DO.same_bits(p.to_dense(), DO.to_dense(q))


_WIDTH_CHILD = r"""
import sys, json, numpy as np
sys.path.insert(0, %(root)r); sys.path.insert(0, %(tests)r)
import sprs_b200 as sp, dense_oracle as DO
from sprs_b200 import generate as G
from test_gpu_dense import seam_matrix
import torch
rng = np.random.default_rng(8)
dense, mask = seam_matrix(sp, rng)
errs = []
ctx = sp.Context.default()
for st, fo in (("CSR", DO.csr_from_dense), ("CSC", DO.csc_from_dense)):
    m, ip, ind, d = G.from_dense(ctx, torch.from_numpy(dense).to(G._device(ctx)), 0.0, st)
    if ip.dtype != torch.int64: errs.append(st + ": indptr is not 64-bit")
    w = fo(dense, 0.0)
    if not (np.array_equal(ip.cpu().numpy().astype(np.uint64), w[0]) and
            np.array_equal(ind.cpu().numpy().view(np.uint32).astype(np.uint64), w[1]) and
            DO.same_bits(d.cpu().numpy(), w[2])): errs.append(st + ": result differs")
    a = (sp.CsMat.csr_from_dense if st == "CSR" else sp.CsMat.csc_from_dense)(dense, 0.0)
    if not DO.same_bits(a.to_dense(), dense): errs.append(st + ": to_dense differs")
    d2 = np.asarray(rng.standard_normal(dense.shape), order="C" if st == "CSR" else "F")
    want = np.zeros(dense.shape, order="C" if st == "CSR" else "F")
    DO.binop_dense(a, DO.ADD, 1.0, 1.0, d2, want)
    if not DO.same_values(a + d2, want): errs.append(st + ": add differs")
print(json.dumps(errs))
"""


def test_dense_indptr64_child_process(tmp_path):
    """SPRS_B200_FORCE_INDPTR64=1: from_dense results and uploaded operands have 64-bit indptr."""
    script = tmp_path / "child.py"
    script.write_text(_WIDTH_CHILD % {"root": ROOT, "tests": os.path.join(ROOT, "tests")})
    r = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, SPRS_B200_FORCE_INDPTR64="1"))
    assert r.returncode == 0, r.stdout + r.stderr
    assert json.loads(r.stdout.strip().splitlines()[-1]) == []


# ---- 8. full size (H100): 32768 x 32768, compared on the device against torch models
N_FULL = 32768


def _full_a(sp):
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    return ctx, G.rand_csr(ctx, N_FULL, N_FULL, 32, seed=0x5EED0D01)


def _model_dense(a):
    """to_dense(A) by index_put: +0.0, then every stored value at (row, col)"""
    import torch
    n = a.rows
    ip = a.indptr.long()
    rows = torch.repeat_interleave(torch.arange(n, device=ip.device), ip[1:] - ip[:-1])
    x = torch.zeros((n, a.cols), dtype=torch.float64, device=ip.device)
    x[rows, a.indices.long()] = a.data
    return x


def _bits_equal(x, y):
    import torch
    return torch.equal(x.contiguous().view(torch.int64), y.contiguous().view(torch.int64))


def test_dense_to_dense_full_size(sp):
    import torch
    from sprs_b200 import generate as G
    ctx, a = _full_a(sp)
    got = G.to_dense(ctx, a)
    want = _model_dense(a)
    torch.cuda.synchronize()
    assert _bits_equal(got, want)
    del got
    csc = a.mirror.to_other_storage()
    got = G.to_dense(ctx, csc)
    torch.cuda.synchronize()
    assert _bits_equal(got, want)


@pytest.mark.parametrize("density", [0.001, 0.5])
def test_dense_from_dense_full_size(sp, density):
    import torch
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    g = torch.Generator(device="cuda").manual_seed(7)
    d = torch.randn((N_FULL, N_FULL), dtype=torch.float64, device="cuda", generator=g)
    d[torch.rand((N_FULL, N_FULL), device="cuda", generator=g) >= density] = 0.0
    eps = 1e-3
    for storage in ("CSR", "CSC") if density < 0.01 else ("CSR",):
        view = d if storage == "CSR" else d.t()       # CSC of d^T has d's rows as its columns
        m, ip, ind, dat = G.from_dense(ctx, view, eps, storage)
        keep = d.abs() > eps                          # outer-major = rows of d in both cases
        counts = keep.sum(dim=1)
        nz = keep.nonzero()
        assert ip.shape[0] == N_FULL + 1 and int(ip[-1]) == nz.shape[0]
        assert torch.equal(ip[1:].long(), counts.cumsum(0))
        assert torch.equal(ind.long(), nz[:, 1])
        assert _bits_equal(dat, d[keep])
        del m, ip, ind, dat, nz, keep


@pytest.mark.parametrize("layout", ["C", "F"])
def test_dense_add_mul_full_size(sp, layout):
    import torch
    from sprs_b200 import generate as G
    ctx, a = _full_a(sp)
    x = _model_dense(a)
    g = torch.Generator(device="cuda").manual_seed(11)
    d = torch.randn((N_FULL, N_FULL), dtype=torch.float64, device="cuda", generator=g)
    if layout == "F":
        d = d.t()                                     # Axis(0) fastest: `&A + &D` converts A
        lhs = a.mirror.to_other_storage()
    else:
        lhs = a
    cases = (("add", 1.0, 1.0), ("mul", -0.5, 0.0)) if layout == "C" else (("add", 1.0, 1.0),)
    for op, alpha, beta in cases:
        out = G.binop_dense(ctx, lhs, d, op, alpha, beta)
        torch.cuda.synchronize()
        assert (out.stride(1) == 1) == (layout == "C")
        step = 4096
        for r0 in range(0, N_FULL, step):
            xs, ds = x[r0:r0 + step], d[r0:r0 + step]
            want = (xs * alpha) + (ds * beta) if op == "add" else (xs * alpha) * ds
            assert _bits_equal(out[r0:r0 + step], want), (op, r0)
        del out


def test_dense_long_rows_full_size(sp):
    """One row of 10^6 columns and 10^5 rows of 3 columns: the tiles cut rows evenly either way."""
    rng = np.random.default_rng(3)
    for rows, cols in ((1, 1_000_000), (100_000, 3)):
        d = rng.standard_normal((rows, cols))
        d[rng.random((rows, cols)) < 0.5] = 0.0
        a = sp.CsMat.csr_from_dense(d, 0.0)
        assert_from_dense(a, DO.csr_from_dense(d, 0.0))
        assert DO.same_bits(a.to_dense(), d)
        e = rng.standard_normal((rows, cols))
        assert DO.same_values(a + e, oracle_binop(a, DO.ADD, 1.0, 1.0, e, "C"))


# ---- 9. the C++ host mirror
def test_cpp_dense_kats(tmp_path):
    exe = str(tmp_path / "test_dense_kats")
    lib_dir = os.path.join(ROOT, "sprs_b200")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-Wall", "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "test_dense_kats.cpp"),
                           "-L" + lib_dir, "-lsprs_b200", "-Wl,-rpath," + lib_dir])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("OK ")
