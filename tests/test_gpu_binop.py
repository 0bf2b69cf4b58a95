"""Sparse addition, subtraction, Hadamard product and scalar scale on the device (csrc/binop.cu)
against the CPU restatement of csmat_binop_same_storage_raw / CsMatBase::map
(tests/binop_oracle.cpp): structure exact and every value bit for bit (NaN by class).

Small tests run on the emulator as well (tests/test_emu_binop.py runs them on the emulated build
that has the binops, tests/emu_binop.py); `*_full_size`, `*_child_process` and `test_cpp*` ones
need the H100."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import binop_oracle as BO
from conftest import ROOT

pytestmark = pytest.mark.gpu

if os.environ.get("SPRS_B200_EMU_BINOP_LIB"):  # test infrastructure: the emulated build with
    import sprs_b200 as _sp                    # the binops (tests/emu_binop.py)
    _sp._lib.LIB_PATH = os.environ["SPRS_B200_EMU_BINOP_LIB"]


@pytest.fixture(scope="module")
def sp():
    import sprs_b200
    lib = sprs_b200._lib.load()  # the product library must export the binops (AttributeError)
    if os.path.basename(sprs_b200._lib.LIB_PATH).startswith("libsprs_b200_emu") and \
            not hasattr(lib, "sprs_b200_csmat_binop"):
        pytest.skip("the emulated build of tests/emu has no binops: tests/test_emu_binop.py "
                    "runs this file on one that has")
    return sprs_b200


@pytest.fixture(scope="module")
def kats():
    with open(os.path.join(ROOT, "tests", "golden", "sprs_fixtures.json")) as f:
        base = json.load(f)
    with open(os.path.join(ROOT, "tests", "golden", "binop_fixtures.json")) as f:
        return dict(base, **json.load(f))


def csmat(sp, m, idx=np.uint64, ptr=None):
    ptr = ptr or idx
    cls = sp.CsMat.new if m["storage"] == "CSR" else sp.CsMat.new_csc
    return cls(tuple(m["shape"]), np.array(m["indptr"], ptr), np.array(m["indices"], idx),
               np.array(m["data"], np.float64))


def arrays(m):
    return m.indptr, m.indices, m.data


def check(got, want):
    err = BO.first_difference(got, want)
    assert err is None, err


def oracle(op, a, b):
    """oracle result of a op b (CsMat operands of one storage) as u64/u32 arrays"""
    cast = lambda m: (m.indptr.astype(np.uint64), m.indices.astype(np.uint32), m.data)  # noqa
    return BO.binop(op, cast(a), cast(b))


# ---- 1. the reference's KATs through the Python mirror
@pytest.mark.parametrize("idx", [np.uint32, np.uint64])
def test_binop_kats(sp, kats, idx):
    a, b = csmat(sp, kats["mat1"], idx), csmat(sp, kats["mat2"], idx)
    for got, key in ((a + b, "mat1_plus_mat2"), (a - b, "mat1_minus_mat2"),
                     (sp.binop.mul_mat_same_storage(a, b), "mat1_times_mat2"),
                     (a * 2.0, "mat1_times_2")):
        assert got == csmat(sp, kats[key], idx), key
        assert got.indices.dtype == idx and got.indptr.dtype == idx and got.is_csr()
    c = csmat(sp, kats["add1_lhs"], idx) + csmat(sp, kats["add1_rhs"], idx)
    assert c == csmat(sp, kats["add1_sum"], idx)


def test_binop_mixed_storage(sp, kats):
    """Add / Sub convert rhs to lhs's storage (binop.rs:20-112): the result is in lhs storage."""
    a, b = csmat(sp, kats["mat1"]), csmat(sp, kats["mat2"])
    ac, bc = a.to_other_storage(), b.to_other_storage()
    want_sum, want_diff = csmat(sp, kats["mat1_plus_mat2"]), csmat(sp, kats["mat1_minus_mat2"])
    assert a + bc == want_sum and a - bc == want_diff                      # CSR + CSC -> CSR
    got = ac + b                                                            # CSC + CSR -> CSC
    assert got.is_csc() and got.to_other_storage() == want_sum
    got = ac - bc                                                           # CSC - CSC -> CSC
    assert got.is_csc() and got.to_other_storage() == want_diff
    got = sp.binop.mul_mat_same_storage(ac, bc)
    assert got.is_csc() and got.to_other_storage() == csmat(sp, kats["mat1_times_mat2"])
    assert (ac * 2.0).to_other_storage() == csmat(sp, kats["mat1_times_2"])


def test_binop_panics(sp, kats):
    a = csmat(sp, kats["mat1"])
    wrong_shape_csc = csmat(sp, kats["mat5"]).to_other_storage()     # 5 x 15, CSC
    for f in (lambda: a + wrong_shape_csc, lambda: a - wrong_shape_csc,
              lambda: sp.binop.mul_mat_same_storage(a, wrong_shape_csc)):
        with pytest.raises(sp.SprsPanic, match="Dimension mismatch"):  # shape before storage
            f()
    with pytest.raises(sp.SprsPanic, match="Storage mismatch"):
        sp.binop.mul_mat_same_storage(a, csmat(sp, kats["mat2"]).to_other_storage())
    # the C ABI: shape first, then storage, then the op code
    ctx = a.context()
    out = C.c_void_p()
    st = ctx.lib.sprs_b200_csmat_binop(ctx.h, a.device().h, wrong_shape_csc.device().h, 0, C.byref(out))
    assert st == sp._lib.ERR_DIMENSION
    bc = csmat(sp, kats["mat2"]).to_other_storage()
    assert ctx.lib.sprs_b200_csmat_binop(ctx.h, a.device().h, bc.device().h, 0, C.byref(out)) == \
        sp._lib.ERR_STORAGE
    assert ctx.lib.sprs_b200_csmat_binop(ctx.h, a.device().h, a.device().h, 3, C.byref(out)) == \
        sp._lib.ERR_ARGUMENT
    assert a.__mul__("2") is NotImplemented and not hasattr(a, "__rmul__")


# ---- 2. the seam matrix: every kind of cut the partition can make
def seam_matrix(rng):
    """rows (A lengths, B lengths, overlap pattern) built so that the tile and lane cuts of
    csrc/binop.cu fall on each seam; test_binop_seams asserts that they do."""
    rows = []  # (cols of A, cols of B, vals of A, vals of B)

    def row(ca, cb, va=None, vb=None):
        ca, cb = np.asarray(ca, np.int64), np.asarray(cb, np.int64)
        va = rng.integers(-4, 5, ca.size).astype(float) if va is None else np.asarray(va, float)
        vb = rng.integers(-4, 5, cb.size).astype(float) if vb is None else np.asarray(vb, float)
        rows.append((ca, cb, va, vb))
    cols = 8192
    # a row spanning >= 3 tiles, A and B interleaved with overlaps (equal pairs on many cuts)
    ca = np.arange(0, 6000, 2)
    cb = np.concatenate([np.arange(1, 3000, 2), np.arange(3000, 6000, 4)])
    row(ca, cb)
    for _ in range(200):                     # more empty rows than one tile holds (64)
        row([], [])
    for n in (40, 3, 100, 17):               # rows where only A / only B has entries
        row(np.sort(rng.choice(cols, n, replace=False)), [])
        row([], np.sort(rng.choice(cols, n, replace=False)))
    for n in (5, 33, 70):                    # rows that cancel to empty under SUB
        c = np.sort(rng.choice(cols, n, replace=False))
        v = rng.integers(1, 9, n).astype(float)
        row(c, c, v, v)
    for k in range(120):                     # equal-pattern rows of many lengths: equal pairs
        n = int(rng.integers(1, 60))         # on lane cuts (the snap)
        c = np.sort(rng.choice(cols, n, replace=False))
        row(c, c if k % 2 else np.sort(rng.choice(cols, n, replace=False)))
    for _ in range(60):
        row(np.sort(rng.choice(cols, int(rng.integers(0, 50)), replace=False)),
            np.sort(rng.choice(cols, int(rng.integers(0, 50)), replace=False)))
    # pad so that the final row ends a tile exactly: total cost a multiple of the tile
    def total():
        return sum(len(r[0]) + len(r[1]) for r in rows) + 16 * len(rows)
    pad = (-(total() + 16)) % 1024
    row(np.arange(pad // 2), np.arange(pad - pad // 2) + 4096)
    assert total() % 1024 == 0

    def build(which):
        lens = [len(r[which]) for r in rows]
        ip = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint32)
        ind = np.concatenate([r[which] for r in rows]).astype(np.uint32)
        d = np.concatenate([r[2 + which] for r in rows])
        return ip, ind, d
    return len(rows), cols, build(0), build(1)


def test_binop_seams(sp):
    rng = np.random.default_rng(2024)
    rows, cols, a, b = seam_matrix(rng)
    d, r, ka, kb, snapped = sp.binop_tiles(a[:2], b[:2])
    tile = d % sp.BINOP_TILE == 0
    ipa, ipb = a[0].astype(np.int64), b[0].astype(np.int64)
    inside = (r < rows) & (ka + kb > ipa[np.minimum(r, rows - 1)] + ipb[np.minimum(r, rows - 1)])
    inside &= (ka < ipa[np.minimum(r + 1, rows)]) | (kb < ipb[np.minimum(r + 1, rows)])
    ia, ib = a[1].astype(np.int64), b[1].astype(np.int64)
    big = 1 << 40  # the next entry of each list after the cut (big: the row's list is done)
    nxt_a = np.where(ka < ipa[np.minimum(r + 1, rows)], ia[np.minimum(ka, ia.size - 1)], big)
    nxt_b = np.where(kb < ipb[np.minimum(r + 1, rows)], ib[np.minimum(kb, ib.size - 1)], big)
    seams = {
        "snap on an equal pair": snapped.any(),
        "snap on a tile cut": (snapped & tile).any(),
        "cut before an A entry": (inside & (nxt_a < nxt_b)).any(),
        "cut before a B entry": (inside & (nxt_b < nxt_a)).any(),
        "cut before an equal pair": (inside & (nxt_a == nxt_b) & (nxt_a < big)).any(),
        "row over >= 3 tiles": np.count_nonzero(tile & (r == 0) & inside) >= 2,
        "tile of empty rows only": np.any(np.diff(r[tile]) >= 64),
        "last row ends a tile": d[-1] % sp.BINOP_TILE == 0,
    }
    assert all(seams.values()), seams
    A, B = sp.CsMat.new((rows, cols), *a), sp.CsMat.new((rows, cols), *b)
    for op, got in ((BO.ADD, A + B), (BO.SUB, A - B), (BO.MUL, sp.binop.mul_mat_same_storage(A, B))):
        check(arrays(got), oracle(op, A, B))
    assert (A - A).nnz() == 0 and (A - A).indptr.tolist() == [0] * (rows + 1)
    check(arrays(A * -3.0), BO.scale(arrays(A), -3.0))


# ---- 3. value classes
def test_binop_value_classes(sp):
    """MUL Left(+-inf / NaN) is a * 0.0 = NaN and kept though B has no entry; SUB Right(b) is
    -b; ADD Left(-0.0) is +0.0 and dropped; explicit zeros disappear; A - A is all empty with the
    full indptr; a * 0.0 keeps every entry (map does not filter)."""
    specials = [np.inf, -np.inf, np.nan, 0.0, -0.0, 1e308, -1e308, 5e-324, 1.5]
    rng = np.random.default_rng(7)
    rows, cols = 40, 60
    lens = rng.integers(0, 20, rows)
    ip = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint32)
    ind = np.concatenate([np.sort(rng.choice(cols, n, replace=False)) for n in lens]).astype(np.uint32)
    da = rng.choice(specials, ind.size)
    lens_b = rng.integers(0, 20, rows)
    ipb = np.concatenate([[0], np.cumsum(lens_b)]).astype(np.uint32)
    indb = np.concatenate([np.sort(rng.choice(cols, n, replace=False)) for n in lens_b]).astype(np.uint32)
    db = rng.choice(specials, indb.size)
    A, B = sp.CsMat.new((rows, cols), ip, ind, da), sp.CsMat.new((rows, cols), ipb, indb, db)
    check(arrays(A + B), oracle(BO.ADD, A, B))
    check(arrays(A - B), oracle(BO.SUB, A, B))
    check(arrays(B + A), oracle(BO.ADD, B, A))
    check(arrays(sp.binop.mul_mat_same_storage(A, B)), oracle(BO.MUL, A, B))
    check(arrays(A - A), oracle(BO.SUB, A, A))
    z = A * 0.0
    assert z.nnz() == A.nnz()
    check(arrays(z), BO.scale(arrays(A), 0.0))
    # the literal cases on one row
    a = sp.CsMat.new((1, 8), np.array([0, 4], np.uint32), np.array([0, 1, 2, 3], np.uint32),
                     np.array([np.inf, np.nan, -0.0, 0.0]))
    b = sp.CsMat.new((1, 8), np.array([0, 2], np.uint32), np.array([4, 5], np.uint32),
                     np.array([2.0, -0.0]))
    m = sp.binop.mul_mat_same_storage(a, b)
    assert m.indices.tolist() == [0, 1] and np.isnan(m.data).all()
    s = a - b
    assert s.indices.tolist() == [0, 1, 4] and s.data[2] == -2.0
    assert (a + b).indices.tolist() == [0, 1, 4]
    e = sp.CsMat.new((3, 0), np.zeros(4, np.uint32), np.zeros(0, np.uint32), np.zeros(0))
    assert (e + e).indptr.tolist() == [0, 0, 0, 0]
    z0 = sp.CsMat.new((0, 5), np.zeros(1, np.uint32), np.zeros(0, np.uint32), np.zeros(0))
    assert (z0 - z0).indptr.tolist() == [0] and (z0 * 2.0).nnz() == 0


# ---- 4. index widths
@pytest.mark.parametrize("idx", [np.uint32, np.uint64])
def test_binop_host_widths(sp, idx):
    rng = np.random.default_rng(11)
    rows, cols, a, b = seam_matrix(rng)
    A = sp.CsMat.new((rows, cols), a[0].astype(idx), a[1].astype(idx), a[2])
    B = sp.CsMat.new((rows, cols), b[0].astype(idx), b[1].astype(idx), b[2])
    got = A - B
    assert got.indptr.dtype == idx and got.indices.dtype == idx
    check(arrays(got), oracle(BO.SUB, A, B))


_WIDTH_CHILD = r"""
import sys, json, numpy as np, torch
sys.path.insert(0, %(root)r); sys.path.insert(0, %(tests)r)
import sprs_b200 as sp, binop_oracle as BO
from sprs_b200 import generate as G
from test_gpu_binop import seam_matrix
rng = np.random.default_rng(5)
rows, cols, a, b = seam_matrix(rng)
A, B = sp.CsMat.new((rows, cols), *a), sp.CsMat.new((rows, cols), *b)
ctx = A.context()
errs = []
def cmp(name, views, want):
    m, ip, ind, d = views
    if ip.dtype != torch.int64: errs.append(name + ": output indptr is not 64-bit")
    e = BO.first_difference(BO._host(ip, ind, d, 0, rows), want)
    if e: errs.append(name + ": " + e)
cast = lambda t: (t[0].astype(np.uint64), t[1], t[2])
for name, op in (("add", BO.ADD), ("sub", BO.SUB), ("mul", BO.MUL)):
    cmp(name + " u64+u64", G.binop(ctx, A.device(), B.device(), name), BO.binop(op, cast(a), cast(b)))
# mixed widths: B adopted from device arrays keeps a 32-bit indptr
dev = G._device(ctx)
Bd = G.DeviceCsr(ctx, rows, cols, torch.from_numpy(b[0].view(np.int32)).to(dev),
                 torch.from_numpy(b[1].view(np.int32)).to(dev), torch.from_numpy(b[2]).to(dev))
cmp("u64-u32", G.binop(ctx, A.device(), Bd, "sub"), BO.binop(BO.SUB, cast(a), cast(b)))
cmp("u32+u64", G.binop(ctx, Bd, A.device(), "add"), BO.binop(BO.ADD, cast(b), cast(a)))
print(json.dumps(errs))
"""


def test_binop_indptr64_child_process(tmp_path):
    """SPRS_B200_FORCE_INDPTR64=1 (read once per process): uploaded operands have 64-bit indptr,
    results too; mixed widths with one operand adopted through from_device (32-bit)."""
    script = tmp_path / "child.py"
    script.write_text(_WIDTH_CHILD % {"root": ROOT, "tests": os.path.join(ROOT, "tests")})
    r = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, SPRS_B200_FORCE_INDPTR64="1"))
    assert r.returncode == 0, r.stdout + r.stderr
    assert json.loads(r.stdout.strip().splitlines()[-1]) == []


# ---- 5. composition with the other device operations
def test_binop_composition(sp):
    import torch
    from sprs_b200 import generate as G
    rng = np.random.default_rng(3)
    rows, cols, a, b = seam_matrix(rng)
    A, B = sp.CsMat.new((rows, cols), *a), sp.CsMat.new((rows, cols), *b)
    ctx = A.context()
    dev = G._device(ctx)
    x = torch.from_numpy(rng.integers(-8, 9, cols).astype(np.float64)).to(dev)
    for got, want in ((A + B, oracle(BO.ADD, A, B)), (A * 0.5, BO.scale(arrays(A), 0.5))):
        ref = sp.CsMat.new((rows, cols), *want)
        ys = []
        for m in (got, ref):
            y = torch.full((rows,), 7.0, dtype=torch.float64, device=dev)
            G.spmv(ctx, m.device(), x, y)
            G._sync()
            ys.append(y.cpu().numpy())
        assert np.array_equal(ys[0].view(np.uint64), ys[1].view(np.uint64))
        assert got.to_other_storage() == ref.to_other_storage()
    # SpGEMM takes a binop result: (A + B) (A + B)^T against the same product of the oracle's
    s = A + B
    ref = sp.CsMat.new((rows, cols), *oracle(BO.ADD, A, B))
    assert s * s.transpose_view().to_other_storage() == ref * ref.transpose_view().to_other_storage()


# ---- 6. full size (H100)
def _identity(ctx, n):
    import torch
    from sprs_b200 import generate as G
    dev = G._device(ctx)
    return G.DeviceCsr(ctx, n, n, torch.arange(n + 1, dtype=torch.int32, device=dev),
                       torch.arange(n, dtype=torch.int32, device=dev),
                       torch.ones(n, dtype=torch.float64, device=dev))


def _full(ctx, a, b, op, n):
    from sprs_b200 import generate as G
    res = G.binop(ctx, a, b, {BO.ADD: "add", BO.SUB: "sub", BO.MUL: "mul"}[op])
    err, _ = BO.compare_chunked(op, (a.indptr, a.indices, a.data), (b.indptr, b.indices, b.data),
                                res[1:], n)
    assert err is None, err
    return res


def test_binop_rand1m_add_full_size(sp):
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    n = 1_000_000
    a = G.rand_csr(ctx, n, n, 32, seed=0x5EED0002)
    b = G.rand_csr(ctx, n, n, 32, seed=0x5EED1002)
    _full(ctx, a, b, BO.ADD, n)
    _full(ctx, a, b, BO.MUL, n)


def test_binop_rmat500k_sym_full_size(sp):
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    n = 500_000
    a = G.rmat_csr(ctx, n, 16, seed=0x5EED0004)
    t, tip, tind, tdat = G._with_views(ctx, a.mirror.to_other_storage())  # CSC of A = CSR of A^T
    at = G.DeviceCsr(ctx, n, n, tip, tind, tdat)
    _full(ctx, a, at, BO.ADD, n)
    del t


def test_binop_rmat10m_shift_full_size(sp):
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    n = 10_000_000
    a = G.rmat_csr(ctx, n, 100, seed=0x5EED0005)
    c = _full(ctx, a, _identity(ctx, n), BO.SUB, n)
    del c
    s = G.scale(ctx, a, 2.0)
    err, _ = BO.compare_chunked(("scale", 2.0), (a.indptr, a.indices, a.data), None, s[1:], n)
    assert err is None, err


# ---- 7. the C++ host mirror
def test_cpp_binop_kats(tmp_path):
    exe = str(tmp_path / "test_binop_kats")
    lib_dir = os.path.join(ROOT, "sprs_b200")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-Wall", "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "test_binop_kats.cpp"),
                           "-L" + lib_dir, "-lsprs_b200", "-Wl,-rpath," + lib_dir])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("OK ")
