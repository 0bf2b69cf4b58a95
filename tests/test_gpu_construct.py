"""Sparse matrix construction on the device (csrc/construct.cu): bmat, vstack, hstack and
kronecker_product against the CPU restatement of the reference's composition
(tests/construct_oracle.cpp + .py): storage, shape and structure exact, stacked values bit for
bit (NaN payloads included), Kronecker values bit for bit with NaN compared by position.

Small tests run on the emulator as well (tests/test_emu_construct.py runs them on the emulated
build that has the construction kernels, tests/emu_construct.py); `*_full_size`,
`*_child_process` and `test_cpp*` ones need the H100."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import construct_oracle as CO
from conftest import ROOT, rand_csr

pytestmark = pytest.mark.gpu

if os.environ.get("SPRS_B200_EMU_CONSTRUCT_LIB"):  # test infrastructure: the emulated build with
    import sprs_b200 as _sp                        # the construction kernels
    _sp._lib.LIB_PATH = os.environ["SPRS_B200_EMU_CONSTRUCT_LIB"]

# output entries per warp tile of both fill kernels, read from the kernel source so that a
# retune moves the seams with it
TILE = int(re.search(r"constexpr uint64_t CONSTRUCT_TILE = (\d+);",
                     open(os.path.join(ROOT, "sprs_b200", "csrc", "construct.cu")).read()).group(1))


@pytest.fixture(scope="module")
def sp():
    import sprs_b200
    lib = sprs_b200._lib.load()  # the product library must export the construction
    if os.path.basename(sprs_b200._lib.LIB_PATH).startswith("libsprs_b200_emu") and \
            not hasattr(lib, "sprs_b200_csmat_bmat"):
        pytest.skip("the emulated build of tests/emu has no construction kernels: "
                    "tests/test_emu_construct.py runs this file on one that has")
    assert sprs_b200.CONSTRUCT_TILE == TILE
    return sprs_b200


@pytest.fixture(scope="module")
def kats():
    import json
    with open(os.path.join(ROOT, "tests", "golden", "sprs_fixtures.json")) as f:
        base = json.load(f)
    with open(os.path.join(ROOT, "tests", "golden", "construct_fixtures.json")) as f:
        return dict(base, **json.load(f))


def csmat(sp, m, idx=np.uint64, ptr=None):
    ptr = ptr or idx
    cls = sp.CsMat.new if m["storage"] == "CSR" else sp.CsMat.new_csc
    return cls(tuple(m["shape"]), np.array(m["indptr"], ptr), np.array(m["indices"], idx),
               np.array(m["data"], np.float64))


def check(got, want, kron=False):
    err = CO.first_difference(got, want, kron=kron)
    assert err is None, err


# values: ordinary normals plus the classes a copy or a multiply must keep
NAN_PAYLOADS = np.array([0x7FF8000000000123, 0xFFF80000DEADBEEF, 0x7FF0000000000001],
                        np.uint64).view(np.float64)
SPECIALS = np.concatenate([[-0.0, 0.0, np.inf, -np.inf, 5e-324, -1e-308], NAN_PAYLOADS])


def values(rng, n, special=0.1):
    v = rng.standard_normal(n) * np.exp2(rng.integers(-20, 21, n))
    hit = rng.random(n) < special
    v[hit] = rng.choice(SPECIALS, int(hit.sum()))
    return v


def rand_mat(sp, rng, storage, rows, cols, per_outer=3.0, idx=np.uint64, empty_frac=0.0,
             special=0.1):
    outer, inner = (rows, cols) if storage == "CSR" else (cols, rows)
    if outer == 0:
        ip, ind = np.zeros(1, np.int64), np.zeros(0, np.int64)
    elif inner == 0:
        ip, ind = np.zeros(outer + 1, np.int64), np.zeros(0, np.int64)
    else:
        ip, ind, _ = rand_csr(rng, outer, inner, per_outer, np.int64, empty_frac=empty_frac)
    dat = values(rng, int(ip[-1]), special)
    cls = sp.CsMat.new if storage == "CSR" else sp.CsMat.new_csc
    return cls((rows, cols), ip.astype(idx), ind.astype(idx), dat)


def row_lengths_mat(sp, rng, lens, cols, storage="CSR", idx=np.uint64):
    """a matrix whose outer vectors have exactly the given lengths"""
    lens = np.asarray(lens, np.int64)
    ip = np.concatenate([[0], np.cumsum(lens)])
    ind = np.concatenate([np.sort(rng.choice(cols, int(n), replace=False)) for n in lens] +
                         [np.zeros(0, np.int64)])
    shape = (len(lens), cols) if storage == "CSR" else (cols, len(lens))
    cls = sp.CsMat.new if storage == "CSR" else sp.CsMat.new_csc
    return cls(shape, ip.astype(idx), ind.astype(idx), values(rng, int(ip[-1])))


def O(m):  # noqa: E743 -- the oracle's view of a CsMat (or None)
    return None if m is None else CO.of(m)


# ---- 1. the reference's KATs through the Python mirror
@pytest.mark.parametrize("idx", [np.uint32, np.uint64])
def test_construct_kats(sp, kats, idx):
    a, b = csmat(sp, kats["mat1"], idx), csmat(sp, kats["mat2"], idx)
    want = csmat(sp, kats["mat1_vstack_mat2"], idx)
    got = sp.vstack([a, b])                                                  # vstack_trivial
    assert got == want and got.is_csr() and got.indices.dtype == idx
    got = sp.hstack([a.transpose_view(), b.transpose_view()])                # hstack_trivial
    assert got == want.transpose_view() and got.is_csc()
    assert sp.vstack([a.to_csc(), b]) == want                                # with conversion
    eye = lambda n: sp.CsMat.eye(n, index_dtype=idx)  # noqa
    assert sp.bmat([[eye(5), None], [None, eye(4)]]) == csmat(sp, kats["bmat_simple"], idx)
    d, e = csmat(sp, kats["mat3"], idx), csmat(sp, kats["mat4"], idx)
    assert sp.bmat([[a, b], [b, None]]) == csmat(sp, kats["bmat_complex_1"], idx)
    assert sp.bmat([[d, a], [None, e]]) == csmat(sp, kats["bmat_complex_2"], idx)
    ka, kb = csmat(sp, kats["kron_a"], idx), csmat(sp, kats["kron_b"], idx)
    want = np.zeros((6, 6))
    for i, j, v in kats["kron_entries"]:
        want[i, j] = v
    for sa in ("CSR", "CSC"):
        for sb in ("CSR", "CSC"):
            x = ka if sa == "CSR" else ka.to_csc()
            y = kb if sb == "CSR" else kb.to_csc()
            c = sp.kronecker_product(x, y)
            assert c.storage == sa and c.shape == (6, 6) and c.nnz() == 16
            assert np.array_equal(c.to_dense(), want)
            check(c, CO.kronecker_product(O(x), O(y)), kron=True)


def test_construct_panics(sp, kats):
    names = {k: csmat(sp, kats[k]) for k in ("mat1", "mat2", "mat3", "mat4")}
    for case in kats["panics"]:
        with pytest.raises(sp.SprsPanic, match=case["message"]):
            if "stack" in case:
                sp.vstack([names[k] for k in case["stack"]])
            else:
                sp.bmat([[names[k] if k else None for k in row] for row in case["blocks"]])
    with pytest.raises(sp.SprsPanic, match="Empty stacking list"):
        sp.hstack([])
    with pytest.raises(sp.SprsPanic, match="Dimension mismatch"):  # hstack: rows differ
        sp.hstack([names["mat1"], names["mat3"].transpose_view()])
    with pytest.raises(sp.SprsPanic, match="Dimension mismatch"):  # bmat: heights in a row
        sp.bmat([[names["mat1"], names["mat3"].transpose_view()]])
    # the C ABI: codes in the reference's order
    a = names["mat1"]
    ctx = a.context()
    lib, out = ctx.lib, C.c_void_p()
    none = (C.c_void_p * 4)(None, None, None, None)
    assert lib.sprs_b200_csmat_bmat(ctx.h, 0, 2, none, C.byref(out)) == sp._lib.ERR_ARGUMENT
    assert lib.sprs_b200_csmat_bmat(ctx.h, 2, 0, none, C.byref(out)) == sp._lib.ERR_ARGUMENT
    grid = (C.c_void_p * 4)(None, None, a.device().h, names["mat3"].device().h)
    assert lib.sprs_b200_csmat_bmat(ctx.h, 2, 2, grid, C.byref(out)) == sp._lib.ERR_ARGUMENT
    assert b"Empty bmat row" in lib.sprs_b200_last_error(ctx.h)
    grid = (C.c_void_p * 2)(a.device().h, names["mat3"].device().h)
    assert lib.sprs_b200_csmat_bmat(ctx.h, 2, 1, grid, C.byref(out)) == sp._lib.ERR_DIMENSION
    assert not out.value


def test_construct_index_range(sp):
    # a result dimension >= 2^32: ERR_INDEX_RANGE even with u64 indices (documented difference)
    tall = sp.CsMat.new((70000, 1), np.zeros(70001, np.uint64), [], [])
    with pytest.raises(sp.SprsPanic, match="Index type is not large enough"):
        sp.kronecker_product(tall, tall)
    # a produced index that does not fit the index dtype: the reference's unwrap panic
    wide = lambda idx: sp.CsMat.new((1, 50000), np.array([0, 1], idx), np.array([49999], idx),  # noqa
                                    [2.0])
    with pytest.raises(sp.SprsPanic, match="Option::unwrap"):
        sp.kronecker_product(wide(np.int32), wide(np.int32))
    c = sp.kronecker_product(wide(np.uint32), wide(np.uint32))
    assert c.shape == (1, 2_500_000_000) and int(c.indices[0]) == 49999 * 50000 + 49999
    assert c.data[0] == 4.0


# ---- 2. every storage combination, both index dtypes
@pytest.mark.parametrize("idx", [np.uint32, np.uint64])
@pytest.mark.parametrize("k", [1, 2, 3, 4])
def test_stack_storage_combinations(sp, idx, k):
    rng = np.random.default_rng(100 + k)
    for combo in range(1 << k):
        st = ["CSC" if combo >> i & 1 else "CSR" for i in range(k)]
        rows = rng.integers(0, 40, k)
        v = [rand_mat(sp, rng, s, int(r), 23, 4.0, idx, empty_frac=0.2) for s, r in zip(st, rows)]
        got = sp.vstack(v)
        check(got, CO.vstack([O(m) for m in v]))
        assert got.is_csr() and got.indices.dtype == idx
        h = [rand_mat(sp, rng, s, 19, int(c), 4.0, idx, empty_frac=0.2) for s, c in zip(st, rows)]
        got = sp.hstack(h)
        check(got, CO.hstack([O(m) for m in h]))
        assert got.is_csc()
        # hstack(ms) == vstack([m.transpose_view() for m in ms]).transpose_view(), bit for bit
        check(got, CO.transpose_view(O(sp.vstack([m.transpose_view() for m in h]))))
        # a block row of k blocks with the same storage mix
        g = [rand_mat(sp, rng, s, 17, int(c) + 1, 3.0, idx) for s, c in zip(st, rows)]
        check(sp.bmat([g, g[::-1]]), CO.bmat([[O(m) for m in g], [O(m) for m in g[::-1]]]))


@pytest.mark.parametrize("idx", [np.uint32, np.uint64])
def test_kron_storage_combinations(sp, idx):
    rng = np.random.default_rng(7)
    for sa in ("CSR", "CSC"):
        for sb in ("CSR", "CSC"):
            for (ra, ca), (rb, cb) in (((13, 9), (7, 11)), ((1, 40), (40, 1)), ((0, 5), (3, 3)),
                                       ((6, 6), (0, 0)), ((30, 30), (5, 2))):
                a = rand_mat(sp, rng, sa, ra, ca, 3.0, idx, empty_frac=0.2)
                b = rand_mat(sp, rng, sb, rb, cb, 2.0, idx, empty_frac=0.2)
                c = sp.kronecker_product(a, b)
                assert c.storage == sa and c.shape == (ra * rb, ca * cb)
                check(c, CO.kronecker_product(O(a), O(b)), kron=True)


def test_bmat_mixed_indptr(sp):
    """Blocks adopted from device arrays (u32 indptr) beside uploaded ones; under
    SPRS_B200_FORCE_INDPTR64 (test_construct_indptr64_child_process) the uploaded blocks and the
    result have u64 indptr, so the widths are mixed across the grid."""
    from sprs_b200 import construct as K, generate as G
    import torch
    rng = np.random.default_rng(11)
    ctx = sp.Context.default()
    dev = G._device(ctx)
    # grid [[h0, None, h2], [h3, h1, None]]: every block 30 rows, h0 and h3 equally wide
    host = [rand_mat(sp, rng, "CSR", 30, c, 5.0, np.uint32) for c in (25, 20, 15, 25)]
    for m in host:
        m._ctx = ctx
    adopted = []
    for m in host[:2]:
        ip = torch.as_tensor(m.indptr.astype(np.uint32).view(np.int32), device=dev)
        ind = torch.as_tensor(m.indices.astype(np.uint32).view(np.int32), device=dev)
        dat = torch.as_tensor(m.data, device=dev)
        adopted.append(G.DeviceCsr(ctx, m.rows(), m.cols(), ip, ind, dat))
    widths = set()
    for mirror in [a.mirror for a in adopted] + [m.device() for m in host[2:]]:
        ipb = C.c_int()
        d = C.c_void_p()
        ctx.check(ctx.lib.sprs_b200_csmat_device_arrays(mirror.h, C.byref(d), C.byref(ipb),
                                                        C.byref(d), C.byref(d)))
        widths.add(ipb.value)
    if os.environ.get("SPRS_B200_FORCE_INDPTR64") == "1":
        assert widths == {4, 8}
    grid = [[adopted[0].mirror, None, host[2].device()], [host[3].device(), adopted[1].mirror, None]]
    res = K.bmat_dev(ctx, grid)
    got = CO.mat("CSR", (res.rows, res.cols), *res.download(np.uint64))
    check(got, CO.bmat([[O(host[0]), None, O(host[2])], [O(host[3]), O(host[1]), None]]))


# ---- 3. the seams of the output tiling
def test_stack_tile_seams(sp):
    rng = np.random.default_rng(21)
    T = TILE
    cols = 3 * T + 50
    for total in (T - 1, T, T + 1, 2 * T, 3 * T + 7):
        # outputs of exactly `total` entries, split over three blocks
        cut = sorted(rng.integers(0, total + 1, 2))
        parts = [cut[0], cut[1] - cut[0], total - cut[1]]
        blocks = [row_lengths_mat(sp, rng, [p], cols) for p in parts]
        check(sp.vstack(blocks), CO.vstack([O(m) for m in blocks]))
        check(sp.hstack([b.transpose_view() for b in blocks]),
              CO.hstack([CO.transpose_view(O(b)) for b in blocks]))
    # rows that start / end exactly on a tile boundary, and rows that straddle one
    for lens in ([T, T, 1, T - 1, 1, T], [T // 2, T // 2, T // 2 - 1, 2, T - 1, T + 1],
                 [1] * (T + 5) + [T + 3], [3 * T + 1]):
        a = row_lengths_mat(sp, rng, lens, cols)
        b = row_lengths_mat(sp, rng, lens[::-1], cols)
        check(sp.vstack([a, b]), CO.vstack([O(a), O(b)]))
        check(sp.bmat([[a, b.transpose_view().transpose_view()], [None, a]]),
              CO.bmat([[O(a), O(b)], [None, O(a)]]))
    # runs of empty rows across tile boundaries (more empty rows than a tile has entries)
    lens = [T - 3] + [0] * (2 * T + 1) + [5] + [0] * 7 + [T + 2] + [0] * (T + 9)
    a = row_lengths_mat(sp, rng, lens, cols)
    z = sp.CsMat.zero((3 * T, cols), index_dtype=np.uint64)
    check(sp.vstack([a, z, a]), CO.vstack([O(a), O(z), O(a)]))
    check(sp.bmat([[a, a], [z, None], [a, a]]), CO.bmat([[O(a), O(a)], [O(z), None],
                                                        [O(a), O(a)]]))


def test_kron_tile_seams(sp):
    rng = np.random.default_rng(22)
    T = TILE
    # b's vectors of 1, 3, 31, 32, 33 entries against a's so that (ia, ib) rows straddle tiles
    for lb in (1, 3, 31, 32, 33, 64):
        for la in (T // lb - 1, T // lb, T // lb + 1, 2 * T // lb + 3):
            la = max(la, 1)
            a = row_lengths_mat(sp, rng, [la, 0, la - 1 if la > 1 else 1, 2], la + 8)
            b = row_lengths_mat(sp, rng, [lb, 1, 0, lb], lb + 5)
            check(sp.kronecker_product(a, b), CO.kronecker_product(O(a), O(b)), kron=True)
    # outputs of exactly T - 1, T, T + 1 entries
    for total in (T - 1, T, T + 1):
        a = row_lengths_mat(sp, rng, [total], total + 1)
        b = row_lengths_mat(sp, rng, [1], 4)
        check(sp.kronecker_product(a, b), CO.kronecker_product(O(a), O(b)), kron=True)
        check(sp.kronecker_product(b, a), CO.kronecker_product(O(b), O(a)), kron=True)
    # runs of empty output rows across tile boundaries: an empty vector of a empties outer(b)
    # rows, an empty vector of b one row per vector of a
    a = row_lengths_mat(sp, rng, [5, 0, 0, 7, 0, 3], 12)
    b = row_lengths_mat(sp, rng, [T // 3] + [0] * (T + 1) + [T // 2, 0, 1], T)
    check(sp.kronecker_product(a, b), CO.kronecker_product(O(a), O(b)), kron=True)


def test_kron_long_row(sp):
    """One output row of more than 10^6 entries, split over hundreds of warps."""
    rng = np.random.default_rng(23)
    a = row_lengths_mat(sp, rng, [1000, 3], 1200)
    b = row_lengths_mat(sp, rng, [1001], 1001)
    c = sp.kronecker_product(a, b)
    assert int(c.indptr[1]) == 1_001_000
    check(c, CO.kronecker_product(O(a), O(b)), kron=True)


# ---- 4. edge shapes
def test_stack_edge_shapes(sp):
    rng = np.random.default_rng(31)
    e0 = sp.CsMat.new((0, 7), np.zeros(1, np.uint64), [], [])
    z = sp.CsMat.zero((4, 7), index_dtype=np.uint64)
    a = rand_mat(sp, rng, "CSR", 5, 7)
    for mats in ([e0], [e0, e0], [e0, a, e0], [z, a, z], [z], [a.to_csc(), e0, z]):
        check(sp.vstack(mats), CO.vstack([O(m) for m in mats]))
        t = [m.transpose_view() for m in mats]
        check(sp.hstack(t), CO.hstack([O(m) for m in t]))
    # None padding, 0-row block rows and 0-column block columns
    b = rand_mat(sp, rng, "CSC", 5, 3)
    e = sp.CsMat.new((0, 3), np.zeros(1, np.uint64), [], [])
    w = sp.CsMat.new((5, 0), np.zeros(6, np.uint64), [], [])
    for grid in ([[a, None], [None, b]], [[a, b], [None, e]], [[a, w, b]], [[e, None], [None, e]],
                 [[w]], [[None, a], [b, None], [e, None]]):
        check(sp.bmat(grid), CO.bmat([[O(m) for m in row] for row in grid]))
    # block rows of widths 3 + 7, 3 + 7 and 3 + 3: both panic
    grid = [[None, a], [b, None], [e, e]]
    with pytest.raises(sp.SprsPanic, match="Dimension mismatch"):
        sp.bmat(grid)
    with pytest.raises(CO.Panic, match="Dimension mismatch"):
        CO.bmat([[O(m) for m in row] for row in grid])
    # unequal widths: valid when the block rows' totals agree (B at column 3, D at column 5)
    A, B = rand_mat(sp, rng, "CSR", 2, 3), rand_mat(sp, rng, "CSC", 2, 5)
    Cm, D = rand_mat(sp, rng, "CSR", 2, 5), rand_mat(sp, rng, "CSR", 2, 3)
    got = sp.bmat([[A, B], [Cm, D]])
    assert got.shape == (4, 8)
    check(got, CO.bmat([[O(A), O(B)], [O(Cm), O(D)]]))
    with pytest.raises(sp.SprsPanic, match="Dimension mismatch"):
        sp.bmat([[A, None], [Cm, D]])  # widths 3 + 3 and 5 + 3
    with pytest.raises(CO.Panic, match="Dimension mismatch"):
        CO.bmat([[O(A), None], [O(Cm), O(D)]])


def test_bmat_64x64_grid(sp):
    rng = np.random.default_rng(32)
    heights = rng.integers(0, 6, 64)
    widths = rng.integers(0, 6, 64)
    grid = []
    for i in range(64):
        row = []
        for j in range(64):
            if rng.random() < 0.3 and i != j:
                row.append(None)
            else:
                row.append(rand_mat(sp, rng, "CSC" if (i + j) % 3 == 0 else "CSR",
                                    int(heights[i]), int(widths[j]), 2.0))
        grid.append(row)
    got = sp.bmat(grid)
    check(got, CO.bmat([[O(m) for m in row] for row in grid]))
    assert got.shape == (int(heights.sum()), int(widths.sum()))


# ---- 5. value classes
def test_value_classes(sp):
    rng = np.random.default_rng(41)
    a = rand_mat(sp, rng, "CSR", 60, 50, 8.0, special=0.5)
    b = rand_mat(sp, rng, "CSC", 60, 50, 8.0, special=0.5)
    check(sp.vstack([a, b, a]), CO.vstack([O(a), O(b), O(a)]))   # bit for bit, NaN payloads too
    check(sp.hstack([a, b]), CO.hstack([O(a), O(b)]))
    check(sp.kronecker_product(a, b.slice_outer(0, 4)), CO.kronecker_product(O(a), O(b.slice_outer(0, 4))),
          kron=True)
    # products that underflow to 0.0 / -0.0 and explicit zeros stay in the structure
    t = sp.CsMat.new((2, 3), np.array([0, 3, 5], np.uint64), np.array([0, 1, 2, 0, 2], np.uint64),
                     [1e-200, -1e-200, 0.0, -0.0, 1e300])
    u = sp.CsMat.new((1, 2), np.array([0, 2], np.uint64), np.array([0, 1], np.uint64),
                     [1e-200, -np.inf])
    c = sp.kronecker_product(t, u)
    assert c.nnz() == 10
    check(c, CO.kronecker_product(O(t), O(u)), kron=True)
    assert np.signbit(c.data[1]) and c.data[0] == 0.0 and not np.signbit(c.data[0])
    assert np.isnan(c.data[5]) and np.isnan(c.data[7])  # 0 * inf


# ---- 6. composition with the rest of the library
def test_laplacian_kron_sum(sp):
    """kron(I, T) + kron(T, I) on the device is the 5-point Laplacian that from_triplets builds,
    bit for bit, and it feeds LdlNumeric and spmv_dev without a download."""
    from sprs_b200 import construct as K, generate as G
    import torch
    n = 40
    ctx = sp.Context.default()
    tri = sp.CsMat.new((n, n), np.concatenate([[0], np.cumsum([2] + [3] * (n - 2) + [2])]),
                       np.concatenate([[0, 1]] + [[i - 1, i, i + 1] for i in range(1, n - 1)] +
                                      [[n - 2, n - 1]]),
                       np.concatenate([[2., -1.]] + [[-1., 2., -1.]] * (n - 2) + [[-1., 2.]]))
    eye = sp.CsMat.eye(n)
    lap = sp.kronecker_product(eye, tri) + sp.kronecker_product(tri, eye)
    r, c, v = [], [], []
    for i in range(n):
        for j in range(n):
            k = i * n + j
            for di, dj, w in ((0, 0, 4.), (-1, 0, -1.), (1, 0, -1.), (0, -1, -1.), (0, 1, -1.)):
                if 0 <= i + di < n and 0 <= j + dj < n:
                    r.append(k)
                    c.append((i + di) * n + j + dj)
                    v.append(w)
    want = sp.CsMat.from_triplets((n * n, n * n), r, c, v)
    check(lap, O(want))
    # device only: kron mirrors -> binop -> LDL and SpMV
    k1 = K.kron_dev(ctx, eye.device(), tri.device())
    k2 = K.kron_dev(ctx, tri.device(), eye.device())
    out = C.c_void_p()
    ctx.check(ctx.lib.sprs_b200_csmat_binop(ctx.h, k1.h, k2.h, sp._lib.BINOP_ADD, C.byref(out)))
    dev = sp.DeviceCsMat(ctx, out)
    if hasattr(ctx.lib, "sprs_b200_ldl_symbolic"):  # (the emulated build has no LDL^T)
        x = sp.ldl.LdlNumeric.new(dev).solve(np.ones(n * n))
        want_x = sp.ldl.LdlNumeric.new(want).solve(np.ones(n * n))
        assert x.view(np.uint64).tolist() == want_x.view(np.uint64).tolist()
    xs = torch.ones(n * n, dtype=torch.float64, device=G._device(ctx))
    y = torch.empty_like(xs)
    G.spmv(ctx, dev, xs, y)
    G._sync()
    assert np.array_equal(y.cpu().numpy(), want.to_dense() @ np.ones(n * n))


def test_kkt_bmat(sp):
    """[[H, J^T], [J, 0]] with J^T a transpose view (a CSC block)."""
    rng = np.random.default_rng(51)
    h = rand_mat(sp, rng, "CSR", 30, 30, 4.0, special=0.0)
    h = h + h.transpose_view().to_csr()
    j = rand_mat(sp, rng, "CSR", 12, 30, 3.0, special=0.0)
    k = sp.bmat([[h, j.transpose_view()], [j, None]])
    assert k.shape == (42, 42) and k.is_csr()
    check(k, CO.bmat([[O(h), CO.transpose_view(O(j))], [O(j), None]]))
    d = k.to_dense()
    assert np.array_equal(d, d.T) and np.array_equal(d[30:, 30:], np.zeros((12, 12)))


# ---- 7. 64-bit indptr everywhere (and mixed with adopted u32 blocks), in a child process
def test_construct_indptr64_child_process(sp):
    env = dict(os.environ, SPRS_B200_FORCE_INDPTR64="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider",
                        os.path.abspath(__file__), "-k",
                        "not child_process and not full_size and not test_cpp"],
                       env=env, cwd=ROOT, capture_output=True, text=True, timeout=3000)
    tail = "\n".join(r.stdout.splitlines()[-10:])
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail, r.stdout[-3000:] + r.stderr[-2000:]


# ---- 8. full size, on the device, checked against the inputs themselves
def _equal_dev(x, y):
    """device arrays equal element for element (values as 64-bit patterns)"""
    import torch
    for p, q in zip(x, y):
        if p.dtype == torch.float64:
            p, q = p.view(torch.int64), q.view(torch.int64)
        if p.dtype != q.dtype or not torch.equal(p, q):
            return False
    return True


def test_vstack_rmat10m_slices_full_size(sp):
    """config 5 (10^9 non-zeros) cut into 7 uneven row slices -- one empty, one cut beside the
    hub row -- and vstack-ed back: equal to config 5."""
    from sprs_b200 import generate as G
    import torch
    ctx = sp.Context.default()
    n = 10_000_000
    a = G.rmat_csr(ctx, n, 100, seed=0x5EED0005)
    lens = (a.indptr[1:].to(torch.int64) - a.indptr[:-1].to(torch.int64)) & 0xFFFFFFFF
    hub = int(torch.argmax(lens).item())
    cuts = sorted({0, 1, hub, hub + 1, 3_000_000, 7_777_777, n})
    slices = [a.slice_rows(r0, r1) for r0, r1 in zip(cuts[:-1], cuts[1:])]
    slices.insert(3, a.slice_rows(5, 5))  # an empty slice
    res = G.bmat(ctx, [[s] for s in slices])
    del slices
    assert res[0].rows == n and res[0].nnz == a.nnz
    assert _equal_dev(res[1:], (a.indptr, a.indices, a.data))


def test_hstack_rmat500k_csc_full_size(sp):
    """The CSC of config 4 cut into column blocks and hstack-ed back: equal to that CSC."""
    from sprs_b200 import generate as G, construct as K
    import torch
    ctx = sp.Context.default()
    n = 500_000
    a = G.rmat_csr(ctx, n, 16, seed=0x5EED0004)
    t, tip, tind, tdat = G._with_views(ctx, a.mirror.to_other_storage())  # CSC of A = CSR of A^T
    at = G.DeviceCsr(ctx, n, n, tip, tind, tdat)
    cuts = [0, 1, 77_777, 250_000, 250_001, 499_999, n]
    blocks = [at.slice_rows(c0, c1) for c0, c1 in zip(cuts[:-1], cuts[1:])]  # CSR of column blocks^T
    views = [K.transpose_view_dev(ctx, b.mirror) for b in blocks]            # CSC column blocks
    tv = [K.transpose_view_dev(ctx, v) for v in views]
    res = G._with_views(ctx, K.transpose_view_dev(ctx, K.bmat_dev(ctx, [[v] for v in tv])))
    assert res[0].storage == "CSC" and (res[0].rows, res[0].cols) == (n, n)
    assert _equal_dev(res[1:], (tip, tind, tdat))
    del t


@pytest.mark.parametrize("rmat_first", [True, False])
def test_kron_rmat500k_dense4_full_size(sp, rmat_first):
    """Kron of the config-4 R-MAT with a dense random 4x4, in both orders, against the oracle."""
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    n = 500_000
    a = G.rmat_csr(ctx, n, 16, seed=0x5EED0004)
    rng = np.random.default_rng(61)
    d = sp.CsMat.new((4, 4), np.arange(0, 17, 4), np.tile(np.arange(4), 4),
                     rng.standard_normal(16))
    d._ctx = ctx
    x, y = (a.mirror, d.device()) if rmat_first else (d.device(), a.mirror)
    res = G.kron(ctx, x, y)
    ah = CO.mat("CSR", (n, n), *a.to_host())
    want = CO.kronecker_product(ah, O(d)) if rmat_first else CO.kronecker_product(O(d), ah)
    got = CO.mat("CSR", (4 * n, 4 * n), res[1].cpu().numpy().view(np.uint32),
                 res[2].cpu().numpy().view(np.uint32), res[3].cpu().numpy())
    check(got, want, kron=True)


# ---- 9. the C++ host mirror
def test_cpp_construct_kats(sp, tmp_path):
    exe = str(tmp_path / "test_construct_kats")
    lib_dir = os.path.join(ROOT, "sprs_b200")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-Wall", "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "test_construct_kats.cpp"),
                           "-L" + lib_dir, "-lsprs_b200", "-Wl,-rpath," + lib_dir])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.startswith("OK "), r.stdout + r.stderr
