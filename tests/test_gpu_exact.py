"""Every product path checked BIT FOR BIT against the oracle, with integer-valued inputs.

The parity gate |got - ref| <= 1e-6 * sum|terms| is loose where sums are long: on a row of 10^6
N(0,1) terms it allows about the size of one product, so a kernel that drops, doubles or misroutes
one product can pass it.  Here the inputs are small integers (tests/exact.py): every partial sum
is exact in f64, every summation order gives the same bits, and each output must equal the
oracle's exactly -- across merge-path tile seams, carries, fix-ups, hot-set gathers, the atomic
SpGEMM bins and the radix-sort passes of the transposes.  The SpMM keeps N(0,1) data: it promises
the reference's storage-order bits for any values.

The SpMV seam matrix is built so that the merge-path partition (csrc/spmv.cu tile_cut_kernel:
W = 1024 cost units per tile, a row end costs 16) shows every seam below, and the test asserts
that each one occurs, so a change of the tile constants fails here instead of testing nothing."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import exact
from conftest import rand_csr

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def sp():
    import sprs_b200
    sprs_b200.Context.default()  # raises without a GPU / without the .so: no fallback
    return sprs_b200


@pytest.fixture(scope="module")
def O():
    from oracle import oracle
    return oracle


def _columns(rng, n, cols):
    """n distinct sorted columns in [0, cols)."""
    if n * 4 < cols:
        c = np.unique(rng.integers(0, cols, size=n + n // 2 + 8))
        while len(c) < n:
            c = np.unique(np.concatenate([c, rng.integers(0, cols, size=n + 8)]))
        return np.sort(rng.choice(c, size=n, replace=False))
    return np.sort(rng.choice(cols, size=n, replace=False))


def _csr_from_lens(rng, lens, cols):
    lens = np.asarray(lens, dtype=np.int64)
    ip = np.zeros(len(lens) + 1, dtype=np.int64)
    np.cumsum(lens, out=ip[1:])
    ind = np.concatenate([_columns(rng, int(n), cols) for n in lens if n] or [np.zeros(0, np.int64)])
    return ip.astype(np.uint32), ind.astype(np.uint32)


# ---------------------------------------------------------------- SpMV seam matrix
SEAM_COLS = 150_000


def seam_lengths(sp):
    """Row lengths whose merge-path partition hits every seam (see test_spmv_seam_matrix_shape):
    each segment starts exactly on a tile cut and fills whole tiles of cost W."""
    w, rc = sp.SPMV_TILE, sp.SPMV_ROW_COST
    lens = []

    def align():  # a filler row that ends exactly on the next cut
        g = -(sum(lens) + rc * len(lens)) % w
        if g:
            lens.append(g - rc if g >= rc else g + w - rc)

    # one tile per lane-group size G = 4 / 8 / 16 / 32 (cnt <= 24 / 48 / 96 * rows), with rows of
    # 8 (tiny), 9 (grouped) and 16G / 16G + 1 (the group's own loop / the whole-warp loop) inside
    lens += [8, 9, 64, 65] + [8] * 33 + [6]
    lens += [8, 9, 128, 129] + [40] * 11 + [54]
    lens += [8, 9, 256, 257] + [80] * 4 + [30]
    lens += [8, 9, 513, 430]
    lens += [8, 9, 512, 431]
    # tiles of 31 / 62 rows (31-row blocks that end exactly) and 32 / 63 (one row over)
    lens += [18] * 29 + [22]
    lens += [0] * 60 + [48]
    lens += [17] * 30 + [18]
    lens += [0] * 61 + [32]
    align()
    # tiles of 64 empty row ends
    lens += [0] * 200
    align()
    # a cut inside the row-end step of a row (clamped to the row's end), twice
    lens += [w - 8, 3]
    align()
    lens += [w - 2, 0, 5]
    align()
    # carry runs of 1, 2 and > 100 tiles, the long row between short ones inside its tiles
    lens += [1500]
    align()
    lens += [2500]
    align()
    lens += [5, 3, 110 * w, 7, 2]
    align()
    lens += [4 * w + 300, 1, 3 * w + 7]
    return lens


def seam_matrix(sp, seed=77):
    rng = np.random.default_rng(seed)
    lens = seam_lengths(sp)
    tail = rng.choice([0, 1, 3, 8, 9, 17, 33, 100, 300], 400)
    ip, ind = _csr_from_lens(rng, list(lens) + list(tail), SEAM_COLS)
    return ip, ind, exact.int_csr_data(ip, seed)


def seams(sp, ip):
    """What the partition of `ip` shows, from the numpy restatement of the tile cuts."""
    _, tr, tk = sp.spmv_rows_cut_by_tiles(ip, tiles=True)
    ip = ip.astype(np.int64)
    rows = len(ip) - 1
    n_tiles = len(tr) - 1
    t = np.arange(1, n_tiles)
    r, k = tr[t], tk[t]
    nxt = ip[np.minimum(r + 1, rows)]
    out = {}
    prev_nonempty = (r > 0) & (ip[np.maximum(r, 1)] > ip[np.maximum(r - 1, 0)])
    out["row ends on a cut"] = int(((k == ip[r]) & prev_nonempty).sum())
    out["cut in a row-end step"] = int((t * sp.SPMV_TILE - sp.SPMV_ROW_COST * r > nxt).sum())
    out["tile of 64 empty row ends"] = int(((tk[1:] == tk[:-1]) & (tr[1:] - tr[:-1] == 64)).sum())
    inside = (k > ip[r]) & (k < nxt)
    runs = np.unique(r[inside], return_counts=True)[1]
    for n in (1, 2):
        out["carry run of %d" % n] = int((runs == n).sum())
    out["carry run of >= 100"] = int((runs >= 100).sum())
    out["carry run of > 64"] = int((runs > 64).sum())
    r0, r1 = tr[:-1], tr[1:]
    nr = np.where(r1 < rows, r1, r1 - 1) - r0 + 1
    cnt = tk[1:] - tk[:-1]
    g = np.where(cnt <= 24 * nr, 4, np.where(cnt <= 48 * nr, 8, np.where(cnt <= 96 * nr, 16, 32)))
    out["31-row blocks end exactly"] = int(((nr % 31 == 0) & (nr >= 31)).sum())
    out["31-row block runs over"] = int(((nr % 31 == 1) & (nr > 31)).sum())
    # rows whose non-zeros all lie in one tile, and that tile's G
    rr = np.arange(rows)
    tile = np.searchsorted(tr, rr, side="right") - 1  # the tile that owns the row's end
    whole = ip[rr] >= tk[tile]
    lens = np.diff(ip)
    for G in (4, 8, 16, 32):
        for L in (8, 9, 16 * G, 16 * G + 1):
            out["G=%d row of %d" % (G, L)] = int((whole & (lens == L) & (g[tile] == G)).sum())
    return out


def test_spmv_seam_matrix_shape(sp):
    """Every seam the seam matrix is built for occurs in its partition."""
    ip, _, _ = seam_matrix(sp)
    missing = [name for name, n in seams(sp, ip).items() if n == 0]
    assert not missing, "the seam matrix no longer produces: %s" % missing


def _spmv_paths(sp, O, ip, ind, data, rows, cols, seed):
    """y = A x and y += A x through every SpMV entry, each bit-exact against the oracle."""
    from sprs_b200 import generate as G
    import torch
    x = exact.x_values(np.arange(cols, dtype=np.int64), seed)
    y0 = exact.y0_values(rows, seed)
    exact.assert_exact_budget(O, ip, ind, data, x, y0)
    ref = O.mul_acc_mat_vec_csr(ip, ind, data, x, np.zeros(rows))
    ref_acc = O.mul_acc_mat_vec_csr(ip, ind, data, x, y0.copy())
    a = sp.CsMat.new((rows, cols), ip, ind, data)
    exact.assert_bits(a * x, ref, "a * x")
    y = y0.copy()
    sp.prod.mul_acc_mat_vec_csr(a, x, y)
    exact.assert_bits(y, ref_acc, "mul_acc_mat_vec_csr")
    ctx = a.context()
    dev = G._device(ctx)
    xt = torch.from_numpy(x).to(dev)
    yt = torch.full((rows,), -3.0, dtype=torch.float64, device=dev)
    G.spmv(ctx, a.device(), xt, yt)
    G._sync()
    exact.assert_bits(yt.cpu().numpy(), ref, "sprs_b200_spmv_dev")
    yt = torch.from_numpy(y0.copy()).to(dev)
    G.spmv(ctx, a.device(), xt, yt, accumulate=True)
    G._sync()
    exact.assert_bits(yt.cpu().numpy(), ref_acc, "sprs_b200_spmv_dev accumulate")
    return a, x, y0, ref, ref_acc


def test_spmv_seam_matrix_exact(sp, O):
    """The seam matrix through a * x, mul_acc_mat_vec_csr (integer y0), the device entry (plain
    and accumulating), CSC mul_acc_mat_vec_csc, the one-SpMV-per-column dense product (k < 8)
    and a row slice with a non-zero-based indptr."""
    ip, ind, data = seam_matrix(sp)
    rows, cols = len(ip) - 1, SEAM_COLS
    a, x, y0, ref, ref_acc = _spmv_paths(sp, O, ip, ind, data, rows, cols, 5)
    # CSC operand: the same matrix stored by columns
    cip, cind, cdat = O.convert_mat_storage(rows, cols, ip, ind, data)
    csc = sp.CsMat.new_csc((rows, cols), cip, cind, cdat)
    y = y0.copy()
    sp.prod.mul_acc_mat_vec_csc(csc, x, y)
    exact.assert_bits(y, O.mul_acc_mat_vec_csc(cip, cind, cdat, x, y0.copy()), "mul_acc_mat_vec_csc")
    # k < 8 columns: csr_mulacc_dense_colmaj runs one SpMV per column
    k = 3
    b = np.asfortranarray(np.stack([exact.x_values(np.arange(cols, dtype=np.int64), 11 + j)
                                    for j in range(k)], axis=1))
    out0 = np.asfortranarray(np.stack([exact.y0_values(rows, 20 + j) for j in range(k)], axis=1))
    got, want = out0.copy(order="F"), out0.copy(order="F")
    sp.prod.csr_mulacc_dense_colmaj(a, b, got)
    O.csr_mulacc_dense_colmaj(ip, ind, data, b, want)
    exact.assert_bits(got, want, "csr_mulacc_dense_colmaj")
    # a row slice starting inside the structure (indptr[0] != 0): tiled from its own first
    # non-zero, so its seams fall elsewhere
    lo, hi = 41, rows - 37
    part = a.slice_outer(lo, hi)
    assert part.indptr[0] != 0
    exact.assert_bits(part * x, ref[lo:hi], "row slice")


# ---------------------------------------------------------------- configurations (child processes)
def _config_cases(out_path):
    """(child) the seam matrix and a 1M R-MAT with integer data through the SpMV entries."""
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import sprs_b200 as sp
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    res = {}
    ip, ind, data = seam_matrix(sp)
    rows = len(ip) - 1
    a = sp.CsMat.new((rows, SEAM_COLS), ip, ind, data)
    x = exact.x_values(np.arange(SEAM_COLS, dtype=np.int64), 5)
    res["seam/host"] = a * x
    y = exact.y0_values(rows, 5)
    sp.prod.mul_acc_mat_vec_csr(a, x, y)
    res["seam/host_acc"] = y
    xt = torch.from_numpy(x).cuda()
    yt = torch.empty(rows, dtype=torch.float64, device="cuda")
    G.spmv(ctx, a.device(), xt, yt)
    res["seam/dev"] = yt.cpu().numpy()
    n = 1_000_000
    r = G.rmat_csr(ctx, n, 16, seed=23)
    ai = exact.device_int_csr(ctx, r, 31)
    del r.mirror
    x = exact.device_x(ctx, n, 6)
    y = torch.empty(n, dtype=torch.float64, device="cuda")
    G.spmv(ctx, ai, x, y)
    res["rmat/dev"] = y.cpu().numpy()
    y = torch.from_numpy(exact.y0_values(n, 6)).cuda()
    G.spmv(ctx, ai, x, y, accumulate=True)
    res["rmat/dev_acc"] = y.cpu().numpy()
    hip, hind, hdat = ai.to_host()
    hx, hy = x.cpu().numpy(), np.empty(n)
    ctx.check(ctx.lib.sprs_b200_mul_mat_vec(ctx.h, ai.mirror.h, hx.ctypes.data_as(C.c_void_p), n,
                                            hy.ctypes.data_as(C.c_void_p), n))
    res["rmat/host"] = hy
    res["rmat/indptr"], res["rmat/indices"], res["rmat/data"] = hip, hind, hdat
    np.savez(out_path, **res)


CONFIGS = {
    "hot_off": dict(SPRS_B200_SPMV_HOT="0"),
    "hot_1023": dict(SPRS_B200_SPMV_HOT="1023"),
    "hot_24576": dict(SPRS_B200_SPMV_HOT="24576"),
    "force_indptr64": dict(SPRS_B200_FORCE_INDPTR64="1"),
    "chunked_host_path": dict(SPRS_B200_E2E_CHUNKS="5", SPRS_B200_E2E_MIN_TILES="1"),
}


@pytest.mark.parametrize("config", sorted(CONFIGS))
def test_spmv_exact_configuration_child_process(tmp_path, O, config):
    """The seam matrix and a 1M R-MAT, integer data, under each switch of the SpMV (read once
    per process): hot set off / K = 1023 / K = 24576, 64-bit indptr instantiations, and the
    chunked host path (tile-range launches + carry fix-ups).  Every y bit-exact vs the oracle."""
    sys.path.insert(0, ROOT)
    import sprs_b200 as sp
    env = {k: v for k, v in os.environ.items() if not k.startswith("SPRS_B200_")}
    env.update(CONFIGS[config])
    out = os.path.join(str(tmp_path), config + ".npz")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), out], capture_output=True,
                       text=True, timeout=900, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    got = dict(np.load(out))
    ip, ind, data = seam_matrix(sp)
    rows = len(ip) - 1
    x = exact.x_values(np.arange(SEAM_COLS, dtype=np.int64), 5)
    ref = O.mul_acc_mat_vec_csr(ip, ind, data, x, np.zeros(rows))
    exact.assert_bits(got["seam/host"], ref, config + ": seam a * x")
    exact.assert_bits(got["seam/dev"], ref, config + ": seam device")
    y0 = exact.y0_values(rows, 5)
    exact.assert_bits(got["seam/host_acc"], O.mul_acc_mat_vec_csr(ip, ind, data, x, y0.copy()),
                      config + ": seam mul_acc")
    hip, hind, hdat = got["rmat/indptr"], got["rmat/indices"], got["rmat/data"]
    n = len(hip) - 1
    # the device generated the same values as the host formula
    exact.assert_bits(hdat, exact.int_csr_data(hip, 31), config + ": device integer data")
    x = exact.x_values(np.arange(n, dtype=np.int64), 6)
    y0 = exact.y0_values(n, 6)
    exact.assert_exact_budget(O, hip, hind, hdat, x, y0)
    ref = O.mul_acc_mat_vec_csr(hip, hind, hdat, x, np.zeros(n))
    exact.assert_bits(got["rmat/dev"], ref, config + ": R-MAT device")
    exact.assert_bits(got["rmat/host"], ref, config + ": R-MAT host path")
    exact.assert_bits(got["rmat/dev_acc"], O.mul_acc_mat_vec_csr(hip, hind, hdat, x, y0.copy()),
                      config + ": R-MAT device accumulate")


# ---------------------------------------------------------------- SpMM (N(0,1): storage-order bits)
SPMM_KS = [1, 7, 8, 31, 32, 33, 63, 64, 65, 66, 127, 128, 129, 130, 200, 256, 257]


@pytest.fixture(scope="module")
def spmm_mat():
    rng = np.random.default_rng(2024)
    ip, ind, d = rand_csr(rng, 120, 300, 9, skew=True, empty_frac=0.1)
    return ip, ind, d


def test_spmm_k_sweep_bits(sp, O, spmm_mat):
    """csr_mulacc_dense_rowmaj (the SpMM kernels: 128-bit for even k, scalar for odd) at every
    k around the column-panel widths (64 / 128 columns per pass), accumulating into a non-zero
    C; and `a * b` (k >= 8) from zero."""
    ip, ind, d = spmm_mat
    rows, cols = len(ip) - 1, 300
    a = sp.CsMat.new((rows, cols), ip, ind, d)
    rng = np.random.default_rng(7)
    for k in SPMM_KS:
        b = rng.standard_normal((cols, k))
        c0 = rng.standard_normal((rows, k))
        got, want = c0.copy(), c0.copy()
        sp.prod.csr_mulacc_dense_rowmaj(a, b, got)
        O.csr_mulacc_dense_rowmaj(ip, ind, d, b, want)
        exact.assert_bits(got, want, "csr_mulacc_dense_rowmaj k=%d" % k)
        if k >= 8:
            exact.assert_bits(a * b, O.csr_mulacc_dense_rowmaj(ip, ind, d, b, np.zeros((rows, k))),
                              "a * b k=%d" % k)


@pytest.mark.parametrize("k", [8, 33, 64, 66, 129, 130, 256])
def test_spmm_rowmaj_dev_strides_bits(sp, O, spmm_mat, k):
    """sprs_b200_spmm_rowmaj_dev with ldb / ldc = k + 1 and k + 3, and with B / C starting 8
    bytes into their buffers (the scalar fallback for even k), plain and accumulating.  Padding
    columns and guard elements hold a sentinel that must survive; B's padding is NaN, so a read
    of it would poison the result."""
    import torch
    from sprs_b200 import generate as G
    ip, ind, d = spmm_mat
    rows, cols = len(ip) - 1, 300
    a = sp.CsMat.new((rows, cols), ip, ind, d)
    ctx = a.context()
    dev = G._device(ctx)
    rng = np.random.default_rng(k)
    b = rng.standard_normal((cols, k))
    c0 = rng.standard_normal((rows, k))
    sentinel, guard = -7.25, 5
    for ld_extra, off in ((1, 0), (3, 0), (0, 1), (3, 1)):
        ldb = ldc = k + ld_extra
        for acc in (0, 1):
            bb = np.full(off + cols * ldb + guard, np.nan)
            bb[off:off + cols * ldb].reshape(cols, ldb)[:, :k] = b
            cc = np.full(off + rows * ldc + guard, sentinel)
            cc[off:off + rows * ldc].reshape(rows, ldc)[:, :k] = c0
            bt, ct = torch.from_numpy(bb).to(dev), torch.from_numpy(cc).to(dev)
            G._sync()
            ctx.check(ctx.lib.sprs_b200_spmm_rowmaj_dev(
                ctx.h, a.device().h, C.c_void_p(bt.data_ptr() + 8 * off), ldb, k,
                C.c_void_p(ct.data_ptr() + 8 * off), ldc, acc, G._stream_ptr()))
            ctx.synchronize()
            G._sync()
            out = ct.cpu().numpy()
            what = "k=%d ld=%d offset=%d accumulate=%d" % (k, ldb, off, acc)
            body = out[off:off + rows * ldc].reshape(rows, ldc)
            want = O.csr_mulacc_dense_rowmaj(ip, ind, d, b, c0.copy() if acc else np.zeros((rows, k)))
            exact.assert_bits(body[:, :k], want, what)
            assert np.all(body[:, k:] == sentinel), what + ": padding columns written"
            assert np.all(out[:off] == sentinel) and np.all(out[off + rows * ldc:] == sentinel), \
                what + ": guard elements written"


# ---------------------------------------------------------------- SpGEMM, integer data
def spgemm_operands(rng, a_units, n_pairs, b_lens, b_cols, seed, b_cols_fn=None):
    """B: rows 2i and 2i + 1 (i < n_pairs) are negations of each other, the others free; A: row
    r takes a_units[r] = (pairs, singles) -- both rows of `pairs` pairs with ONE coefficient (so
    their products cancel to +0.0 where nothing else lands) and `singles` unpaired rows."""
    n_b = len(b_lens)
    b_lens = np.array(b_lens, dtype=np.int64)
    b_lens[1:2 * n_pairs:2] = b_lens[0:2 * n_pairs:2]
    b_ip = np.zeros(n_b + 1, dtype=np.int64)
    np.cumsum(b_lens, out=b_ip[1:])
    b_ind = np.zeros(int(b_ip[-1]), dtype=np.int64)
    for r in range(n_b):
        if r < 2 * n_pairs and r % 2 == 1:
            b_ind[b_ip[r]:b_ip[r + 1]] = b_ind[b_ip[r - 1]:b_ip[r]]
        elif b_lens[r]:
            b_ind[b_ip[r]:b_ip[r + 1]] = (b_cols_fn or _columns)(rng, int(b_lens[r]), b_cols)
    b_dat = exact.int_csr_data(b_ip, seed)
    for i in range(n_pairs):
        b_dat[b_ip[2 * i + 1]:b_ip[2 * i + 2]] = -b_dat[b_ip[2 * i]:b_ip[2 * i + 1]]
    rows = []
    for pairs, singles in a_units:
        p = rng.choice(n_pairs, size=pairs, replace=False) if pairs else np.zeros(0, np.int64)
        s = 2 * n_pairs + rng.choice(n_b - 2 * n_pairs, size=singles, replace=False) if singles \
            else np.zeros(0, np.int64)
        rows.append(np.sort(np.concatenate([2 * p, 2 * p + 1, s])))
    a_ip = np.zeros(len(rows) + 1, dtype=np.int64)
    np.cumsum([len(r) for r in rows], out=a_ip[1:])
    a_ind = np.concatenate(rows) if rows else np.zeros(0, np.int64)
    a_dat = exact.int_csr_data(a_ip, seed + 1)
    paired = (a_ind < 2 * n_pairs) & (a_ind % 2 == 1)  # second row of a pair: same coefficient
    a_dat[paired] = a_dat[np.flatnonzero(paired) - 1]
    u = np.uint32
    return ((a_ip.astype(u), a_ind.astype(u), a_dat), (len(rows), n_b),
            (b_ip.astype(u), b_ind.astype(u), b_dat), (n_b, b_cols))


def spgemm_exact(sp, O, a, a_shape, b, b_shape, what):
    """C = A B on the device, all three arrays bit-exact vs the oracle; returns the oracle's C."""
    exact.assert_spgemm_budget(O, a_shape, a, b_shape, b)
    want = O.mul_csr_csr(a_shape, a, b_shape, b, threads=1)
    c = sp.CsMat.new(a_shape, *a) * sp.CsMat.new(b_shape, *b)
    exact.assert_csr_bits((c.indptr, c.indices, c.data), want, what)
    return want


def _row_stats(O, a, a_shape, b, b_shape, want):
    """n_prod and nnz(C) per row (what the bins route by)."""
    b_len = np.diff(b[0].astype(np.int64))
    cs = np.concatenate([[0], np.cumsum(b_len[a[1].astype(np.int64)])])
    a_ip = a[0].astype(np.int64)
    return cs[a_ip[1:]] - cs[a_ip[:-1]], np.diff(want[0].astype(np.int64)), np.diff(a_ip)


def _cancelled(want):
    """C entries that cancelled to exactly +0.0 (kept, with their index, like the reference)."""
    return int(np.sum(want[2].view(np.uint64) == 0))


def test_spgemm_exact_warp_bin(sp, O):
    """C rows of <= 128 entries: one warp per row, symbolic and numeric."""
    rng = np.random.default_rng(1)
    units = [(int(rng.integers(0, 3)), int(rng.integers(0, 5))) for _ in range(400)]
    a, ash, b, bsh = spgemm_operands(rng, units, 100, rng.integers(0, 12, 500), 3000, 10)
    want = spgemm_exact(sp, O, a, ash, b, bsh, "warp bin")
    nprod, nnzc, _ = _row_stats(O, a, ash, b, bsh, want)
    assert nprod.max() <= 128 and (nnzc > 0).sum() > 250
    assert _cancelled(want) > 0


def test_spgemm_exact_cta_hash_bins(sp, O):
    """128 < n_prod <= B.cols / 256: the CTA hash set (symbolic); 128 < nnz(C_i) <= 1024: the
    CTA hash map with shared-memory atomics (numeric)."""
    rng = np.random.default_rng(2)
    cols = 400_000
    units = [(int(rng.integers(2, 6)), int(rng.integers(8, 20))) for _ in range(60)]
    a, ash, b, bsh = spgemm_operands(rng, units, 200, rng.integers(10, 40, 1000), cols, 20)
    want = spgemm_exact(sp, O, a, ash, b, bsh, "CTA hash bins")
    nprod, nnzc, _ = _row_stats(O, a, ash, b, bsh, want)
    assert np.sum((nprod > 128) & (nprod <= cols // 256)) >= 20
    assert np.sum((nnzc > 128) & (nnzc <= 1024)) >= 20
    assert _cancelled(want) > 0


def test_spgemm_exact_symbolic_bitmaps(sp, O):
    """n_prod > B.cols / 256: the symbolic bitmap in shared memory (B.cols <= 1.6M) and, for
    B.cols > 1.6M and n_prod > 8192, in global memory."""
    rng = np.random.default_rng(3)
    units = [(int(rng.integers(2, 6)), int(rng.integers(8, 20))) for _ in range(40)]
    a, ash, b, bsh = spgemm_operands(rng, units, 100, rng.integers(10, 40, 600), 20_000, 30)
    want = spgemm_exact(sp, O, a, ash, b, bsh, "shared-memory bitmap")
    nprod, _, _ = _row_stats(O, a, ash, b, bsh, want)
    assert np.sum(nprod > 20_000 // 256) >= 30 and _cancelled(want) > 0
    cols = 1_700_000
    units = [(20, 80), (5, 90), (0, 3), (30, 70)]
    a, ash, b, bsh = spgemm_operands(rng, units, 60, rng.integers(80, 120, 300), cols, 40)
    want = spgemm_exact(sp, O, a, ash, b, bsh, "global-memory bitmap")
    nprod, _, _ = _row_stats(O, a, ash, b, bsh, want)
    assert np.sum(nprod > 8192) >= 3 and _cancelled(want) > 0


def _skip_middle_panel(rng, n, cols):
    """columns of a B row with nothing in the middle panel [16384, 32768)."""
    lo = _columns(rng, n // 2, 16384)
    hi = 32768 + _columns(rng, n - n // 2, cols - 32768)
    return np.concatenate([lo, hi])


@pytest.mark.parametrize("cols", [16384, 16385, 40_000])
def test_spgemm_exact_panel_kernel(sp, O, cols):
    """nnz(C_i) > 1024 with <= 4096 A non-zeros: dense shared-memory panels of 16384 columns.
    A rows of 1, 2, 3, 16, 17 and 40 non-zeros (G = 32, 16, 8, 2 warps per B row, and G = 1);
    at 40000 columns half the B rows have nothing in the middle panel (the skip branch)."""
    rng = np.random.default_rng(cols)
    n_b, n_pairs = 300, 60
    b_lens = rng.integers(1100, 1600, n_b)
    fn = _skip_middle_panel if cols > 32768 else None
    units = []
    for na in (1, 2, 3, 16, 17, 40):
        units += [(0, na), (na // 2, na - 2 * (na // 2))] * 2
    a, ash, b, bsh = spgemm_operands(rng, units, n_pairs, b_lens, cols, 50,
                                     b_cols_fn=(lambda r, n, c: fn(r, n, c) if r.integers(0, 2) else
                                                _columns(r, n, c)) if fn else None)
    want = spgemm_exact(sp, O, a, ash, b, bsh, "panel kernel, %d columns" % cols)
    _, nnzc, na = _row_stats(O, a, ash, b, bsh, want)
    assert np.all(nnzc > 1024) and set(na.tolist()) >= {1, 2, 3, 16, 17, 40}
    assert _cancelled(want) > 0


def _hub_case(sp, O, rng, n_hub, what):
    n_b, n_pairs, cols = 6000, 1500, 8000
    units = [(int(rng.integers(1100, 1500)), int(rng.integers(2000, 2900))) for _ in range(n_hub)]
    a, ash, b, bsh = spgemm_operands(rng, units, n_pairs, rng.integers(1, 4, n_b), cols, 60)
    want = spgemm_exact(sp, O, a, ash, b, bsh, what)
    _, nnzc, na = _row_stats(O, a, ash, b, bsh, want)
    assert np.all(na > 4096) and np.all(nnzc > 1024) and _cancelled(want) > 0


def test_spgemm_exact_hub_rows_few(sp, O):
    """Fewer hub rows (> 4096 A non-zeros) than SMs: the 1024-thread launch, one row per CTA."""
    n = max(1, min(3, sp.Context.default().sm_count - 1))
    _hub_case(sp, O, np.random.default_rng(5), n, "%d hub rows" % n)


def test_spgemm_exact_hub_rows_many(sp, O):
    """At least 2 * sm_count + 5 hub rows: the 256-thread launch of 2 * sm_count CTAs, some CTAs
    taking a second row on the accumulator the first one left zeroed."""
    n = 2 * sp.Context.default().sm_count + 5
    _hub_case(sp, O, np.random.default_rng(6), n, "%d hub rows" % n)


# ---------------------------------------------------------------- non-finite isolation
def test_spmv_nonfinite_isolation(sp, O):
    """NaN, +Inf and -Inf in x at chosen columns, each row touching at most one of them (long
    rows across tiles and carries included): rows that touch none stay bit-exact, the others
    match the oracle's class and sign."""
    rng = np.random.default_rng(8)
    ip, ind, data = seam_matrix(sp)
    rows, n_bad = len(ip) - 1, 150
    cols = SEAM_COLS + n_bad  # columns no row of the seam matrix uses
    x = exact.x_values(np.arange(cols, dtype=np.int64), 5)
    ip64 = ip.astype(np.int64)
    ind = ind.copy()
    # each chosen row's last entry moves to its own poisoned column (above all others: the row
    # stays sorted); every long row across tiles is among them
    lens = np.diff(ip64)
    long_rows = np.flatnonzero(lens > 2 * sp.SPMV_TILE)
    others = np.setdiff1d(np.flatnonzero(lens > 0), long_rows)
    chosen = np.concatenate([long_rows, rng.choice(others, n_bad - len(long_rows), replace=False)])
    bad_cols = SEAM_COLS + np.arange(n_bad)
    ind[ip64[chosen + 1] - 1] = bad_cols
    x[bad_cols[0::3]], x[bad_cols[1::3]], x[bad_cols[2::3]] = np.nan, np.inf, -np.inf
    a = sp.CsMat.new((rows, cols), ip, ind, data)
    ref = O.mul_acc_mat_vec_csr(ip, ind, data, x, np.zeros(rows))
    hit = ~np.isfinite(ref)
    assert hit.sum() >= 100 and (~hit).sum() > rows // 2
    exact.assert_same_class(a * x, ref, "spmv with non-finite x")


def test_spmm_nonfinite_isolation(sp, O, spmm_mat):
    """A B row holding NaN / +-Inf: C rows that do not use it bit-exact, the others by class."""
    ip, ind, d = spmm_mat
    rows, cols = len(ip) - 1, 300
    a = sp.CsMat.new((rows, cols), ip, ind, d)
    rng = np.random.default_rng(9)
    j = int(np.bincount(ind.astype(np.int64), minlength=cols).argmax())
    for k in (8, 66, 129):
        b = rng.standard_normal((cols, k))
        b[j, 0::3], b[j, 1::3], b[j, 2::3] = np.nan, np.inf, -np.inf
        ref = O.csr_mulacc_dense_rowmaj(ip, ind, d, b, np.zeros((rows, k)))
        assert (~np.isfinite(ref)).any() and np.isfinite(ref).all(axis=1).sum() > rows // 2
        exact.assert_same_class(a * b, ref, "spmm k=%d with a non-finite B row" % k)


def test_spgemm_nonfinite_isolation(sp, O):
    """One B row of each kind holds NaN / +-Inf.  The medium (hash map), panel and hub bins get
    more rows than their launches have CTAs (8 / 1 / 2 per SM), with the poisoned rows spread
    among clean ones: a CTA that leaks its accumulator into its next row shows up as a NaN or a
    wrong value in a clean row.  Which CTA takes which row is decided at run time, so this
    makes a leak likely to show, not certain."""
    rng = np.random.default_rng(10)
    sm = sp.Context.default().sm_count
    n_short, n_long, cols = 5000, 1000, 40_000
    b_lens = np.concatenate([rng.integers(1, 3, n_short), rng.integers(30, 50, n_long)])
    n_med, n_pan, n_hub = 8 * sm + 5, 3 * sm + 5, 3 * sm + 5
    kinds = rng.permutation(np.repeat([0, 1, 2], [n_med, n_pan, n_hub]))
    bad_short, bad_long = 100, n_short + 500
    b_lens[bad_short] = 3
    rows = []
    for i, kd in enumerate(kinds):
        if kd == 2:
            r = rng.choice(n_short, size=4200, replace=False)
        else:
            r = n_short + rng.choice(n_long, size=10 if kd == 0 else 40, replace=False)
        r = r[(r != bad_short) & (r != bad_long)]
        if i % 3 == 0:
            r = np.append(r, bad_short if kd == 2 else bad_long)
        rows.append(np.sort(r))
    a_ip = np.zeros(len(rows) + 1, dtype=np.int64)
    np.cumsum([len(r) for r in rows], out=a_ip[1:])
    a = (a_ip.astype(np.uint32), np.concatenate(rows).astype(np.uint32), exact.int_csr_data(a_ip, 70))
    b_ip = np.zeros(len(b_lens) + 1, dtype=np.int64)
    np.cumsum(b_lens, out=b_ip[1:])
    b_ind = np.concatenate([_columns(rng, int(n), cols) for n in b_lens]).astype(np.uint32)
    b_dat = exact.int_csr_data(b_ip, 71)
    for r in (bad_short, bad_long):
        s = b_ip[r]
        b_dat[s:b_ip[r + 1]][:3] = [np.nan, np.inf, -np.inf][:b_ip[r + 1] - s]
    b = (b_ip.astype(np.uint32), b_ind, b_dat)
    ash, bsh = (len(rows), len(b_lens)), (len(b_lens), cols)
    want = O.mul_csr_csr(ash, a, bsh, b, threads=1)
    _, nnzc, na = _row_stats(O, a, ash, b, bsh, want)
    assert np.sum((nnzc > 128) & (nnzc <= 1024)) > 8 * sm and np.sum(na > 4096) > 2 * sm
    assert np.sum((nnzc > 1024) & (na <= 4096)) > sm
    c = sp.CsMat.new(ash, *a) * sp.CsMat.new(bsh, *b)
    exact.assert_csr_bits((c.indptr, c.indices, np.zeros(len(c.data))),
                          (want[0], want[1], np.zeros(len(want[2]))), "structure")
    poisoned = ~np.isfinite(want[2])
    assert poisoned.sum() >= n_med // 3
    exact.assert_same_class(c.data, want[2], "spgemm with non-finite B rows")


# ---------------------------------------------------------------- conversions
@pytest.mark.parametrize("inner", [200, 60_000, 3_000_000, 20_000_000])
def test_to_other_storage_radix_passes_exact(sp, O, inner):
    """CSR -> CSC and back, bit-exact, for inner dimensions that need 1, 2, 3 and 4 passes of
    the 8-bit radix sort (hypersparse: a few thousand non-zeros)."""
    rng = np.random.default_rng(inner)
    rows = 3000
    lens = rng.integers(0, 8, rows)
    ip, ind = _csr_from_lens(rng, lens, inner)
    data = rng.standard_normal(len(ind))
    a = sp.CsMat.new((rows, inner), ip, ind, data)
    t = a.to_other_storage()
    want = O.convert_mat_storage(rows, inner, ip, ind, data)
    exact.assert_csr_bits((t.indptr, t.indices, t.data), want, "to_other_storage, %d columns" % inner)
    back = t.to_other_storage()
    exact.assert_csr_bits((back.indptr, back.indices, back.data), (ip, ind, data), "round trip")


@pytest.mark.parametrize("shape", [(700, 900), (1 << 24 | 5, (1 << 25) + 3)])
def test_from_triplets_integer_duplicates_exact(sp, O, shape):
    """COO with duplicates (integer values: every duplicate sum exact, whatever the order)
    against triplets_to_csr, all three arrays -- also with both dimensions above 2^24."""
    rng = np.random.default_rng(shape[0] & 0xFFFF)
    n = 6000
    pr = rng.integers(0, shape[0], 1500)
    pc = rng.integers(0, shape[1], 1500)
    take = rng.integers(0, 1500, n)
    r, c = pr[take], pc[take]
    v = exact.mat_values(np.arange(n, dtype=np.int64), 90)
    m = sp.CsMat.from_triplets(shape, r, c, v)
    want = O.triplets_to_csr(shape, r, c, v, np.uint64)
    exact.assert_csr_bits((m.indptr, m.indices, m.data), want, "from_triplets %s" % (shape,))


# ---------------------------------------------------------------- full size
def test_spmv_rmat_10m_exact_full_size(sp, O):
    """BASELINE config 5 (10M x 10M R-MAT, ~1e9 non-zeros, rows up to ~1e6) with integer data
    and the default hot-set setting (`auto` builds it at this size): the whole y, plain and
    accumulating, bit-exact against the oracle."""
    import torch
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    n = 10_000_000
    a = G.rmat_csr(ctx, n, 100, seed=0x5EED0005)
    ai = exact.device_int_csr(ctx, a, 101)
    del a  # the structure is shared; the N(0,1) values and their mirror go
    torch.cuda.empty_cache()
    x = exact.device_x(ctx, n, 102)
    y = torch.empty(n, dtype=torch.float64, device="cuda")
    G.spmv(ctx, ai, x, y)
    y0 = exact.y0_values(n, 103)
    ya = torch.from_numpy(y0).cuda()
    G.spmv(ctx, ai, x, ya, accumulate=True)
    G._sync()
    hip, hind, hdat = ai.to_host()
    hx = x.cpu().numpy()
    exact.assert_bits(hx, exact.x_values(np.arange(n, dtype=np.int64), 102), "device x")
    exact.assert_exact_budget(O, hip, hind, hdat, hx, y0)
    exact.assert_bits(y.cpu().numpy(), O.mul_acc_mat_vec_csr(hip, hind, hdat, hx, np.zeros(n)), "y = A x")
    exact.assert_bits(ya.cpu().numpy(), O.mul_acc_mat_vec_csr(hip, hind, hdat, hx, y0.copy()), "y += A x")


def test_spmv_rand_1m_exact_full_size(sp, O):
    """BASELINE config 2 (1M x 1M sprs-rand, 32 non-zeros per row), integer data: whole y."""
    import torch
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    n = 1_000_000
    a = G.rand_csr(ctx, n, n, 32, seed=0x5EED0002)
    ai = exact.device_int_csr(ctx, a, 201)
    del a
    x = exact.device_x(ctx, n, 202)
    y = torch.empty(n, dtype=torch.float64, device="cuda")
    G.spmv(ctx, ai, x, y)
    G._sync()
    hip, hind, hdat = ai.to_host()
    hx = x.cpu().numpy()
    exact.assert_exact_budget(O, hip, hind, hdat, hx)
    exact.assert_bits(y.cpu().numpy(), O.mul_acc_mat_vec_csr(hip, hind, hdat, hx, np.zeros(n)), "y = A x")


def test_spgemm_rmat_500k_row_block_exact_full_size(sp, O):
    """BASELINE config 4 (two 500k x 500k R-MAT, ~16 non-zeros per row), integer data: a row
    block of A holding >= 1e8 products, indptr, indices and EVERY value bit-exact."""
    import torch
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    n = 500_000
    A = exact.device_int_csr(ctx, G.rmat_csr(ctx, n, 16, seed=0x5EED0004), 301)
    B = exact.device_int_csr(ctx, G.rmat_csr(ctx, n, 16, seed=0x5EED1004), 302)
    torch.cuda.empty_cache()
    cmir, cip, cind, cdat = G.spgemm(ctx, A, B)
    aip = A.indptr.to(torch.int64) & 0xFFFFFFFF
    blen = (B.indptr[1:].to(torch.int64) & 0xFFFFFFFF) - (B.indptr[:-1].to(torch.int64) & 0xFFFFFFFF)
    per_nnz = blen[A.indices.to(torch.int64) & 0xFFFFFFFF]
    csum = torch.cumsum(per_nnz, 0)
    r0 = 2000
    base = int(csum[int(aip[r0]) - 1].item()) if int(aip[r0]) > 0 else 0
    k_end = int(torch.searchsorted(csum, torch.tensor([base + 100_000_000], device=csum.device))[0])
    r1 = min(n, int(torch.searchsorted(aip, torch.tensor([k_end], device=aip.device))[0]) + 1)
    assert int(csum[int(aip[r1]) - 1].item()) - base >= 100_000_000
    # exact: every C value is a sum of at most max(n_prod_i) products of magnitude <= 64
    row_prod = torch.zeros(n, dtype=torch.int64, device=aip.device)
    row_prod.index_add_(0, torch.repeat_interleave(torch.arange(n, device=aip.device), aip[1:] - aip[:-1]),
                        per_nnz)
    assert int(row_prod.max()) * 64 < exact.EXACT_LIMIT
    blk = A.slice_rows(r0, r1)
    want = O.mul_csr_csr((r1 - r0, n), blk.to_host(), (n, n), B.to_host(), threads=0)
    cip64 = cip.to(torch.int64)
    if cip.dtype == torch.int32:
        cip64 &= 0xFFFFFFFF
    s, e = int(cip64[r0]), int(cip64[r1])
    got = ((cip64[r0:r1 + 1] - s).cpu().numpy(), cind[s:e].cpu().numpy().view(np.uint32),
           cdat[s:e].cpu().numpy())
    exact.assert_csr_bits(got, want, "config 4 row block")
    del cmir


if __name__ == "__main__":
    _config_cases(sys.argv[1])
