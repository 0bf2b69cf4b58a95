"""SpGEMM values BIT FOR BIT against the oracle with real-valued inputs, in every numeric bin.

The reference adds row i's products into tmp[j] one A non-zero after the other, in storage
order, each sum starting from +0.0, multiply and add rounded separately (smmp.rs:151-189), so
`O.mul_csr_csr(..., threads=1)` is the exact bit reference.  The integer-valued tests
(test_gpu_exact.py) cannot see the order: every partial sum is exact there.  Here the values are
N(0,1), and N(0,1) scaled by 2^k (k uniform in [-20, 20], per B row and per A entry), where
almost any re-association changes a bit, and every value must match the oracle (NaN by class).

Two-term sums are order-free ((0 + a) + b == (0 + b) + a), so each test asserts on the host that
its bin is reached AND that the bin holds a few hundred C entries of three or more terms, and --
with the oracle alone -- that summing the same product in another order (A P times P^T B for a
random permutation P of the inner dimension) changes a stated share of those entries: the test
would see a kernel that adds in another order.

Value edges are planted in every bin: -0.0 in A and in B, products that underflow to -0.0, a
column of terms near 1e308 whose overflow depends on the order (1e308 + 1e308 - 1e308 is +Inf in
storage order, 1e308 in another), exact cancellation (pairs of negated B rows under one A
coefficient), and NaN / +-Inf entries of B beside clean rows."""
import ctypes as C

import numpy as np
import pytest

import exact
from test_gpu_exact import _columns, _row_stats, spgemm_operands

pytestmark = pytest.mark.gpu
BIG = 1e308


@pytest.fixture(scope="module")
def sp():
    import sprs_b200
    sprs_b200.Context.default()  # raises without a GPU / without the .so: no fallback
    return sprs_b200


@pytest.fixture(scope="module")
def O():
    from oracle import oracle
    return oracle


# ---------------------------------------------------------------- operands and values
def _pairs_of_operands(b, n_pairs):
    """B rows that are the negation of the row before them (spgemm_operands' pairs)."""
    second = np.zeros(len(b[0]) - 1, dtype=bool)
    second[1:2 * n_pairs:2] = True
    return second


def designed(rng, specs, cols):
    """One A row per spec (n_c, na, blen, hot) over B rows of its own: the A row has na B rows
    whose columns come from one set S of n_c columns (so nnz(C_i) == n_c), the first ones
    covering S, the others blen columns of S each; its first two B rows are a negated pair.
    `hot`: every B row of the A row also holds S[0].  Returns (a, a_shape, b, b_shape, second)."""
    b_rows, second, a_rows = [], [], []
    for n_c, na, blen, hot in specs:
        s = np.sort(rng.choice(cols, n_c, replace=False))
        cover = [np.sort(c) for c in np.array_split(rng.permutation(s), -(-n_c // blen))]
        assert len(cover) + 1 <= na
        rows = [cover[0], cover[0].copy()] + cover[1:]
        while len(rows) < na:
            rows.append(np.sort(rng.choice(s, min(blen, n_c), replace=False)))
        if hot:
            rows = [np.union1d(r, s[:1]) for r in rows]
        a_rows.append(len(b_rows) + np.arange(len(rows)))
        second += [False, True] + [False] * (len(rows) - 2)
        b_rows += rows
    return _assemble(a_rows, b_rows, cols) + (np.array(second),)


def _assemble(a_rows, b_rows, cols):
    u = np.uint32
    b_ip = np.zeros(len(b_rows) + 1, dtype=np.int64)
    np.cumsum([len(r) for r in b_rows], out=b_ip[1:])
    a_ip = np.zeros(len(a_rows) + 1, dtype=np.int64)
    np.cumsum([len(r) for r in a_rows], out=a_ip[1:])
    a = (a_ip.astype(u), np.concatenate(a_rows).astype(u), np.zeros(int(a_ip[-1])))
    b = (b_ip.astype(u), np.concatenate(b_rows).astype(u), np.zeros(int(b_ip[-1])))
    return a, (len(a_rows), len(b_rows)), b, (len(b_rows), cols)


def realize(rng, a, b, second, scaled):
    """N(0,1) data (times 2^k, k in [-20, 20] per B row and per A entry, when `scaled`), with
    each negated pair of B rows under one A coefficient: their products cancel exactly."""
    b_ip = b[0].astype(np.int64)
    b_len = np.diff(b_ip)
    bd = rng.standard_normal(int(b_ip[-1]))
    ad = rng.standard_normal(len(a[1]))
    if scaled:
        bd *= np.repeat(np.exp2(rng.integers(-20, 21, len(b_len))), b_len)
        ad *= np.exp2(rng.integers(-20, 21, len(ad)))
    for r in np.flatnonzero(second):
        assert b_len[r] == b_len[r - 1]
        bd[b_ip[r]:b_ip[r + 1]] = -bd[b_ip[r - 1]:b_ip[r]]
    a_ind = a[1].astype(np.int64)
    hit = np.flatnonzero(second[a_ind])
    assert np.all(a_ind[hit - 1] == a_ind[hit] - 1), "a pair's rows must be adjacent in A"
    ad[hit] = ad[hit - 1]
    return (a[0], a[1], ad), (b[0], b[1], bd)


def plant_edges(rng, a, b, second, n_nonfinite=3):
    """-0.0 in A and B, a B row of tiny values under tiny A coefficients (products underflow to
    +-0.0), a column of terms +1e308, +1e308, -1e308 in storage order (overflow depends on the
    order), and NaN / +Inf / -Inf in `n_nonfinite` B rows.  Pairs are left alone."""
    a_ip, a_ind = a[0].astype(np.int64), a[1].astype(np.int64)
    b_ip, b_ind = b[0].astype(np.int64), b[1].astype(np.int64)
    ad, bd = a[2].copy(), b[2].copy()
    paired = second | np.append(second[1:], False)  # either row of a pair
    free_rows = np.flatnonzero(~paired & (np.diff(b_ip) > 0))
    free_b = np.flatnonzero(~paired[np.repeat(np.arange(len(second)), np.diff(b_ip))])
    free_a = np.flatnonzero(~paired[a_ind])
    bd[rng.choice(free_b, max(1, len(free_b) // 100), replace=False)] = -0.0
    ad[rng.choice(free_a, max(1, len(free_a) // 100), replace=False)] = -0.0
    used = np.intersect1d(free_rows, a_ind)
    tiny = rng.choice(used, max(1, len(used) // 50), replace=False)
    for r in tiny:
        bd[b_ip[r]:b_ip[r + 1]] = 1e-200 * np.where(rng.random(b_ip[r + 1] - b_ip[r]) < 0.5, -1.0, 1.0)
    on_tiny = np.isin(a_ind, tiny)
    ad[on_tiny] = 1e-200 * np.where(rng.random(on_tiny.sum()) < 0.5, -1.0, 1.0)
    # order-dependent overflow: the first C entry (in a random row order) with three terms from
    # rows that are neither paired nor tiny
    ok = ~paired.copy()
    ok[tiny] = False
    planted = 0
    for i in rng.permutation(len(a_ip) - 1):
        ks = a_ind[a_ip[i]:a_ip[i + 1]]
        pos = np.arange(a_ip[i], a_ip[i + 1])
        sel = ok[ks]
        if sel.sum() < 3:
            continue
        ks, pos = ks[sel], pos[sel]
        cols = np.concatenate([b_ind[b_ip[k]:b_ip[k + 1]] for k in ks])
        u, cnt = np.unique(cols, return_counts=True)
        if not (cnt >= 3).any():
            continue
        h = u[np.argmax(cnt >= 3)]
        where = [(k, p) for k, p in zip(ks, pos) if h in b_ind[b_ip[k]:b_ip[k + 1]]][:3]
        for (k, p), v in zip(where, (BIG, BIG, -BIG)):
            ad[p] = 1.0
            bd[b_ip[k] + int(np.flatnonzero(b_ind[b_ip[k]:b_ip[k + 1]] == h)[0])] = v
            ok[k] = False
        planted += 1
        if planted == 2:
            break
    assert planted, "no C entry with three plantable terms"
    for r, v in zip(rng.choice(np.intersect1d(np.flatnonzero(ok & (np.diff(b_ip) > 0)), a_ind),
                               n_nonfinite, replace=False),
                    [np.nan, np.inf, -np.inf] * n_nonfinite):
        bd[b_ip[r] + int(rng.integers(0, b_ip[r + 1] - b_ip[r]))] = v
    return (a[0], a[1], ad), (b[0], b[1], bd)


# ---------------------------------------------------------------- bins, terms and reorders
def bins_of(O, a, ash, b, bsh, want):
    """Numeric bin of every C entry: 0 warp (nnz(C_i) <= 128), 1 hash map (<= 1024), 2 panels
    (<= 4096 A non-zeros), 3 hub rows; and the number of terms of every C entry."""
    _, nnzc, na = _row_stats(O, a, ash, b, bsh, want)
    row_bin = np.where(nnzc <= 128, 0, np.where(nnzc <= 1024, 1, np.where(na <= 4096, 2, 3)))
    ones = O.mul_csr_csr(ash, (a[0], a[1], np.ones(len(a[1]))), bsh,
                         (b[0], b[1], np.ones(len(b[1]))), threads=1)[2]
    return np.repeat(row_bin, nnzc), ones


def reordered(O, rng, a, ash, b, bsh):
    """The oracle's A P times P^T B for a random permutation P of the inner dimension: the same
    terms, summed in another order."""
    m = ash[1]
    perm = rng.permutation(m)
    inv = np.argsort(perm)
    a_ip = a[0].astype(np.int64)
    rows = np.repeat(np.arange(ash[0]), np.diff(a_ip))
    new_k = perm[a[1].astype(np.int64)]
    o = np.lexsort((new_k, rows))
    ap = (a[0], new_k[o].astype(np.uint32), a[2][o])
    b_ip = b[0].astype(np.int64)
    lens = np.diff(b_ip)[inv]
    bp_ip = np.zeros(m + 1, dtype=np.int64)
    np.cumsum(lens, out=bp_ip[1:])
    src = np.repeat(b_ip[:-1][inv] - bp_ip[:-1], lens) + np.arange(int(bp_ip[-1]))
    bp = (bp_ip.astype(np.uint32), b[1][src], b[2][src])
    return O.mul_csr_csr(ash, ap, bsh, bp, threads=1)


def check_case(sp, O, rng, built, want_bins, what, min_three=300, min_share=0.15):
    """Seam + sensitivity assertions on clean values, then the device product bit for bit on
    the scaled values with the edges planted."""
    a, ash, b, bsh, second = built
    ac, bc = realize(rng, a, b, second, scaled=True)
    want = O.mul_csr_csr(ash, ac, bsh, bc, threads=1)
    ebin, terms = bins_of(O, ac, ash, bc, bsh, want)
    other = reordered(O, rng, ac, ash, bc, bsh)
    assert np.array_equal(other[0], want[0]) and np.array_equal(other[1], want[1])
    for bn in want_bins:
        three = (ebin == bn) & (terms >= 3)
        assert three.sum() >= min_three, "%s: bin %d has %d entries of >= 3 terms" % (
            what, bn, three.sum())
        differ = other[2][three].view(np.uint64) != want[2][three].view(np.uint64)
        assert differ.mean() >= min_share, "%s: a reorder changes only %.2f of bin %d" % (
            what, differ.mean(), bn)
    # the device, on the scaled values with every edge planted
    a2, b2 = plant_edges(rng, ac, bc, second)
    want = O.mul_csr_csr(ash, a2, bsh, b2, threads=1)
    c = sp.CsMat.new(ash, *a2) * sp.CsMat.new(bsh, *b2)
    exact.assert_csr_bits((c.indptr, c.indices, np.zeros(len(c.data))),
                          (want[0], want[1], np.zeros(len(want[2]))), what + ": structure")
    exact.assert_same_class(c.data, want[2], what)
    assert np.isinf(want[2]).any() and np.isnan(want[2]).any(), what + ": edges not reached"
    return a2, ash, b2, bsh, want


# ---------------------------------------------------------------- one test per bin
def test_spgemm_bits_warp_bin(sp, O):
    rng = np.random.default_rng(101)
    units = [(int(rng.integers(0, 3)), int(rng.integers(2, 7))) for _ in range(500)]
    a, ash, b, bsh = spgemm_operands(rng, units, 100, rng.integers(0, 12, 500), 40, 10)
    check_case(sp, O, rng, (a, ash, b, bsh, _pairs_of_operands(b, 100)), [0], "warp bin")


@pytest.mark.parametrize("n_c", [129, 1024])
def test_spgemm_bits_hash_bin_ends(sp, O, n_c):
    """nnz(C_i) == 129 and == 1024: both ends of the CTA hash map."""
    rng = np.random.default_rng(n_c)
    lo, hi = (20, 60) if n_c < 500 else (60, 120)
    specs = [(n_c, int(rng.integers(30, 40)), int(rng.integers(lo, hi)), False) for _ in range(8)]
    built = designed(rng, specs, 50_000)
    a, ash, b, bsh, want = check_case(sp, O, rng, built, [1], "hash bin, %d entries" % n_c)
    _, nnzc, _ = _row_stats(O, a, ash, b, bsh, want)
    assert np.all(nnzc == n_c)


def test_spgemm_bits_hash_bin_many_terms(sp, O):
    """A hash-map row with far more A non-zeros than C entries: columns of hundreds of terms,
    long B rows (finished by the whole CTA) among short ones."""
    rng = np.random.default_rng(103)
    specs = [(150, 1500, 30, False), (300, 400, 200, False), (600, 200, 500, True)]
    a, ash, b, bsh, want = check_case(sp, O, rng, designed(rng, specs, 20_000), [1],
                                      "hash bin, many terms")
    nprod, nnzc, _ = _row_stats(O, a, ash, b, bsh, want)
    assert nprod[0] >= 200 * nnzc[0]


def _skip_middle_panel(rng, n, cols):
    lo = _columns(rng, n // 2, 16384)
    return np.concatenate([lo, 32768 + _columns(rng, n - n // 2, cols - 32768)])


@pytest.mark.parametrize("cols", [16384, 16385, 40_000])
def test_spgemm_bits_panel_kernel(sp, O, cols):
    """nnz(C_i) > 1024 with <= 4096 A non-zeros: 16384-column shared-memory panels, A rows of
    1, 2, 3, 16, 17 and 40 non-zeros; at 40000 columns half the B rows skip the middle panel."""
    rng = np.random.default_rng(cols + 7)
    b_lens = rng.integers(1100, 1600, 300)
    units = []
    for na in (1, 2, 3, 16, 17, 40):
        units += [(0, na), (na // 2, na - 2 * (na // 2))] * 2
    fn = (lambda r, n, c: _skip_middle_panel(r, n, c) if r.integers(0, 2) else _columns(r, n, c)) \
        if cols > 32768 else None
    a, ash, b, bsh = spgemm_operands(rng, units, 60, b_lens, cols, 50, b_cols_fn=fn)
    a, ash, b, bsh, want = check_case(sp, O, rng, (a, ash, b, bsh, _pairs_of_operands(b, 60)), [2],
                                      "panel kernel, %d columns" % cols)
    _, nnzc, na = _row_stats(O, a, ash, b, bsh, want)
    assert np.all(nnzc > 1024) and set(na.tolist()) >= {1, 2, 3, 16, 17, 40}


def test_spgemm_bits_panel_hot_column(sp, O):
    """Panel rows whose A non-zeros all hit one hot column (40 and 300 terms in it)."""
    rng = np.random.default_rng(105)
    specs = [(3000, 40, 1200, True), (5000, 300, 200, True), (2000, 64, 40, True)]
    a, ash, b, bsh, want = check_case(sp, O, rng, designed(rng, specs, 60_000), [2],
                                      "panel kernel, hot column")
    _, nnzc, na = _row_stats(O, a, ash, b, bsh, want)
    assert np.all(nnzc > 1024) and np.all(na <= 4096)


def _hub(sp, O, rng, n_hub, what):
    n_b, n_pairs, cols = 6000, 1500, 8000
    units = [(int(rng.integers(1100, 1500)), int(rng.integers(2000, 2900))) for _ in range(n_hub)]
    b_lens = rng.integers(1, 4, n_b)
    b_lens[2 * n_pairs:2 * n_pairs + 40] = 200  # long B rows: finished by the whole CTA
    a, ash, b, bsh = spgemm_operands(rng, units, n_pairs, b_lens, cols, 60)
    a, ash, b, bsh, want = check_case(sp, O, rng, (a, ash, b, bsh, _pairs_of_operands(b, n_pairs)),
                                      [3], what)
    _, nnzc, na = _row_stats(O, a, ash, b, bsh, want)
    assert np.all(na > 4096) and np.all(nnzc > 1024)


def test_spgemm_bits_hub_rows_few(sp, O):
    """Fewer hub rows (> 4096 A non-zeros) than SMs: the 1024-thread launch."""
    n = max(1, min(3, sp.Context.default().sm_count - 1))
    _hub(sp, O, np.random.default_rng(106), n, "%d hub rows" % n)


def test_spgemm_bits_hub_rows_many(sp, O):
    """More than 2 * sm_count hub rows: the 256-thread launch, CTAs taking a second row (NaN
    rows beside clean ones on one accumulator)."""
    n = 2 * sp.Context.default().sm_count + 5
    _hub(sp, O, np.random.default_rng(107), n, "%d hub rows" % n)


# ---------------------------------------------------------------- entry points
def _mixed_case(O, rng):
    """Rows in the warp, hash and panel bins, scaled values, edges planted."""
    specs = [(200, 40, 30, False), (1024, 30, 60, True), (2500, 20, 400, False),
             (60, 10, 20, False), (129, 30, 20, True)] * 2
    a, ash, b, bsh, second = designed(rng, specs, 30_000)
    a, b = realize(rng, a, b, second, scaled=True)
    a, b = plant_edges(rng, a, b, second, n_nonfinite=2)
    return a, ash, b, bsh


def _csc(O, shape, m):
    return O.convert_mat_storage(shape[0], shape[1], *m)


def _check(got, want, what):
    exact.assert_csr_bits((got[0], got[1], np.zeros(len(got[2]))),
                          (want[0], want[1], np.zeros(len(want[2]))), what + ": structure")
    exact.assert_same_class(got[2], want[2], what)


@pytest.mark.parametrize("storages", ["csr_csr", "csr_csc", "csc_csr", "csc_csc"])
def test_spgemm_bits_storage_combinations(sp, O, storages):
    """CsMat * CsMat in all four storages (csmat.rs:1930-1949): CSR x CSR; CSR x CSC converts B
    to CSR; CSC x CSC is the CSR product B^T A^T of the raw arrays, a CSC result; CSC x CSR
    converts B to CSC first."""
    rng = np.random.default_rng(108)
    a, ash, b, bsh = _mixed_case(O, rng)
    a_csc, b_csc = _csc(O, ash, a), _csc(O, bsh, b)
    sa, sb = storages.split("_")
    A = sp.CsMat.new(ash, *a) if sa == "csr" else sp.CsMat.new_csc(ash, *a_csc)
    B = sp.CsMat.new(bsh, *b) if sb == "csr" else sp.CsMat.new_csc(bsh, *b_csc)
    c = A * B
    if sa == "csr":
        want = O.mul_csr_csr(ash, a, bsh, b, threads=1)
        assert c.is_csr()
    else:  # C^T = B^T A^T on the CSC arrays (the CSR arrays of the transposes)
        want = O.mul_csr_csr((bsh[1], bsh[0]), b_csc, (ash[1], ash[0]), a_csc, threads=1)
        assert c.is_csc()
    _check((c.indptr, c.indices, c.data), want, "CsMat * CsMat, " + storages)


def test_spgemm_bits_csvec_times_csmat(sp, O):
    """&v * &A = row_view(v) * A (vec.rs:1084-1102), vectors long enough for the hash map and
    the panels."""
    rng = np.random.default_rng(109)
    m, p = 3000, 40_000
    b_lens = np.where(rng.random(m) < 0.05, rng.integers(100, 400, m), rng.integers(1, 12, m))
    b_ip = np.zeros(m + 1, dtype=np.int64)
    np.cumsum(b_lens, out=b_ip[1:])
    b_ind = np.concatenate([_columns(rng, int(n), p) for n in b_lens]).astype(np.uint32)
    bd = rng.standard_normal(int(b_ip[-1])) * np.repeat(np.exp2(rng.integers(-20, 21, m)), b_lens)
    b = (b_ip.astype(np.uint32), b_ind, bd)
    B = sp.CsMat.new((m, p), *b)
    seen = set()
    for nv, cap in ((60, 1024), (2000, None)):
        idx = np.sort(rng.choice(m, nv, replace=False))
        if cap:  # short B rows only: nnz(C) stays in the hash map
            idx = np.sort(rng.choice(np.flatnonzero(b_lens < 12), nv, replace=False))
        vd = rng.standard_normal(nv) * np.exp2(rng.integers(-20, 21, nv))
        vd[::17] = -0.0
        a = (np.array([0, nv], dtype=np.uint32), idx.astype(np.uint32), vd)
        want = O.mul_csr_csr((1, m), a, (m, p), b, threads=1)
        n = int(want[0][1])
        seen.add(0 if n <= 128 else 1 if n <= 1024 else 2)
        got = sp.CsVec(m, idx, vd) * B
        exact.assert_bits(got.indices.astype(np.float64), want[1].astype(np.float64), "indices")
        exact.assert_bits(got.data, want[2], "CsVec * CsMat, %d non-zeros" % nv)
    assert seen == {1, 2}


@pytest.mark.parametrize("idx", [np.uint32, np.uint64])
def test_spgemm_bits_smmp_index_widths(sp, O, idx):
    """smmp::mul_csr_csr with u32 and u64 indices (the device kernels see the same product)."""
    rng = np.random.default_rng(110)
    a, ash, b, bsh = _mixed_case(O, rng)
    A = sp.CsMat.new(ash, a[0].astype(idx), a[1].astype(idx), a[2])
    B = sp.CsMat.new(bsh, b[0].astype(idx), b[1].astype(idx), b[2])
    c = sp.smmp.mul_csr_csr(A, B)
    assert c.indices.dtype == idx
    _check((c.indptr, c.indices, c.data), O.mul_csr_csr(ash, a, bsh, b, threads=1),
           "smmp.mul_csr_csr, %s" % np.dtype(idx).name)


def test_spgemm_bits_numeric_dev_plan_twice(sp, O):
    """sprs_b200_spgemm_numeric_dev run twice on one symbolic plan: both results bit for bit."""
    rng = np.random.default_rng(111)
    a, ash, b, bsh = _mixed_case(O, rng)
    ctx = sp.Context.default()
    A, B = sp.CsMat.new(ash, *a), sp.CsMat.new(bsh, *b)
    want = O.mul_csr_csr(ash, a, bsh, b, threads=1)
    plan, nnz_c = C.c_void_p(), C.c_uint64()
    ctx.check(ctx.lib.sprs_b200_spgemm_symbolic(ctx.h, A.device().h, B.device().h, C.byref(plan),
                                                C.byref(nnz_c)))
    try:
        assert nnz_c.value == len(want[1])
        for run in range(2):
            cm = C.c_void_p()
            ctx.check(ctx.lib.sprs_b200_spgemm_numeric_dev(ctx.h, plan, C.byref(cm)))
            _check(sp.DeviceCsMat(ctx, cm).download(), want, "numeric_dev run %d" % run)
    finally:
        ctx.lib.sprs_b200_spgemm_free(plan)


# ---------------------------------------------------------------- full size
def test_spgemm_rmat_500k_bits_full_size(sp, O):
    """BASELINE config 4 (two 500k x 500k R-MAT) with the generator's N(0,1) values: the leading
    rows (the R-MAT hubs) and a block of ~1e8 products in the middle bit for bit against the
    oracle, reaching all four numeric bins between them; and two runs give the same digest of
    the whole C value array (C is 42 GB: two copies do not fit)."""
    import torch
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    n = 500_000
    A = G.rmat_csr(ctx, n, 16, seed=0x5EED0004)
    B = G.rmat_csr(ctx, n, 16, seed=0x5EED1004)
    aip = A.indptr.to(torch.int64) & 0xFFFFFFFF
    blen = (B.indptr[1:].to(torch.int64) & 0xFFFFFFFF) - (B.indptr[:-1].to(torch.int64) & 0xFFFFFFFF)
    csum = torch.cumsum(blen[A.indices.to(torch.int64) & 0xFFFFFFFF], 0)

    def prod_at(r):
        return int(csum[int(aip[r]) - 1].item()) if int(aip[r]) > 0 else 0

    def rows_for(r0, budget):
        k_end = int(torch.searchsorted(csum, torch.tensor([prod_at(r0) + budget], device=csum.device))[0])
        return min(n, int(torch.searchsorted(aip, torch.tensor([k_end], device=aip.device))[0]) + 1)

    blocks = [(0, rows_for(0, 100_000_000)), (n // 2, rows_for(n // 2, 100_000_000))]
    bh = B.to_host()

    def digest(cdat):
        h = torch.zeros((), dtype=torch.int64, device=cdat.device)
        bits = cdat.view(torch.int64)
        for s in range(0, bits.numel(), 1 << 26):
            e = min(bits.numel(), s + (1 << 26))
            w = torch.arange(s, e, dtype=torch.int64, device=cdat.device) * 0x1E3779B97F4A7C15 | 1
            h += (bits[s:e] * w).sum()
        return int(h.item())

    torch.cuda.empty_cache()
    cmir, cip, cind, cdat = G.spgemm(ctx, A, B)
    cip64 = cip.to(torch.int64)
    if cip.dtype == torch.int32:
        cip64 &= 0xFFFFFFFF
    nnzc = (cip64[1:] - cip64[:-1]).cpu().numpy()
    na = (aip[1:] - aip[:-1]).cpu().numpy()
    seen = set()
    for r0, r1 in blocks:
        want = O.mul_csr_csr((r1 - r0, n), A.slice_rows(r0, r1).to_host(), (n, n), bh, threads=0)
        s, e = int(cip64[r0]), int(cip64[r1])
        got = ((cip64[r0:r1 + 1] - s).cpu().numpy(), cind[s:e].cpu().numpy().view(np.uint32),
               cdat[s:e].cpu().numpy())
        exact.assert_csr_bits(got, want, "config 4 rows [%d, %d)" % (r0, r1))
        c, k = nnzc[r0:r1], na[r0:r1]
        seen |= set(np.where(c <= 128, 0, np.where(c <= 1024, 1, np.where(k <= 4096, 2, 3)))[c > 0].tolist())
    assert seen == {0, 1, 2, 3}, "bins reached: %s" % sorted(seen)
    d1 = digest(cdat)
    del cmir, cip, cind, cdat
    torch.cuda.empty_cache()
    cmir, cip, cind, cdat = G.spgemm(ctx, A, B)
    assert digest(cdat) == d1, "two runs of config 4 differ"
    del cmir, cip, cind, cdat
