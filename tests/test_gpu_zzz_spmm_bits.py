"""The row-major SpMM (csrc/spmm.cu) BIT FOR BIT with real-valued inputs, at its window, batch,
panel and grid-stride seams, and config 3 whole at full size.

The reference adds `out[i,:] += a_ij * B[j,:]` one non-zero after the other in storage order,
multiply and add rounded separately (prod.rs:189-214), so `O.csr_mulacc_dense_rowmaj` is the
exact bit reference.  The kernel keeps that order through four mechanisms, each a place where
another order could slip in:
  * a window of 32 (index, value) pairs read by the warp and broadcast by shuffle;
  * in the vector kernels, batches of U = 4 (k <= 64) or U = 2 (k > 64) non-zeros whose B rows
    are loaded before their products are added;
  * column panels of 32 / 64 (scalar) or 64 / 128 (vector) columns, each re-reading C;
  * a grid-stride loop over rows: one warp per row, at most sm_count * 64 CTAs of 8 warps, so
    P = sm_count * 512 rows per pass (2048 on the 4-SM emulator, 67584 on a 132-SM H100).
Values are N(0,1) * 2^k with k uniform in [-20, 20] for A, B and C0, where almost any
re-association moves a bit; tests/test_spmm_operands.py shows with host models that a batch
added in reverse or pre-summed, C added after the row's sum, or a window taken in reverse,
changes at least 15 % of the outputs of rows with three or more terms.

The seam matrix has n = 2P + 37 rows, so a warp takes up to three rows and the last pass is
partly filled.  Rows of SEAM_LENS terms sit in all three passes (every residue mod 4 and mod 2 in
the last batch; full and partial windows at 1, 2 and 3 windows); a warp's first row is empty and
its next a hub of 4097 terms; another hub sits in the last pass; rows whose every product is -0.0
test the sign of zero.  Each case asserts on the host, from its operands alone, that the seams it
claims are reached, and which kernel and panel split the launch picks (`kernel_of` restates
`spmm_rowmaj_launch`).

Small cases run on the CPU emulator too (tests/test_emu_preflight.py); `*_full_size` and
`*_child_process` ones need the H100."""
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np
import pytest

import exact
from conftest import ROOT

pytestmark = pytest.mark.gpu

# the launch shape of spmm_rowmaj_launch (tests/test_spmm_operands.py reads them from the source)
THREADS = 256           # SPMM_NT: 8 warps per CTA
CTAS_PER_SM = 64        # the grid cap, sm_count * 64 CTAs
WINDOW = 32             # pairs per shuffle window (kk += 32)
EMU_P = 4 * CTAS_PER_SM * THREADS // 32      # the emulator reports 4 SMs
H100_P = 132 * CTAS_PER_SM * THREADS // 32

KS = (1, 7, 31, 32, 33, 63, 64, 65, 66, 127, 128, 129, 130, 257)
SEAM_LENS = (0, 1, 2, 3, 4, 5, 31, 32, 33, 34, 35, 36, 37, 63, 64, 65, 96, 97)
HUB = 4097
BIG_HUB = 100_003
TAIL = 37               # rows of the last, partly filled pass: n = 2P + TAIL
SEAM_COLS = 4200
ZERO_COLS = 40          # the last ZERO_COLS rows of B are +0.0
NEGZERO_LENS = (1, 5, 37)
# warps (rows of the first pass) of the special rows; the same warp takes row w + P, w + 2P
SEAM_WARP0 = 1          # warps 1 .. len(SEAM_LENS)
EMPTY_HUB_WARP = 20     # row 20 empty, row P + 20 a hub
LATE_HUB_WARP = 22      # row 2P + 22 a hub
NEGZERO_WARP0 = 24      # warps 24 .. 26 in every pass: products all -0.0
LAST_ROW_LEN = 65
FILL_MAX = 5            # filler rows have 0 to FILL_MAX terms

NAN_A = np.array([0x7FF8000000000123], np.uint64).view(np.float64)[0]
NAN_B = np.array([0xFFF80000DEADBEEF], np.uint64).view(np.float64)[0]
SPECIALS = (-0.0, np.inf, -np.inf, NAN_A, NAN_B)


@pytest.fixture(scope="module")
def sp():
    import sprs_b200
    sprs_b200.Context.default()  # raises without a GPU / without the .so: no fallback
    return sprs_b200


@pytest.fixture(scope="module")
def O():
    from oracle import oracle
    return oracle


def pass_rows(sm_count):
    """Rows of one grid pass: the warps of the largest launch."""
    return sm_count * CTAS_PER_SM * (THREADS // 32)


@pytest.fixture(scope="module")
def P(sp):
    return pass_rows(sp.Context.default().sm_count)


def real_values(rng, shape):
    n = int(np.prod(shape))
    return (rng.standard_normal(n) * np.exp2(rng.integers(-20, 21, n))).reshape(shape)


# ---------------------------------------------------------------- the launch, restated
def kernel_of(k, ldb, ldc, pb, pc):
    """spmm_rowmaj_launch's choice: (name, panel width, U) -- the 128-bit flavour iff k, ldb and
    ldc are even and B and C are 16-byte aligned; 4-deep batches up to k = 64; the scalar
    kernel has one column per lane up to k = 32, else two."""
    if k % 2 == 0 and ldb % 2 == 0 and ldc % 2 == 0 and ((pb | pc) & 15) == 0:
        return ("vec_u4", 64, 4) if k <= 64 else ("vec_u2", 128, 2)
    return ("scalar_32", 32, 1) if k <= 32 else ("scalar_64", 64, 1)


def panels_of(k, width):
    """(panel count, columns of the last panel)."""
    n = -(-k // width)
    return n, k - width * (n - 1)


def host_kernel(k):
    """The host-buffer route stages B and C contiguously in device scratch (256-byte aligned):
    ld = k, so an even k always takes the vector kernel."""
    return kernel_of(k, k, k, 0, 0)


# dev layouts (ld - k, offset of B and C in elements): even k reaches both flavours
EVEN_LAYOUTS = ((0, 0), (0, 1), (1, 0), (2, 0))
ODD_LAYOUTS = ((0, 0), (3, 1))


def dev_cases():
    return [(k, e, o) for k in KS for e, o in (EVEN_LAYOUTS if k % 2 == 0 else ODD_LAYOUTS)]


def claimed_kernel(k, ld_extra, off):
    """What a dev layout must take, given 16-byte aligned allocations."""
    return kernel_of(k, k + ld_extra, k + ld_extra, 8 * off, 8 * off)


# ---------------------------------------------------------------- operands
def seam_lens(P, rng):
    """Row lengths of the seam matrix and each row's role (0 filler, 1 seam, 2 hub, 3 -0.0)."""
    n = 2 * P + TAIL
    lens = rng.integers(0, FILL_MAX + 1, n)
    role = np.zeros(n, np.int8)
    m = len(SEAM_LENS)
    for p in range(3):
        for j in range(m):  # each warp sees different lengths in its three passes
            r = p * P + SEAM_WARP0 + j
            lens[r], role[r] = SEAM_LENS[(j + 5 * p) % m], 1
        for j, L in enumerate(NEGZERO_LENS):
            r = p * P + NEGZERO_WARP0 + j
            lens[r], role[r] = L, 3
    lens[EMPTY_HUB_WARP], role[EMPTY_HUB_WARP] = 0, 1
    lens[P + EMPTY_HUB_WARP], role[P + EMPTY_HUB_WARP] = HUB, 2
    lens[2 * P + LATE_HUB_WARP], role[2 * P + LATE_HUB_WARP] = HUB, 2
    lens[n - 1], role[n - 1] = LAST_ROW_LEN, 1
    return lens, role


def build_rows(rng, lens, role, cols, zero_cols):
    """CSR arrays for the given lengths: filler rows (at most FILL_MAX terms) draw ascending
    columns in one vectorised pass, the other rows distinct sorted columns; -0.0 rows (role 3)
    take only the zero columns of B, with negative values."""
    n = lens.size
    ip = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=ip[1:])
    ind = np.empty(int(ip[-1]), np.int64)
    free = cols - zero_cols
    fill = np.flatnonzero((role == 0) & (lens > 0))
    assert lens[fill].max(initial=0) <= FILL_MAX
    c0 = rng.integers(0, free - 50 * FILL_MAX, fill.size)
    steps = np.cumsum(rng.integers(1, 50, (fill.size, FILL_MAX)), axis=1)
    for t in range(FILL_MAX):
        sel = lens[fill] > t
        ind[ip[fill[sel]] + t] = c0[sel] + steps[sel, t]
    for r in np.flatnonzero((role != 0) & (lens > 0)):
        L = int(lens[r])
        if role[r] == 3:
            ind[ip[r]:ip[r + 1]] = free + np.sort(rng.choice(zero_cols, L, replace=False))
        else:
            ind[ip[r]:ip[r + 1]] = np.sort(rng.choice(free, L, replace=False))
    data = real_values(rng, ind.size)
    neg = np.repeat(role == 3, lens)
    data[neg] = -np.abs(data[neg])
    return ip.astype(np.uint32), ind.astype(np.uint32), data


class Case:
    def __init__(self, P, lens, role, ip, ind, data, cols, zero_cols):
        self.P, self.lens, self.role = P, lens, role
        self.ip, self.ind, self.data = ip, ind, data
        self.n, self.cols, self.zero_cols = lens.size, cols, zero_cols

    def b(self, rng, k):
        """B with real values and its last zero_cols rows +0.0."""
        b = real_values(rng, (self.cols, k))
        b[self.cols - self.zero_cols:] = 0.0
        return b

    def oracle(self, O, b, c0):
        return O.csr_mulacc_dense_rowmaj(self.ip, self.ind, self.data, b, c0.copy())


def seam_case(P, seed=1):
    rng = np.random.default_rng(seed)
    lens, role = seam_lens(P, rng)
    return Case(P, lens, role, *build_rows(rng, lens, role, SEAM_COLS, ZERO_COLS), SEAM_COLS,
                ZERO_COLS)


def hub_case(P, seed=2):
    """P + 8 rows of 0 to 3 terms; warp 5's first row is empty and its second a hub of
    BIG_HUB terms; row 6 a hub of HUB terms."""
    rng = np.random.default_rng(seed)
    n = P + 8
    lens, role = rng.integers(0, 4, n), np.zeros(n, np.int8)
    lens[5], role[5] = 0, 1
    lens[P + 5], role[P + 5] = BIG_HUB, 2
    lens[6], role[6] = HUB, 2
    cols = BIG_HUB + 61
    return Case(P, lens, role, *build_rows(rng, lens, role, cols, 0), cols, 0)


def window_shape(L):
    """(windows, entries of the last window) of a row of L > 0 terms."""
    w = -(-L // WINDOW)
    return w, L - WINDOW * (w - 1)


def assert_seam_case(case):
    """Everything the seam cases claim, from the operands alone."""
    P, lens, role, n = case.P, case.lens, case.role, case.n
    assert n == 2 * P + TAIL and n // P == 2 and n % P == TAIL
    passes = np.arange(n) // P
    # every seam length in every pass of a warp
    for L in SEAM_LENS:
        got = set(passes[(lens == L) & (role == 1)].tolist())
        assert got == {0, 1, 2}, (L, got)
    # the last window's length takes every residue mod 4 (and mod 2) in windows 1 and 2, and
    # rows end on full and on partial windows at 1, 2 and 3 windows
    shapes = {window_shape(L) for L in SEAM_LENS if L}
    for w in (1, 2):
        assert {r % 4 for ww, r in shapes if ww == w} == {0, 1, 2, 3}, w
    for w in (1, 2, 3):
        assert (w, WINDOW) in shapes and (w + 1, 1) in shapes, w
    # a warp whose first row is empty and whose second a hub; a hub in the last pass
    assert lens[EMPTY_HUB_WARP] == 0 and lens[P + EMPTY_HUB_WARP] == HUB
    assert lens[2 * P + LATE_HUB_WARP] == HUB and passes[2 * P + LATE_HUB_WARP] == 2
    assert HUB % WINDOW == 1 and HUB % 4 == 1
    # the last row of the matrix is in the partly filled third pass, non-empty
    assert lens[n - 1] == LAST_ROW_LEN and (n - 1) % P < TAIL
    # the -0.0 rows take only zero B rows, with negative values, in every pass
    ip = case.ip.astype(np.int64)
    for r in np.flatnonzero(role == 3):
        cols = case.ind[ip[r]:ip[r + 1]]
        assert cols.size and cols.min() >= case.cols - case.zero_cols
        assert np.all(case.data[ip[r]:ip[r + 1]] < 0)
    assert set(passes[role == 3].tolist()) == {0, 1, 2}
    # columns distinct and ascending per row
    rows = np.repeat(np.arange(n), lens)
    same = rows[1:] == rows[:-1]
    assert np.all(case.ind[1:][same].astype(np.int64) > case.ind[:-1][same])


@pytest.fixture(scope="module")
def seam(P):
    case = seam_case(P)
    assert_seam_case(case)
    return case


@pytest.fixture(scope="module")
def seam_mat(sp, seam):
    return sp.CsMat.new((seam.n, seam.cols), seam.ip, seam.ind, seam.data)


# ---------------------------------------------------------------- runs
def dev_run(sp, a, b, c0, ld_extra, off, acc, sentinel=-7.25, guard=5):
    """sprs_b200_spmm_rowmaj_dev on torch tensors with ld = k + ld_extra and B / C starting `off`
    elements into their buffers.  B's padding is NaN, so a read of it would poison the result;
    C's padding and guard elements hold a sentinel that must survive.  Returns (C, kernel)."""
    import torch
    from sprs_b200 import generate as G
    rows, k = c0.shape
    cols = b.shape[0]
    ctx = a.context()
    dev = G._device(ctx)
    ldb = ldc = k + ld_extra
    bb = np.full(off + cols * ldb + guard, np.nan)
    bb[off:off + cols * ldb].reshape(cols, ldb)[:, :k] = b
    cc = np.full(off + rows * ldc + guard, sentinel)
    cc[off:off + rows * ldc].reshape(rows, ldc)[:, :k] = c0
    bt, ct = torch.from_numpy(bb).to(dev), torch.from_numpy(cc).to(dev)
    pb, pc = bt.data_ptr() + 8 * off, ct.data_ptr() + 8 * off
    G._sync()
    ctx.check(ctx.lib.sprs_b200_spmm_rowmaj_dev(ctx.h, a.device().h, C.c_void_p(pb), ldb, k,
                                                C.c_void_p(pc), ldc, acc, G._stream_ptr()))
    ctx.synchronize()
    G._sync()
    out = ct.cpu().numpy()
    what = "k=%d ld=%d offset=%d accumulate=%d" % (k, ldb, off, acc)
    body = out[off:off + rows * ldc].reshape(rows, ldc)
    assert np.all(body[:, k:] == sentinel), what + ": padding columns written"
    assert np.all(out[:off] == sentinel) and np.all(out[off + rows * ldc:] == sentinel), \
        what + ": guard elements written"
    return body[:, :k].copy(), kernel_of(k, ldb, ldc, pb, pc)


def indptr_bytes(a):
    ctx = a.context()
    ip, w, ind, d = C.c_void_p(), C.c_int(), C.c_void_p(), C.c_void_p()
    ctx.check(ctx.lib.sprs_b200_csmat_device_arrays(a.device().h, C.byref(ip), C.byref(w),
                                                    C.byref(ind), C.byref(d)))
    return w.value


# ================================================================ tests
def test_spmm_indptr_width(sp, seam_mat):
    """The seam matrix runs the 32-bit indptr instantiations, or with SPRS_B200_FORCE_INDPTR64=1
    (test_spmm_bits_indptr64_child_process) the 64-bit ones."""
    force = os.environ.get("SPRS_B200_FORCE_INDPTR64") == "1"
    assert indptr_bytes(seam_mat) == (8 if force else 4)


@pytest.mark.parametrize("k", KS)
def test_spmm_host_seams_bits(sp, O, seam, seam_mat, k):
    """prod.csr_mulacc_dense_rowmaj from a random C0 (always accumulating: even k takes the
    vector kernel), and `a * b` from zero for k >= 8."""
    rng = np.random.default_rng(100 + k)
    b = seam.b(rng, k)
    c0 = real_values(rng, (seam.n, k))
    got = c0.copy()
    sp.prod.csr_mulacc_dense_rowmaj(seam_mat, b, got)
    name = host_kernel(k)[0]
    exact.assert_bits(got, seam.oracle(O, b, c0), "host %s k=%d" % (name, k))
    if k >= 8:
        exact.assert_bits(seam_mat * b, seam.oracle(O, b, np.zeros((seam.n, k))),
                          "a * b %s k=%d" % (name, k))


@pytest.mark.parametrize("k,ld_extra,off", dev_cases())
def test_spmm_dev_seams_bits(sp, O, seam, seam_mat, k, ld_extra, off):
    """sprs_b200_spmm_rowmaj_dev, plain (C overwritten: empty rows +0.0, the -0.0 rows +0.0) and
    accumulating onto a random C0."""
    rng = np.random.default_rng(200 + 7 * k + 3 * ld_extra + off)
    b = seam.b(rng, k)
    c0 = real_values(rng, (seam.n, k))
    empty = seam.lens == 0
    negzero = seam.role == 3
    for acc in (0, 1):
        got, kern = dev_run(sp, seam_mat, b, c0, ld_extra, off, acc)
        assert kern == claimed_kernel(k, ld_extra, off), (kern, k, ld_extra, off)
        want = seam.oracle(O, b, c0 if acc else np.zeros((seam.n, k)))
        if not acc:  # the seams of a plain run, in the oracle's bits
            assert np.all(want[empty].view(np.uint64) == 0)
            assert np.all(want[negzero].view(np.uint64) == 0)
        exact.assert_bits(got, want, "dev %s k=%d ld=%d offset=%d accumulate=%d"
                          % (kern[0], k, k + ld_extra, off, acc))


SPECIAL_CASES = [(31, "host", 0, 0), (64, "host", 0, 0), (64, "dev", 0, 1), (130, "dev", 0, 0),
                 (130, "dev", 3, 1)]


def special_c0(rng, case, k):
    """C0 with -0.0, +-inf and two NaN payloads: every entry of the empty rows cycles through
    them, 5 % of the other entries hold one, and the -0.0 rows are -0.0 throughout."""
    c0 = real_values(rng, (case.n, k))
    empty = case.lens == 0
    cyc = np.resize(np.array(SPECIALS), (int(empty.sum()), k))
    c0[empty] = np.roll(cyc, rng.integers(0, len(SPECIALS)), axis=1)
    hit = (rng.random((case.n, k)) < 0.05) & ~empty[:, None]
    c0[hit] = np.array(SPECIALS)[rng.integers(0, len(SPECIALS), int(hit.sum()))]
    c0[case.role == 3] = -0.0
    return c0


@pytest.mark.parametrize("k,route,ld_extra,off", SPECIAL_CASES)
def test_spmm_special_c_bits(sp, O, seam, seam_mat, k, route, ld_extra, off):
    """Accumulating onto a C0 with -0.0, +-inf and NaN payloads 0x7FF8000000000123 and
    0xFFF80000DEADBEEF: empty rows hand C0 back bit for bit (payloads included); the other rows
    match the oracle with NaN by class (whether the hardware's add keeps a payload is not
    assumed); -0.0 products onto -0.0 stay -0.0."""
    rng = np.random.default_rng(300 + k + off)
    b = seam.b(rng, k)
    c0 = special_c0(rng, seam, k)
    if route == "host":
        got = c0.copy()
        sp.prod.csr_mulacc_dense_rowmaj(seam_mat, b, got)
        kern = host_kernel(k)
    else:
        got, kern = dev_run(sp, seam_mat, b, c0, ld_extra, off, 1)
    assert kern == (host_kernel(k) if route == "host" else claimed_kernel(k, ld_extra, off))
    want = seam.oracle(O, b, c0)
    empty, negzero = seam.lens == 0, seam.role == 3
    what = "%s %s k=%d" % (route, kern[0], k)
    for rows in (empty, ~empty & ~negzero):  # every special, payloads included, in both kinds
        held = c0[rows].view(np.uint64)
        assert all((held == x).any() for x in np.array(SPECIALS).view(np.uint64))
    assert np.all(np.signbit(want[negzero]) & (want[negzero] == 0))
    exact.assert_bits(got[empty], c0[empty], what + ": empty rows")
    exact.assert_same_class(got, want, what)


@pytest.mark.parametrize("k", [8, 33, 130])
def test_spmm_hub_rows_bits(sp, O, P, k):
    """prod.csr_mulacc_dense_rowmaj with a hub of 100003 terms as a warp's second row (its first
    is empty) and one of 4097: the 4-deep vector batch, the 64-column scalar kernel and two
    panels of the 2-deep vector batch."""
    case = hub_case(P)
    assert case.lens[5] == 0 and case.lens[P + 5] == BIG_HUB and 5 < P
    a = sp.CsMat.new((case.n, case.cols), case.ip, case.ind, case.data)
    rng = np.random.default_rng(400 + k)
    b = case.b(rng, k)
    c0 = real_values(rng, (case.n, k))
    got = c0.copy()
    sp.prod.csr_mulacc_dense_rowmaj(a, b, got)
    kern = host_kernel(k)
    assert kern[0] == {8: "vec_u4", 33: "scalar_64", 130: "vec_u2"}[k]
    exact.assert_bits(got, case.oracle(O, b, c0), "hub rows %s k=%d" % (kern[0], k))


# ---------------------------------------------------------------- 64-bit indptr
def test_spmm_bits_indptr64_child_process():
    """This file's small cases again with SPRS_B200_FORCE_INDPTR64=1 (read once per process):
    the four kernels' 64-bit indptr instantiations."""
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu",
                        os.path.abspath(__file__), "-k", "not full_size and not child_process"],
                       capture_output=True, text=True, timeout=1500, cwd=ROOT,
                       env=dict(os.environ, SPRS_B200_FORCE_INDPTR64="1"))
    tail = "\n".join(r.stdout.splitlines()[-15:])
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail, \
        tail + r.stderr[-2000:]


# ---------------------------------------------------------------- full size (H100)
def whole_check(O, a, b, c0, acc, what):
    """C of a DeviceCsr times b (+ c0), whole, against the oracle (single thread, timed)."""
    import torch
    from sprs_b200 import generate as G
    ctx = a.ctx
    dev = G._device(ctx)
    bt = torch.from_numpy(b).to(dev)
    ct = torch.from_numpy(c0).to(dev) if acc else \
        torch.full(c0.shape, float("nan"), dtype=torch.float64, device=dev)
    G.spmm_rowmaj(ctx, a, bt, ct, accumulate=acc)
    G._sync()
    got = ct.cpu().numpy()
    del bt, ct
    ip, ind, d = a.to_host()
    want = c0.copy() if acc else np.zeros_like(c0)
    t = time.perf_counter()
    O.csr_mulacc_dense_rowmaj(ip, ind, d, b, want)
    dt = time.perf_counter() - t
    print("%s: oracle %.1f s for %.3g multiply-adds" % (what, dt, float(ind.size) * b.shape[1]))
    exact.assert_bits(got, want, what)


def test_spmm_config3_full_size(sp, O):
    """BASELINE config 3 (1M x 1M sprs-rand, 32 per row) times a 1M x 64 B: the whole C, from
    zero (C filled with NaN first: it must be overwritten) and accumulating onto a random C0."""
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    a = G.rand_csr(ctx, 1_000_000, 1_000_000, 32, seed=0x5EED0002)
    assert a.nnz == 32_000_000
    rng = np.random.default_rng(500)
    b = real_values(rng, (a.cols, 64))
    c0 = real_values(rng, (a.rows, 64))
    whole_check(O, a, b, c0, False, "config 3 k=64 from zero")
    whole_check(O, a, b, c0, True, "config 3 k=64 accumulating")


def test_spmm_rmat_full_size(sp, O):
    """BASELINE config 4's R-MAT (500k, 16 per row, hub rows) times B for k = 8 / 33 / 130,
    accumulating onto a random C0: the 4-deep vector batch, the 64-column scalar kernel and two
    panels of the 2-deep vector batch."""
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    a = G.rmat_csr(ctx, 500_000, 16, seed=0x5EED0004)
    lens = np.diff(a.indptr.cpu().numpy().view(np.uint32).astype(np.int64))
    assert lens.max() > 1000
    rng = np.random.default_rng(600)
    for k in (8, 33, 130):
        b = real_values(rng, (a.cols, k))
        c0 = real_values(rng, (a.rows, k))
        whole_check(O, a, b, c0, True, "config 4 R-MAT k=%d" % k)
