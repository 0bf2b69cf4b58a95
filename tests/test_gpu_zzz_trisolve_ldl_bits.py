"""The triangular solves (csrc/trisolve.cu) and the LDL^T factorization (csrc/ldl.cu) BIT FOR BIT
with real-valued data, across ticket waves, at their group seams and at full size.

Both kernels run one warp per row, claim rows through a ticket counter and order them with
acquire / release flags; at most sm_count * 8 CTAs of 8 warps run, so a warp takes a second row
only past W = sm_count * 64 tickets (8448 on an H100, 256 on the 4-SM emulator).  Every case here
is sized from W and asserts on the host, from the matrix and the oracles alone, that the seam it
claims is reached: tickets past W, the term count of each group-seam row, the hub rows' term
counts around TRI_HEARTBEAT, the singular ticket, the pattern and column-prefix lengths of the
factor's rows.  Values are N(0,1) * 2^k with k uniform in [-20, 20] on a dominant diagonal
(symmetric for LDL^T), so almost any re-association of a sum moves a bit; the host models of
tests/test_trisolve_ldl_operands.py show that another order of the same terms changes at least
15 % of the rows of three or more terms.

- Trisolve, the four forms: n in {W - 1, W, W + 1, 3W + 5} with row r depending on r - 1 and on
  r - W (the upper forms mirrored); rows of 31 / 32 / 33 / 63 / 64 / 65 / 95 / 96 / 97 terms in
  the solved triangle in both waves, with entries of the other triangle that the kernel ignores;
  hub rows of 8191 / 8192 / 8193 / 16385 terms claimed last; singular at ticket W + 3 and at the
  last ticket (missing, 0.0, -0.0: index, reason and the whole partial rhs, the CSC forms' partial
  sums included); the 2-D Laplacian with random values; `ldl_lsolve` / `ldl_ltsolve` with
  columns of more than 32 entries; two plans of one matrix on two streams at once.
- LDL^T, CSR and CSC, the identity and scrambled permutations: a band of half-bandwidth 40 at
  n in {W - 1, W + 1, 3W + 5}; the 2-D and 3-D nested-dissection Laplacian patterns; pattern and prefix
  lengths of 31 / 32 / 33 / 63 / 64 / 65 past the first wave; input rows longer than 32 with the
  diagonal in different lanes; `DontCheckSymmetry` on a non-symmetric matrix of W + 1 rows; a
  zero pivot past the first wave and the update after it; factor / solve_dev / update repeated.
  A scrambled permutation stores the matrix as Q A Q^T and factors it with perm = Q: the factor
  has A's structure, but each row's entries come in another stored order.  Where the
  elimination tree branches (the nested-dissection cases, the arrows' hubs) that order decides
  the order of the row's pattern steps; a band or a dense block has a chain for a tree, whose
  only topological order is ascending, so there the steps are ascending whatever the storage.

Small cases run on the CPU emulator too (tests/test_emu_trisolve_ldl_bits.py); `*_full_size`
and `*_child_process` ones need the H100, and `*_streams` needs CUDA streams."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sps

import ldl_oracle as LO
import test_gpu_ldl as TL
import test_gpu_trisolve as TT
import trisolve_oracle as TO
from conftest import ROOT

pytestmark = pytest.mark.gpu

if os.environ.get("SPRS_B200_EMU_LDL_LIB"):  # test infrastructure: the emulated build with the
    import sprs_b200 as _sp                  # solves and the factorization (tests/emu_ldl.py)
    _sp._lib.LIB_PATH = os.environ["SPRS_B200_EMU_LDL_LIB"]

# the kernels' launch shapes (tests/test_trisolve_ldl_operands.py reads them from the sources)
THREADS = 256            # TRI_THREADS, LDL_THREADS
CTAS_PER_SM = 8          # TRI_CTAS_PER_SM, LDL_CTAS_PER_SM
GROUP = 32               # terms of a trisolve group; entries per LDL loop step
HEARTBEAT = 8192         # TRI_HEARTBEAT
EMU_W = 4 * CTAS_PER_SM * THREADS // 32    # the emulator reports 4 SMs
H100_W = 132 * CTAS_PER_SM * THREADS // 32
GROUP_LENS = (31, 32, 33, 63, 64, 65, 95, 96, 97)
HUB_LENS = (8191, 8192, 8193, 16385)
SEAM_LENS = (31, 32, 33, 63, 64, 65)
LATE = 3                 # the singular ticket W + LATE
BAND = 40


def wave_of(sm_count):
    """Warps of the largest launch: the tickets of the first wave."""
    return sm_count * CTAS_PER_SM * (THREADS // 32)


@pytest.fixture(scope="module")
def sp():
    import sprs_b200
    lib = sprs_b200._lib.load()  # the product library must export the solves and the factor
    if os.path.basename(sprs_b200._lib.LIB_PATH).startswith("libsprs_b200_emu") and \
            not hasattr(lib, "sprs_b200_ldl_symbolic"):
        pytest.skip("the emulated build of tests/emu has neither: tests/test_emu_trisolve_ldl_"
                    "bits.py runs this file on one that has")
    return sprs_b200


@pytest.fixture(scope="module")
def W(sp):
    return wave_of(sp.Context.default().sm_count)


def real_values(rng, n):
    return rng.standard_normal(n) * np.exp2(rng.integers(-20, 21, n))


# ---------------------------------------------------------------- trisolve operands
def tri_matrix(rng, n, t_rows, t_cols, upper, diag=True):
    """n x n CSR from off-diagonal entries given in TICKET space (ticket t is row t of a lower
    solve, row n - 1 - t of an upper one, so one construction serves both triangles): real
    values, duplicates dropped, and a diagonal 1 + sum |row| unless diag is False."""
    t_rows, t_cols = np.asarray(t_rows, np.int64), np.asarray(t_cols, np.int64)
    keep = t_rows != t_cols
    key = np.unique(t_rows[keep] * n + t_cols[keep])
    r, c = key // n, key % n
    if upper:
        r, c = n - 1 - r, n - 1 - c
    m = sps.csr_matrix((real_values(rng, key.size), (r, c)), shape=(n, n))
    if diag:
        m = sps.csr_matrix(m + sps.diags(1.0 + np.asarray(abs(m).sum(axis=1)).ravel()))
    m.sort_indices()
    return m


def random_entries(rng, n, per_side, skip=()):
    """per_side entries before and after each ticket (not for the tickets in skip)."""
    t = np.setdiff1d(np.arange(n), np.asarray(skip, np.int64))
    t = np.repeat(t, per_side)
    lo = (rng.random(t.size) * t).astype(np.int64)
    hi = t + 1 + (rng.random(t.size) * (n - 1 - t)).astype(np.int64)
    ok_lo, ok_hi = t > 0, t < n - 1
    return (np.concatenate([t[ok_lo], t[ok_hi]]), np.concatenate([lo[ok_lo], hi[ok_hi]]))


def wave_case(rng, n, W, upper):
    """Ticket t depends on t - 1 and t - W, plus three random earlier tickets; three entries of
    the other triangle per row."""
    t = np.arange(n)
    r0, c0 = random_entries(rng, n, 3)
    rows = np.concatenate([t[1:], t[W:], r0])
    cols = np.concatenate([t[:-1], t[:-W] if W < n else t[:0], c0])
    return tri_matrix(rng, n, rows, cols, upper)


def group_tickets(W):
    """(ticket, terms) of the group-seam rows: one set in the first wave, one past it."""
    return [(100 + 11 * j, L) for j, L in enumerate(GROUP_LENS)] + \
           [(W + 50 + 11 * j, L) for j, L in enumerate(GROUP_LENS)]


def group_case(rng, W, upper):
    """n = 3W + 5; the group-seam rows have exactly L terms in the solved triangle (always the
    ticket just before them) and 0 to 39 entries of the other triangle, so their diagonal sits at
    different positions of the stored row."""
    n = 3 * W + 5
    special = group_tickets(W)
    r0, c0 = random_entries(rng, n, 3, skip=[t for t, _ in special])
    rows, cols = [r0], [c0]
    for t, L in special:
        before = np.concatenate([[t - 1], rng.choice(t - 1, L - 1, replace=False)])
        after = t + 1 + rng.choice(n - 1 - t, int(rng.integers(0, 40)), replace=False)
        rows.append(np.full(L + after.size, t))
        cols.append(np.concatenate([before, after]))
    return tri_matrix(rng, n, np.concatenate(rows), np.concatenate(cols), upper)


def hub_n(W):
    return HUB_LENS[-1] + 2 * W + 8


def hub_case(rng, W, upper):
    """Hub rows of HUB_LENS terms at the last tickets, claimed after every other row: each reads
    the five tickets before it, still pending when it starts, and the other hubs' columns lie in
    its other triangle."""
    n = hub_n(W)
    hubs = [(n - len(HUB_LENS) + j, L) for j, L in enumerate(HUB_LENS)]
    r0, c0 = random_entries(rng, n, 3, skip=[t for t, _ in hubs])
    rows, cols = [r0], [c0]
    for t, L in hubs:
        near = np.arange(t - 5, t)
        far = rng.choice(t - 5, L - near.size, replace=False)
        after = np.arange(t + 1, n)
        rows.append(np.full(L + after.size, t))
        cols.append(np.concatenate([near, far, after]))
    return tri_matrix(rng, n, np.concatenate(rows), np.concatenate(cols), upper)


def singular_case(rng, W, upper, kind, at):
    """The wave case at n = 3W + 5, singular at ticket `at`: its diagonal missing, 0.0 or -0.0."""
    n = 3 * W + 5
    m = wave_case(rng, n, W, upper)
    r = n - 1 - at if upper else at
    j = m.indptr[r] + np.flatnonzero(m.indices[m.indptr[r]:m.indptr[r + 1]] == r)[0]
    if kind == "missing":
        m = m.tolil()
        m[r, r] = 0.0
        m = sps.csr_matrix(m)
        m.eliminate_zeros()
    else:
        m.data[j] = 0.0 if kind == "zero" else -0.0
    m.sort_indices()
    return m


def lap2d_case(rng, side):
    """The 5-point Laplacian pattern of a side x side grid with real values on a dominant
    diagonal (both triangles stored: the kernel reads only the one it solves)."""
    n = side * side
    t = np.arange(n)
    right = t[(t % side) < side - 1]
    down = t[t < n - side]
    rows = np.concatenate([right + 1, down + side])
    cols = np.concatenate([right, down])
    rows, cols = np.concatenate([rows, cols]), np.concatenate([cols, rows])
    return tri_matrix(rng, n, rows, cols, False)


def csr_of(m, form):
    """The rows the kernel solves (a CSC matrix is solved on its CSR, the same matrix)."""
    return TT.as_storage(m, "lsolve_csr")


def tri_terms(m, form):
    """Per row: the number of terms of the solved triangle."""
    c = csr_of(m, form)
    rows = np.repeat(np.arange(c.shape[0]), np.diff(c.indptr))
    sel = c.indices < rows if form.startswith("l") else c.indices > rows
    return np.bincount(rows[sel], minlength=c.shape[0])


def ticket_row(n, t, form):
    return n - 1 - t if form.startswith("u") else t


def tri_seams(m, form, W):
    """What a case reaches, from the matrix alone: rows past the first wave, the term count of
    every row, the rows of three or more terms, the diagonal's position in each stored row."""
    n = m.shape[0]
    c = csr_of(m, form)
    rows = np.repeat(np.arange(n), np.diff(c.indptr))
    below = np.bincount(rows[c.indices < rows], minlength=n)
    terms = tri_terms(m, form)
    return {"late": max(0, n - W), "terms": terms, "three": int(np.count_nonzero(terms >= 3)),
            "diag_pos": below}


def assert_wave_seams(m, form, W):
    n = m.shape[0]
    s = tri_seams(m, form, W)
    assert s["late"] == max(0, n - W)
    c = csr_of(m, form)
    for t in range(1, n):  # every ticket reads the one before it, and the one a wave before it
        r = ticket_row(n, t, form)
        need = [ticket_row(n, t - 1, form)] + ([ticket_row(n, t - W, form)] if t >= W else [])
        assert np.isin(need, c.indices[c.indptr[r]:c.indptr[r + 1]]).all()
    return s


def assert_group_seams(m, form, W):
    n = m.shape[0]
    s = tri_seams(m, form, W)
    pos = []
    for t, L in group_tickets(W):
        r = ticket_row(n, t, form)
        assert s["terms"][r] == L, (t, L, s["terms"][r])
        pos.append(s["diag_pos"][r])
    assert sum(t >= W for t, _ in group_tickets(W)) == len(GROUP_LENS)
    assert len(set(pos)) >= 8  # the diagonal at many positions of the stored rows
    return s


def assert_hub_seams(m, form, W):
    n = m.shape[0]
    s = tri_seams(m, form, W)
    for j, L in enumerate(HUB_LENS):
        t = n - len(HUB_LENS) + j
        assert t >= 2 * W and s["terms"][ticket_row(n, t, form)] == L
    assert sorted(L % HEARTBEAT for L in HUB_LENS) == [0, 1, 1, HEARTBEAT - 1]
    return s


def tri_run(sp, form, m, rng, idx=np.uint32):
    """The device against the oracle (tests/test_gpu_trisolve.py `run`): x bit for bit, and the
    SingularMatrix index and reason when there is one."""
    b = real_values(rng, m.shape[0])
    return TT.run(sp, form, m, b, idx=idx)


# ---------------------------------------------------------------- LDL^T operands
def spd(rng, n, r, c):
    """Symmetric on the pattern {(r, c), (c, r)} (strictly lower pairs given), real values, and
    a diagonal 1 + sum |row|: positive definite."""
    r, c = np.asarray(r, np.int64), np.asarray(c, np.int64)
    key = np.unique(np.maximum(r, c) * n + np.minimum(r, c))
    key = key[key // n != key % n]
    lo = sps.coo_matrix((real_values(rng, key.size), (key // n, key % n)), shape=(n, n))
    a = (lo + lo.T).tocsr()
    a = sps.csr_matrix(a + sps.diags(1.0 + np.asarray(abs(a).sum(axis=1)).ravel()))
    a.sort_indices()
    return a


def band_pairs(n, bw):
    i = np.repeat(np.arange(n), bw)
    j = i - np.tile(np.arange(1, bw + 1), n)
    return i[j >= 0], j[j >= 0]


def band_case(rng, n, bw=BAND):
    return spd(rng, n, *band_pairs(n, bw))


def scramble(rng, a):
    """(Q A Q^T, perm = Q): factoring the result with perm gives a's factor structure, with each
    row's entries in a random stored order."""
    n = a.shape[0]
    q = rng.permutation(n)
    c = a.tocoo()
    b = sps.csr_matrix((c.data, (q[c.row], q[c.col])), shape=(n, n))
    b.sort_indices()
    return b, q


def nd3d_case(rng, side):
    """The 7-point Laplacian pattern of a side^3 grid, random SPD values, nested dissection."""
    lap = TL.laplacian((side,) * 3).tocoo()
    return spd(rng, lap.shape[0], lap.row, lap.col), TL.nested_dissection((side,) * 3)


def nd2d_case(rng, side):
    lap = TL.laplacian((side, side)).tocoo()
    return spd(rng, lap.shape[0], lap.row, lap.col), TL.nested_dissection((side, side))


def seam_blocks(W):
    """Block sizes of the pattern-seam case: a band of W + 3 rows (so the rest is past the first
    wave), dense blocks of 67 (row patterns 0..66, column prefixes 0..65, input rows of 67
    entries), and arrows whose hub rows have SEAM_LENS pattern entries."""
    return [("band", W + 3), ("dense", 67)] + [("arrow", L + 1) for L in SEAM_LENS] + \
           [("dense", 67)]


def seam_case(rng, W):
    r, c, at = [], [], 0
    for kind, size in seam_blocks(W):
        if kind == "band":
            i, j = band_pairs(size, 4)
        elif kind == "dense":
            i, j = np.tril_indices(size, -1)
        else:  # every leaf connects to the hub, the block's last row
            i, j = np.full(size - 1, size - 1), np.arange(size - 1)
        r.append(i + at)
        c.append(j + at)
        at += size
    return spd(rng, at, np.concatenate(r), np.concatenate(c))


def nonsym_case(rng, n):
    """A band of half-bandwidth 8, then: 10 % of the strictly upper entries take other values,
    10 % of the strictly lower ones are dropped, and entries a distance 9 to 12 below the
    diagonal are added without partners.  Not symmetric in values or in pattern."""
    a = band_case(rng, n, 8).tocoo()
    up = a.row < a.col
    lo = a.row > a.col
    data = a.data.copy()
    change = up & (rng.random(a.nnz) < 0.1)
    data[change] = real_values(rng, int(change.sum()))
    keep = ~(lo & (rng.random(a.nnz) < 0.1))
    i = rng.choice(np.arange(12, n), n // 20, replace=False)
    j = i - rng.integers(9, 13, i.size)
    rows = np.concatenate([a.row[keep], i])
    cols = np.concatenate([a.col[keep], j])
    vals = np.concatenate([data[keep], real_values(rng, i.size)])
    m = sps.csr_matrix((vals, (rows, cols)), shape=(n, n))
    m.sort_indices()
    return m


def oracle_factor(m, storage, perm):
    m = TL.as_storage(m, storage)
    fa = LO.Factor(m.indptr, m.indices, perm)
    return fa, fa.update(m.data)


def ldl_seams(fa, W):
    """From the oracle's L: every row's pattern length, every pattern entry's column prefix
    (the entries of its column before it: slot - colptr[i]) with its row, and the pattern steps
    in all (the numeric phase's work)."""
    cp, li, _ = fa.l()
    n = fa.n
    li = li.astype(np.int64)
    pat = np.bincount(li, minlength=n)
    prefix = np.arange(li.size) - np.repeat(cp[:-1].astype(np.int64), np.diff(cp).astype(np.int64))
    return {"late": max(0, n - W), "pattern": pat, "prefix": prefix, "prefix_row": li,
            "steps": int(li.size), "three": int(np.count_nonzero(pat >= 3))}


def input_seams(m, storage, perm):
    """Per row k of P A P^T: the stored length of its outer vector, the position of its
    diagonal there and the number of its entries with pinv[j] > k."""
    m = TL.as_storage(m, storage)
    n = m.shape[0]
    perm = np.arange(n) if perm is None else np.asarray(perm)
    pinv = np.empty(n, np.int64)
    pinv[perm] = np.arange(n)
    lens, diag_pos, above = np.zeros(n, np.int64), np.full(n, -1), np.zeros(n, np.int64)
    for k in range(n):
        o = perm[k]
        j = pinv[m.indices[m.indptr[o]:m.indptr[o + 1]]]
        lens[k] = j.size
        hit = np.flatnonzero(j == k)
        if hit.size:
            diag_pos[k] = hit[0]
        above[k] = np.count_nonzero(j > k)
    return {"len": lens, "diag_pos": diag_pos, "above": above}


def ldl_run(sp, m, storage, perm, check=True, idx=np.uint32, seed=0):
    """tests/test_gpu_ldl.py `run` (L's colptr, indices and values, D, x of solve, the singular
    index), then x of solve_dev against the oracle."""
    num = TL.run(sp, m, storage, perm, check=check, idx=idx, seed=seed)
    if num is not None:
        fa, err = oracle_factor(m, storage, perm)
        assert err is None
        b = real_values(np.random.default_rng(seed + 1), m.shape[0])
        TL.same(dev_solve(num, [b])[0], fa.solve(b), "x of solve_dev")
    return num


def dev_solve(num, bs):
    """solve_dev of each b, enqueued back to back; the results after one synchronise."""
    import torch
    from sprs_b200 import generate as G
    dev = G._device(num._ctx)
    db = [torch.from_numpy(np.array(b, np.float64)).to(dev) for b in bs]
    dx = [torch.empty_like(b) for b in db]
    for b, x in zip(db, dx):
        num.solve_dev(b.data_ptr(), x.data_ptr())
    G._sync()
    return [x.cpu().numpy() for x in dx]


# ================================================================ trisolve tests
@pytest.mark.parametrize("form", TO.FORMS)
@pytest.mark.parametrize("at", ["W-1", "W", "W+1", "3W+5"])
def test_trisolve_wave_seams_bits(sp, W, form, at):
    n = {"W-1": W - 1, "W": W, "W+1": W + 1, "3W+5": 3 * W + 5}[at]
    rng = np.random.default_rng(10 + 4 * TO.FORMS.index(form) + ["W-1", "W", "W+1", "3W+5"].index(at))
    m = wave_case(rng, n, W, form.startswith("u"))
    s = assert_wave_seams(m, form, W)
    assert s["late"] == {"W-1": 0, "W": 0, "W+1": 1, "3W+5": 2 * W + 5}[at]
    tri_run(sp, form, m, rng)


@pytest.mark.parametrize("form", TO.FORMS)
def test_trisolve_group_seams_bits(sp, W, form):
    rng = np.random.default_rng(20 + TO.FORMS.index(form))
    m = group_case(rng, W, form.startswith("u"))
    assert_group_seams(m, form, W)
    tri_run(sp, form, m, rng)


@pytest.mark.parametrize("form", TO.FORMS)
def test_trisolve_heartbeat_seams_bits(sp, W, form):
    rng = np.random.default_rng(30 + TO.FORMS.index(form))
    m = hub_case(rng, W, form.startswith("u"))
    assert_hub_seams(m, form, W)
    tri_run(sp, form, m, rng)


@pytest.mark.parametrize("form", TO.FORMS)
@pytest.mark.parametrize("kind", ["missing", "zero", "negzero"])
@pytest.mark.parametrize("where", ["W+3", "last"])
def test_trisolve_singular_late_bits(sp, W, form, kind, where):
    """Singular past the first wave: the index, the reason and the whole partial rhs; for the
    CSC forms the rows from the singular ticket on hold b_r minus the terms of the columns
    processed before it."""
    n = 3 * W + 5
    at = W + LATE if where == "W+3" else n - 1
    rng = np.random.default_rng(40 + 3 * TO.FORMS.index(form) + ["missing", "zero", "negzero"].index(kind))
    m = singular_case(rng, W, form.startswith("u"), kind, at)
    st = TT.as_storage(m, form)
    probe = np.ones(n)
    err = TO.solve(form, st.indptr, st.indices, st.data, probe)
    assert err is not None and err[0] == ticket_row(n, at, form) and at >= W
    if form.endswith("csc") and where == "W+3":
        # rows past the singular ticket that read a column processed before it
        c = csr_of(m, form)
        partial = 0
        for t in range(at + 1, n):
            r = ticket_row(n, t, form)
            cols = c.indices[c.indptr[r]:c.indptr[r + 1]]
            tick = n - 1 - cols if form.startswith("u") else cols
            partial += int(np.any(tick < at))
        assert partial >= W
    tri_run(sp, form, m, rng)


@pytest.mark.parametrize("form", TO.FORMS)
def test_trisolve_lap2d_bits(sp, W, form):
    """The 2-D Laplacian of a 500^2 grid with random values: row i reads i - 1 and i - 500."""
    rng = np.random.default_rng(50 + TO.FORMS.index(form))
    m = lap2d_case(rng, 500)
    assert m.shape[0] > 3 * W and TO.levels(m.indptr, m.indices, form.startswith("u")) == 999
    tri_run(sp, form, m, rng)


@pytest.mark.parametrize("form", TO.FORMS)
def test_trisolve_lap2d_full_size(sp, W, form):
    rng = np.random.default_rng(60 + TO.FORMS.index(form))
    m = lap2d_case(rng, 2000)
    tri_run(sp, form, m, rng)


def unit_lower_case(rng, n):
    """A strictly lower L (CSC) whose columns have GROUP_LENS entries where they fit, values
    N(0,1) * 2^k with k in [-24, -10] so that x stays finite without a dominant diagonal."""
    rows, cols = [], []
    for i in range(n - 1):
        cnt = min(GROUP_LENS[i % len(GROUP_LENS)], n - 1 - i)
        rows.append(i + 1 + rng.choice(n - 1 - i, cnt, replace=False))
        cols.append(np.full(cnt, i))
    r, c = np.concatenate(rows), np.concatenate(cols)
    v = rng.standard_normal(r.size) * np.exp2(rng.integers(-24, -9, r.size))
    lm = sps.csc_matrix((v, (r, c)), shape=(n, n))
    lm.sort_indices()
    return lm


def test_ldl_unit_solves_bits(sp, W):
    """ldl_lsolve / ldl_ltsolve as free functions, against the oracle's column sweeps."""
    rng = np.random.default_rng(70)
    n = W + 200
    lm = unit_lower_case(rng, n)
    counts = np.diff(lm.indptr)
    assert counts.max() == 97 and np.count_nonzero(counts > GROUP) >= 100
    assert np.count_nonzero(np.bincount(lm.indices, minlength=n) > GROUP) >= 100  # rows too
    mat = sp.CsMat.new_csc((n, n), lm.indptr.astype(np.uint32), lm.indices.astype(np.uint32),
                           lm.data)
    for fn in ("lsolve", "ltsolve"):
        b = real_values(rng, n)
        got, want = b.copy(), b.copy()
        getattr(sp.ldl, "ldl_" + fn)(mat, got)
        getattr(LO, fn)(lm.indptr, lm.indices, lm.data, want)
        assert np.isfinite(want).all()
        TL.same(got, want, fn)


def test_trisolve_two_streams(sp, W):
    """The lower and upper plans of one matrix solved on two streams at once, a second matrix's
    plan between them on one of the streams: every x equals the oracle's."""
    import torch
    from sprs_b200 import generate as G
    rng = np.random.default_rng(80)
    n = 3 * W + 5
    a = wave_case(rng, n, W, False)
    a = sps.csr_matrix(a + wave_case(rng, n, W, True))  # both triangles: row r reads r -+ 1, r -+ W
    b = group_case(rng, W, False)
    ma = sp.CsMat.new((n, n), a.indptr, a.indices, a.data)
    mb = sp.CsMat.new((n, n), b.indptr, b.indices, b.data)
    ctx = ma.context()
    plans = [(sp.linalg.TriSolvePlan(ma, lower=True), "lsolve_csr", a),
             (sp.linalg.TriSolvePlan(ma, lower=False), "usolve_csr", a),
             (sp.linalg.TriSolvePlan(mb, lower=True), "lsolve_csr", b)]
    rhs = [real_values(rng, n) for _ in plans]
    xs = [torch.from_numpy(r.copy()).to(G._device(ctx)) for r in rhs]
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s1):
        assert G.trisolve_dev(ctx, plans[0][0], xs[0]) is None
    with torch.cuda.stream(s2):
        assert G.trisolve_dev(ctx, plans[2][0], xs[2]) is None
        assert G.trisolve_dev(ctx, plans[1][0], xs[1]) is None
    s1.synchronize()
    s2.synchronize()
    for (plan, form, m), r, x in zip(plans, rhs, xs):
        want = r.copy()
        assert TO.solve(form, m.indptr, m.indices, m.data, want) is None
        d = TO.first_difference(x.cpu().numpy(), want)
        assert d is None, "%s: %s" % (form, d)
        plan.free()


# ================================================================ LDL^T tests
LDL_COMBOS = [("CSR", False), ("CSC", True), ("CSR", True), ("CSC", False)]


@pytest.mark.parametrize("at,storage,scrambled",
                         [(at, st, sc) for at in ("W-1", "W+1") for st, sc in LDL_COMBOS] +
                         [("3W+5", st, sc) for st, sc in LDL_COMBOS[:2]])
def test_ldl_band_wave_bits(sp, W, storage, scrambled, at):
    """A band of half-bandwidth 40: rows of about 40 pattern entries whose column prefixes run up
    to 39, each waiting for the row before it, across ticket waves (at 3W + 5 rows, about 10^6
    pattern steps on an H100, one combination of each storage)."""
    n = {"W-1": W - 1, "W+1": W + 1, "3W+5": 3 * W + 5}[at]
    rng = np.random.default_rng(90 + LDL_COMBOS.index((storage, scrambled)))
    m, perm = band_case(rng, n), None
    if scrambled:
        m, perm = scramble(rng, m)
    fa, err = oracle_factor(m, storage, perm)
    assert err is None
    s = ldl_seams(fa, W)
    assert s["late"] == {"W-1": 0, "W+1": 1, "3W+5": 2 * W + 5}[at]
    assert s["pattern"].max() == BAND and np.count_nonzero(s["pattern"] == BAND) == n - BAND
    assert s["prefix"].max() == BAND - 1
    ldl_run(sp, m, storage, perm, seed=n)


@pytest.mark.parametrize("storage,scrambled", LDL_COMBOS[:2])
def test_ldl_nd3d_bits(sp, W, storage, scrambled):
    """The 7-point Laplacian pattern of a 12^3 grid in nested-dissection order, random values."""
    rng = np.random.default_rng(100 + scrambled)
    m, perm = nd3d_case(rng, 12)
    if scrambled:
        m, q = scramble(rng, m)
        perm = q[perm]
    fa, err = oracle_factor(m, storage, perm)
    assert err is None
    s = ldl_seams(fa, W)
    assert s["pattern"].max() > 3 * GROUP and s["prefix"].max() > 3 * GROUP
    ldl_run(sp, m, storage, perm, seed=1728)


def nd2d_wave_side(W):
    """The side of a square grid of more than 3W + 5 points."""
    return int(np.ceil(np.sqrt(3 * W + 5)))


@pytest.mark.parametrize("storage,scrambled", LDL_COMBOS)
def test_ldl_nd2d_wave_bits(sp, W, storage, scrambled):
    """The 5-point Laplacian pattern in nested-dissection order on more than 3W + 5 rows: a
    branching elimination tree, so the pattern order is the reference's stack order, not the
    ascending one, on rows in every wave."""
    rng = np.random.default_rng(105 + LDL_COMBOS.index((storage, scrambled)))
    m, perm = nd2d_case(rng, nd2d_wave_side(W))
    if scrambled:
        m, q = scramble(rng, m)
        perm = q[perm]
    fa, err = oracle_factor(m, storage, perm)
    assert err is None
    s = ldl_seams(fa, W)
    assert s["late"] > 2 * W and s["pattern"].max() > 2 * GROUP
    ldl_run(sp, m, storage, perm, seed=m.shape[0])


def test_ldl_nd3d_20_full_size(sp, W):
    rng = np.random.default_rng(110)
    m, perm = nd3d_case(rng, 20)
    ldl_run(sp, m, "CSC", perm, seed=8000)


def test_ldl_nd2d_300_full_size(sp, W):
    rng = np.random.default_rng(111)
    m, perm = nd2d_case(rng, 300)
    fa, _ = oracle_factor(m, "CSR", perm)
    assert ldl_seams(fa, W)["late"] > 0
    ldl_run(sp, m, "CSR", perm, seed=90000)


@pytest.mark.parametrize("storage,scrambled", LDL_COMBOS)
def test_ldl_pattern_prefix_seams_bits(sp, W, storage, scrambled):
    """Rows past the first wave whose patterns, and pattern entries whose column prefixes, have
    31 / 32 / 33 / 63 / 64 / 65 entries; input rows of 67 entries, half of them with
    pinv[j] > k, the diagonal in many lanes."""
    rng = np.random.default_rng(120 + LDL_COMBOS.index((storage, scrambled)))
    m, perm = seam_case(rng, W), None
    if scrambled:
        m, perm = scramble(rng, m)
    fa, err = oracle_factor(m, storage, perm)
    assert err is None
    s = ldl_seams(fa, W)
    late_pat = set(s["pattern"][W:].tolist())
    late_prefix = set(s["prefix"][s["prefix_row"] >= W].tolist())
    for L in SEAM_LENS:
        assert L in late_pat and L in late_prefix, L
    inp = input_seams(m, storage, perm)
    long_rows = inp["len"] > GROUP
    assert np.count_nonzero(long_rows) >= 134
    assert len(set((inp["diag_pos"][long_rows] % GROUP).tolist())) >= 24
    assert np.count_nonzero(inp["above"][long_rows] > GROUP) >= 60
    ldl_run(sp, m, storage, perm, seed=7)


@pytest.mark.parametrize("storage", ["CSR", "CSC"])
def test_ldl_dont_check_symmetry_wave_bits(sp, W, storage):
    """A non-symmetric matrix of W + 1 rows factored from the entries the reference reads: CSR
    and CSC store different rows, and the oracle's results for the two storages differ."""
    rng = np.random.default_rng(130)
    n = W + 1
    m, perm = nonsym_case(rng, n), None
    if storage == "CSC":
        m, perm = scramble(rng, m)
    assert (m != m.T).nnz > 0
    fr, er = oracle_factor(m, "CSR", perm)
    fc, ec = oracle_factor(m, "CSC", perm)
    assert er is None and ec is None
    assert TO.first_difference(fr.diag(), fc.diag()) is not None
    s = ldl_seams(fr if storage == "CSR" else fc, W)
    assert s["late"] == 1 and 4 * W < s["steps"] < 20 * n  # a band's fill, not a random one's
    with pytest.raises(sp.SprsPanic, match="^Matrix is not symmetric$"):
        TL.run(sp, m, storage, perm)
    ldl_run(sp, m, storage, perm, check=False, seed=n)


def late_pivot(rng, n, k, how, scrambled):
    """A band of half-bandwidth 8 whose D_k is zero; the good matrix of the same pattern; perm.
    0.0 / -0.0: row and column k's other entries are stored zeros and a_kk is 0.0 / -0.0.
    cancel: row k keeps only a_{k,k-1} = v, and a_kk = (v / D_{k-1}) * v, the one term D_k
    subtracts that is not zero (D_{k-1} does not depend on row k)."""
    good = band_case(rng, n, 8)
    a = good.copy()
    rows = np.repeat(np.arange(n), np.diff(a.indptr))
    diag = rows == a.indices
    if how == "cancel":
        kill = ((rows == k) & (a.indices < k - 1)) | ((a.indices == k) & (rows < k - 1))
        a.data[kill] = 0.0
        fa, _ = oracle_factor(a, "CSR", None)
        v = a[k, k - 1]
        a.data[diag & (rows == k)] = (v / fa.diag()[k - 1]) * v
    else:
        a.data[((rows == k) | (a.indices == k)) & ~diag] = 0.0
        a.data[diag & (rows == k)] = float(how)
    perm = None
    if scrambled:
        q = rng.permutation(n)
        out = []
        for x in (a, good):
            c = x.tocoo()
            y = sps.csr_matrix((c.data, (q[c.row], q[c.col])), shape=(n, n))
            y.sort_indices()
            out.append(y)
        a, good, perm = out[0], out[1], q
    return a, good, perm


@pytest.mark.parametrize("how", ["0.0", "-0.0", "cancel"])
@pytest.mark.parametrize("storage,scrambled", LDL_COMBOS[:2])
def test_ldl_singular_late_bits(sp, W, how, storage, scrambled):
    """A zero pivot past the first wave: the index, from `factor` and from `update` of a good
    factor; then an update to good values gives the oracle's bits again."""
    n, k = W + 40, W + 17
    rng = np.random.default_rng(140 + ["0.0", "-0.0", "cancel"].index(how))
    bad, good, perm = late_pivot(rng, n, k, how, scrambled)
    fb, err = oracle_factor(bad, storage, perm)
    assert err == k and k >= W
    assert TL.run(sp, bad, storage, perm) is None  # factor raises the same SingularMatrix
    ms = lambda x: TL.mirror(sp, TL.as_storage(x, storage), storage)  # noqa: E731
    sym = sp.ldl.LdlSymbolic.new_perm(ms(good), np.arange(n) if perm is None else perm)
    num = sym.factor(ms(good))
    fa, err = oracle_factor(good, storage, perm)
    assert err is None
    with pytest.raises(sp.SingularMatrix) as e:
        num.update(ms(bad))
    assert (e.value.index, e.value.reason) == (k, TL.NUMERIC)
    assert fa.update(TL.as_storage(bad, storage).data) == k
    good2 = revalue(rng, good)
    assert np.array_equal(TL.as_storage(good2, storage).indices, TL.as_storage(good, storage).indices)
    num.update(ms(good2))
    assert fa.update(TL.as_storage(good2, storage).data) is None
    TL.same(num.l().data, fa.l()[2], "L after recovery")
    TL.same(num.d(), fa.diag(), "D after recovery")
    b = real_values(rng, n)
    TL.same(num.solve(b), fa.solve(b), "x after recovery")
    TL.same(dev_solve(num, [b])[0], fa.solve(b), "x of solve_dev after recovery")


def revalue(rng, m):
    """The same symmetric pattern (a band), new real values on a dominant diagonal."""
    lo = sps.tril(m, -1).tocoo()
    return spd(rng, m.shape[0], lo.row, lo.col)


@pytest.mark.parametrize("storage,scrambled", LDL_COMBOS[:2])
def test_ldl_update_solve_dev_sequence_bits(sp, W, storage, scrambled):
    """factor, solve_dev, update, solve_dev, update, solve_dev on W + 1 rows, nothing waited for
    between them: every stage's L and D, and every x, equal the oracle's.  An update overwrites
    L and D only after the solves enqueued before it are done."""
    n = W + 1
    rng = np.random.default_rng(150 + scrambled)
    base = band_case(rng, n, 12)
    stages = [base] + [revalue(rng, base) for _ in range(2)]
    perm = None
    if scrambled:
        q = rng.permutation(n)
        stages = [scramble_with(x, q) for x in stages]
        perm = q
    ms = [TL.mirror(sp, TL.as_storage(x, storage), storage) for x in stages]
    assert all(np.array_equal(x.indices, ms[0].indices) for x in ms)
    fa = LO.Factor(TL.as_storage(stages[0], storage).indptr,
                   TL.as_storage(stages[0], storage).indices, perm)
    import torch
    from sprs_b200 import generate as G
    num = sp.ldl.LdlNumeric.new_perm(ms[0], np.arange(n) if perm is None else perm)
    dev = G._device(num._ctx)
    bs = [real_values(rng, n) for _ in stages]
    db = [torch.from_numpy(b.copy()).to(dev) for b in bs]
    dx = [torch.empty_like(b) for b in db]
    want_x = []
    for i, x in enumerate(stages):
        if i:
            num.update(ms[i])
        assert fa.update(TL.as_storage(x, storage).data) is None
        TL.same(num.l().data, fa.l()[2], "L of stage %d" % i)
        TL.same(num.d(), fa.diag(), "D of stage %d" % i)
        num.solve_dev(db[i].data_ptr(), dx[i].data_ptr())
        want_x.append(fa.solve(bs[i]))
    G._sync()
    for i in range(len(stages)):
        TL.same(dx[i].cpu().numpy(), want_x[i], "x of stage %d" % i)


def scramble_with(a, q):
    n = a.shape[0]
    c = a.tocoo()
    b = sps.csr_matrix((c.data, (q[c.row], q[c.col])), shape=(n, n))
    b.sort_indices()
    return b


# ================================================================ 64-bit indptr
_WIDTH_CHILD = r"""
import json, sys
sys.path.insert(0, %(root)r); sys.path.insert(0, %(tests)r)
import numpy as np
import test_gpu_zzz_trisolve_ldl_bits as T
import sprs_b200 as sp
W = T.wave_of(sp.Context.default().sm_count)
errs = []
def check(name, fn):
    try:
        fn()
    except AssertionError as e:
        errs.append("%%s: %%s" %% (name, e))
for form in T.TO.FORMS:
    up = form.startswith("u")
    rng = np.random.default_rng(200 + T.TO.FORMS.index(form))
    check(form + " wave", lambda: T.tri_run(sp, form, T.wave_case(rng, 3 * W + 5, W, up), rng,
                                            idx=np.uint64))
    check(form + " groups", lambda: T.tri_run(sp, form, T.group_case(rng, W, up), rng,
                                              idx=np.uint64))
    check(form + " singular", lambda: T.tri_run(
        sp, form, T.singular_case(rng, W, up, "zero", W + T.LATE), rng, idx=np.uint64))
for storage, scrambled in T.LDL_COMBOS[:2]:
    rng = np.random.default_rng(210 + scrambled)
    for name, m in (("band", T.band_case(rng, W + 1)), ("seams", T.seam_case(rng, W))):
        perm = None
        if scrambled:
            m, perm = T.scramble(rng, m)
        check(storage + " " + name, lambda: T.ldl_run(sp, m, storage, perm, idx=np.uint64))
    check(storage + " nonsym", lambda: T.ldl_run(sp, T.nonsym_case(rng, W + 1), storage, None,
                                                 check=False, idx=np.uint64))
print(json.dumps(errs))
"""


def test_trisolve_ldl_indptr64_child_process(tmp_path):
    script = tmp_path / "child.py"
    script.write_text(_WIDTH_CHILD % {"root": ROOT, "tests": os.path.join(ROOT, "tests")})
    r = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=900,
                       env=dict(os.environ, SPRS_B200_FORCE_INDPTR64="1"))
    assert r.returncode == 0, r.stdout + r.stderr
    assert json.loads(r.stdout.strip().splitlines()[-1]) == []
