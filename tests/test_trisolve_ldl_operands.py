"""The operands of tests/test_gpu_zzz_trisolve_ldl_bits.py reach the seams they claim, with the
oracles alone (no GPU), for the emulator's wave (W = 256) and an H100's (W = 8448); another
order of the same terms changes at least 15 % of the rows of three or more terms of the medium
cases, so the device tests can tell the orders apart; and the kernel constants those tests are
sized from still match the sources.

The alternative orders are host models written here; the oracles keep the reference's order:
  * trisolve, terms taken in groups of 32 in the reference's order as the kernel takes them:
    each group's products subtracted in reverse order, or summed first and subtracted once;
  * LDL^T, each row's pattern walked in ascending column order instead of the reference's stack
    order.  Ascending order is a valid topological order of the elimination tree (a parent has a
    larger index than its children), so it gives the same factor up to rounding."""
import os
import re

import numpy as np
import pytest

import ldl_oracle as LO
import test_gpu_zzz_trisolve_ldl_bits as T
import trisolve_oracle as TO
from conftest import ROOT

MIN_SHARE = 0.15
WAVES = (T.EMU_W, T.H100_W)


# ---------------------------------------------------------------- the kernels' constants
def constants(name):
    src = open(os.path.join(ROOT, "sprs_b200", "csrc", name)).read()
    out = {}
    for m in re.finditer(r"^constexpr \w+(?: \w+)? (\w+) = ([^;]+);", src, re.M):
        expr = m.group(2)
        if re.fullmatch(r"[\d\s*+]+", expr):
            out[m.group(1)] = eval(expr)
    return out


def test_kernel_constants_match_the_sources():
    """A retune of the launch shape or the heartbeat must show up here, not as a silent loss of
    the seams the GPU tests are sized for."""
    tri, ldl = constants("trisolve.cu"), constants("ldl.cu")
    assert tri["TRI_THREADS"] == T.THREADS and ldl["LDL_THREADS"] == T.THREADS
    assert tri["TRI_CTAS_PER_SM"] == T.CTAS_PER_SM and ldl["LDL_CTAS_PER_SM"] == T.CTAS_PER_SM
    assert tri["TRI_HEARTBEAT"] == T.HEARTBEAT
    assert T.wave_of(4) == T.EMU_W == 256 and T.wave_of(132) == T.H100_W == 8448
    # the group of 32 terms and the 32-strided LDL loops are the warp's width
    tsrc = open(os.path.join(ROOT, "sprs_b200", "csrc", "trisolve.cu")).read()
    lsrc = open(os.path.join(ROOT, "sprs_b200", "csrc", "ldl.cu")).read()
    lsrc = lsrc[lsrc.index("ldl_numeric_kernel(LdlArgs<P> a)"):lsrc.index("symmetric_kernel")]
    assert "base += 32" in tsrc and "(base + 32) % TRI_HEARTBEAT" in tsrc
    # the row's pattern zeroed, its input entries, its waits; the pattern steps; the prefixes
    assert lsrc.count("p += 32") == 3 and "base += 32" in lsrc and "q += 32" in lsrc


# ---------------------------------------------------------------- trisolve host models
def tri_model(form, m, b, mode):
    """x of `form` on m (no singular row) with the terms of each row taken in groups of 32 in the
    reference's order: mode "reference" subtracts them one by one in that order, "reverse"
    subtracts each group's products in reverse order, "sum" adds each group's products first and
    subtracts the sum once."""
    c = T.csr_of(m, form)
    n = c.shape[0]
    upper = form.startswith("u")
    x = np.array(b, np.float64)
    for t in range(n):
        r = n - 1 - t if upper else t
        cols = c.indices[c.indptr[r]:c.indptr[r + 1]]
        vals = c.data[c.indptr[r]:c.indptr[r + 1]]
        sel = cols > r if upper else cols < r
        tc, tv = cols[sel], vals[sel]
        if form == "usolve_csc":  # its column sweep subtracts a row's terms in descending order
            tc, tv = tc[::-1], tv[::-1]
        acc = float(x[r])
        for g in range(0, tc.size, T.GROUP):
            prods = [float(v) * float(x[j]) for j, v in zip(tc[g:g + T.GROUP], tv[g:g + T.GROUP])]
            if mode == "reverse":
                prods = prods[::-1]
            if mode == "sum":
                s = prods[0]
                for p in prods[1:]:
                    s = s + p
                prods = [s]
            for p in prods:
                acc = acc - p
        x[r] = acc / float(vals[np.flatnonzero(cols == r)[0]])
    return x


def tri_medium_cases():
    """The medium cases at the emulator's wave: the wave seam at 3W + 5 and the group seams."""
    W = T.EMU_W
    for form in TO.FORMS:
        up = form.startswith("u")
        yield form, "wave", T.wave_case(np.random.default_rng(1), 3 * W + 5, W, up)
        yield form, "groups", T.group_case(np.random.default_rng(2), W, up)


@pytest.mark.parametrize("case", range(2 * len(TO.FORMS)))
def test_trisolve_orders_are_told_apart(case):
    form, name, m = list(tri_medium_cases())[case]
    b = T.real_values(np.random.default_rng(3), m.shape[0])
    want = b.copy()
    assert TO.solve(form, *(lambda s: (s.indptr, s.indices, s.data))(T.TT.as_storage(m, form)),
                    want) is None
    ref = tri_model(form, m, b, "reference")
    assert TO.first_difference(ref, want) is None  # the model's reference order is the oracle's
    three = T.tri_terms(m, form) >= 3
    assert np.count_nonzero(three) >= 100
    for mode in ("reverse", "sum"):
        alt = tri_model(form, m, b, mode)
        share = np.count_nonzero((alt.view(np.uint64) != want.view(np.uint64)) & three) / \
            np.count_nonzero(three)
        assert share >= MIN_SHARE, (form, name, mode, share)


# ---------------------------------------------------------------- trisolve seams
@pytest.mark.parametrize("W", WAVES)
@pytest.mark.parametrize("form", TO.FORMS)
def test_trisolve_cases_reach_their_seams(W, form):
    up = form.startswith("u")
    rng = np.random.default_rng(4)
    for n in (W - 1, W, W + 1, 3 * W + 5):
        s = T.assert_wave_seams(T.wave_case(rng, n, W, up), form, W)
        assert s["late"] == max(0, n - W) and s["three"] >= n // 2
    T.assert_group_seams(T.group_case(rng, W, up), form, W)
    T.assert_hub_seams(T.hub_case(rng, W, up), form, W)
    n = 3 * W + 5
    for kind in ("missing", "zero", "negzero"):
        for at in (W + T.LATE, n - 1):
            m = T.singular_case(rng, W, up, kind, at)
            st = T.TT.as_storage(m, form)
            err = TO.solve(form, st.indptr, st.indices, st.data, np.ones(n))
            assert err[0] == T.ticket_row(n, at, form), (kind, at, err)


# ---------------------------------------------------------------- LDL^T host model
def stack_orders(fa, ip, idx):
    """Every row's pattern in the reference's order, restated from its two-sided stack: each
    input entry's elimination-tree path bottom-up, the paths in reverse stored-entry order."""
    n = fa.n
    parent = fa.parent[:n].astype(np.int64)
    perm, pinv = fa.perm.astype(np.int64), fa.pinv.astype(np.int64)
    flag = np.full(n, -1)
    out = []
    for k in range(n):
        flag[k] = k
        paths = []
        o = perm[k]
        for j in pinv[idx[ip[o]:ip[o + 1]]]:
            path = []
            if j < k:
                while flag[j] != k:
                    path.append(j)
                    flag[j] = k
                    j = parent[j]
            paths.append(path)
        out.append([i for p in reversed(paths) for i in p])
    return out


def ldl_model(m, storage, perm, ascending):
    """ldl_numeric with each row's pattern in the reference's order or in ascending order:
    (L's values in the oracle's CSC layout, D)."""
    a = T.TL.as_storage(m, storage)
    ip, idx, val = a.indptr.astype(np.int64), a.indices.astype(np.int64), a.data
    fa = LO.Factor(a.indptr, a.indices, perm)
    n, cp = fa.n, fa.colptr.astype(np.int64)
    perm_, pinv = fa.perm.astype(np.int64), fa.pinv.astype(np.int64)
    orders = stack_orders(fa, ip, idx)
    y, d = np.zeros(n), np.zeros(n)
    nz = np.zeros(n, np.int64)
    l_idx, l_val = np.zeros(cp[-1], np.int64), np.zeros(cp[-1])
    for k in range(n):
        o = perm_[k]
        for p in range(ip[o], ip[o + 1]):
            j = pinv[idx[p]]
            if j <= k:
                y[j] = y[j] + val[p]
        dk = float(y[k])
        y[k] = 0.0
        for i in (sorted(orders[k]) if ascending else orders[k]):
            yi = float(y[i])
            y[i] = 0.0
            s = slice(cp[i], cp[i] + nz[i])
            y[l_idx[s]] = y[l_idx[s]] - l_val[s] * yi
            lki = yi / float(d[i])
            dk = dk - lki * yi
            l_idx[cp[i] + nz[i]] = k
            l_val[cp[i] + nz[i]] = lki
            nz[i] += 1
        d[k] = dk
        assert dk != 0.0
    return l_val, d


def ldl_medium_cases():
    """The medium cases at the emulator's wave whose elimination tree branches: the 2-D
    nested-dissection Laplacian past the wave and the 12^3 3-D one, each in both permutations.
    (A band or a dense block has a chain for a tree: see test_ldl_chain_orders_are_ascending.)"""
    W = T.EMU_W
    rng = np.random.default_rng(5)
    m, perm = T.nd2d_case(rng, T.nd2d_wave_side(W))
    yield "nd2d", m, "CSR", perm
    m2, q = T.scramble(rng, m)
    yield "nd2d, scrambled", m2, "CSC", q[perm]
    m, perm = T.nd3d_case(rng, 12)
    yield "nd3d 12^3", m, "CSC", perm
    m2, q = T.scramble(rng, m)
    yield "nd3d 12^3, scrambled", m2, "CSR", q[perm]


@pytest.mark.parametrize("case", range(4))
def test_ldl_orders_are_told_apart(case):
    name, m, storage, perm = list(ldl_medium_cases())[case]
    fa, err = T.oracle_factor(m, storage, perm)
    assert err is None
    cp, li, lv = fa.l()
    ref_l, ref_d = ldl_model(m, storage, perm, False)
    assert TO.first_difference(ref_l, lv) is None and TO.first_difference(ref_d, fa.diag()) is None
    alt_l, alt_d = ldl_model(m, storage, perm, True)
    n = fa.n
    row_of = li.astype(np.int64)
    changed = alt_d.view(np.uint64) != ref_d.view(np.uint64)
    changed[row_of[alt_l.view(np.uint64) != ref_l.view(np.uint64)]] = True
    three = T.ldl_seams(fa, T.EMU_W)["pattern"] >= 3
    assert np.count_nonzero(three) >= 100
    share = np.count_nonzero(changed & three) / np.count_nonzero(three)
    assert share >= MIN_SHARE, (name, share)


def test_ldl_chain_orders_are_ascending():
    """A full band or a dense block has a chain for an elimination tree, and a chain has one
    topological order: each row's pattern steps are ascending in the reference's order too,
    whatever order its entries are stored in.  So the band and seam cases check values, waits
    and hand-offs, and the nested-dissection cases check the order.  The arrows' hubs are the
    exception: their leaves are independent, and their steps come in reverse stored order."""
    rng = np.random.default_rng(6)
    for m, perm in ((T.band_case(rng, 300), None), T.scramble(rng, T.band_case(rng, 300)),
                    T.scramble(rng, T.seam_case(rng, 0))):
        a = T.TL.as_storage(m, "CSR")
        fa = LO.Factor(a.indptr, a.indices, perm)
        orders = stack_orders(fa, a.indptr.astype(np.int64), a.indices.astype(np.int64))
        rising = [o == sorted(o) for o in orders]
        hubs = np.cumsum([size for _, size in T.seam_blocks(0)]) - 1 if m.shape[0] != 300 else []
        for k, ok in enumerate(rising):
            assert ok or k in hubs, k


# ---------------------------------------------------------------- LDL^T seams
@pytest.mark.parametrize("W", WAVES)
def test_ldl_cases_reach_their_seams(W):
    rng = np.random.default_rng(7)
    for n in (W - 1, W + 1, 3 * W + 5):
        for scrambled in (False, True):
            m, perm = T.band_case(rng, n), None
            if scrambled:
                m, perm = T.scramble(rng, m)
            fa, err = T.oracle_factor(m, "CSC", perm)
            s = T.ldl_seams(fa, W)
            assert err is None and s["late"] == max(0, n - W)
            assert s["pattern"].max() == T.BAND and s["prefix"].max() == T.BAND - 1
    m = T.seam_case(rng, W)
    for scrambled in (False, True):
        mm, perm = (T.scramble(rng, m) if scrambled else (m, None))
        fa, err = T.oracle_factor(mm, "CSR", perm)
        s = T.ldl_seams(fa, W)
        late_pat = set(s["pattern"][W:].tolist())
        late_prefix = set(s["prefix"][s["prefix_row"] >= W].tolist())
        assert set(T.SEAM_LENS) <= late_pat and set(T.SEAM_LENS) <= late_prefix
        inp = T.input_seams(mm, "CSR", perm)
        long_rows = inp["len"] > T.GROUP
        assert len(set((inp["diag_pos"][long_rows] % T.GROUP).tolist())) >= 24
        assert np.count_nonzero(inp["above"][long_rows] > T.GROUP) >= 60
    for how in ("0.0", "-0.0", "cancel"):
        for scrambled in (False, True):
            bad, good, perm = T.late_pivot(rng, W + 40, W + 17, how, scrambled)
            assert T.oracle_factor(bad, "CSR", perm)[1] == W + 17
            assert T.oracle_factor(good, "CSR", perm)[1] is None


def test_ldl_case_costs():
    """Pattern steps of the H100 cases (the numeric phase's work, about 3 us per step on a
    chain): the small cases stay within a few seconds each."""
    W = T.H100_W
    rng = np.random.default_rng(8)
    fa, _ = T.oracle_factor(T.band_case(rng, 3 * W + 5), "CSR", None)
    assert T.ldl_seams(fa, W)["steps"] < 1_100_000
    m, perm = T.nd3d_case(rng, 12)
    fa, _ = T.oracle_factor(m, "CSC", perm)
    assert T.ldl_seams(fa, W)["steps"] < 400_000
    m, perm = T.nd2d_case(rng, T.nd2d_wave_side(W))
    fa, _ = T.oracle_factor(m, "CSR", perm)
    assert T.ldl_seams(fa, W)["steps"] < 1_000_000
    for storage in ("CSR", "CSC"):
        m, perm = T.scramble(rng, T.nonsym_case(rng, W + 1))
        fa, _ = T.oracle_factor(m, storage, perm)
        assert T.ldl_seams(fa, W)["steps"] < 20 * (W + 1)
