"""The operands of tests/test_gpu_zzz_spmm_bits.py reach the seams they claim, with the oracle
alone (no GPU), for the emulator's pass (P = 2048 rows) and an H100's (P = 67584); another order
of the same terms changes at least 15 % of the outputs of rows with three or more terms of the
medium cases, so the device tests can tell the orders apart; and the kernel constants those tests
are sized from still match csrc/spmm.cu.

The alternative orders are host models written here, one IEEE operation at a time, each row's
terms taken as the kernel takes them (windows of 32, batches of U inside a window); the oracle
keeps the reference's order:
  * each U-batch's products added in reverse;
  * each U-batch's products summed first and the sum added once;
  * the row's products summed first and C added once after;
  * each 32-entry window's products added in reverse."""
import os
import re

import numpy as np
import pytest

import test_gpu_zzz_spmm_bits as T
from conftest import ROOT

MIN_SHARE = 0.15
PASSES = (T.EMU_P, T.H100_P)


@pytest.fixture(scope="module")
def O():
    from oracle import oracle
    return oracle


# ---------------------------------------------------------------- the kernel's constants
def spmm_source():
    return open(os.path.join(ROOT, "sprs_b200", "csrc", "spmm.cu")).read()


def test_kernel_constants_match_the_source():
    """A retune of the launch shape, the batch depths, the panel widths or the window must show
    up here, not as a silent loss of the seams the GPU tests are sized for."""
    src = spmm_source()
    assert re.search(r"^constexpr int SPMM_NT = (\d+);", src, re.M).group(1) == str(T.THREADS)
    assert "const uint64_t cap = (uint64_t)ctx->sm_count * %d;" % T.CTAS_PER_SM in src
    assert T.pass_rows(4) == T.EMU_P == 2048 and T.pass_rows(132) == T.H100_P == 67584
    # the four kernels in the order the launch tries them, and their thresholds
    launch = src[src.index("#define SPMM_LAUNCH"):src.index("#undef SPMM_LAUNCH")]
    picks = re.findall(r"(if \(vec && k <= 64\)|else if \(vec\)|else if \(k <= 32\)|else)\s*\\\s*"
                       r"\n\s*(spmm_rowmaj(?:_vec)?_kernel<P, [^>]+>)", launch)
    assert [(c, re.sub(r"\s", "", kern)) for c, kern in picks] == [
        ("if (vec && k <= 64)", "spmm_rowmaj_vec_kernel<P,1,4>"),
        ("else if (vec)", "spmm_rowmaj_vec_kernel<P,2,2>"),
        ("else if (k <= 32)", "spmm_rowmaj_kernel<P,1>"),
        ("else", "spmm_rowmaj_kernel<P,2>")]
    assert "(k % 2 == 0) && (ldb % 2 == 0) && (ldc % 2 == 0)" in src
    assert "(((uintptr_t)d_b | (uintptr_t)d_c) & 15) == 0" in src
    # panels of 32 * KV (scalar) / 64 * KV2 (vector) columns, windows of 32 pairs in both
    assert "c0 += 32 * KV)" in src and "c0 += 64 * KV2)" in src
    assert src.count("kk += 32)") == 2
    assert src.count("SPMM_LAUNCH(uint32_t)") == 1 and src.count("SPMM_LAUNCH(uint64_t)") == 1
    # the restatement agrees
    assert T.kernel_of(64, 64, 64, 0, 0) == ("vec_u4", 64, 4)
    assert T.kernel_of(66, 66, 66, 0, 0) == ("vec_u2", 128, 2)
    assert T.kernel_of(32, 33, 33, 0, 0) == ("scalar_32", 32, 1)
    assert T.kernel_of(64, 64, 64, 8, 0) == ("scalar_64", 64, 1)


def test_flavours_and_panels_are_covered():
    """The dev layouts reach all four kernels, the vector and scalar form of every even k, and
    every panel count of each kernel that the k list allows, with a last panel of one column
    (scalar) and of one column pair (vector)."""
    seen = {}
    for k, e, o in T.dev_cases():
        name, width, _ = T.claimed_kernel(k, e, o)
        seen.setdefault(name, set()).add(T.panels_of(k, width))
    for k in T.KS:
        seen.setdefault(T.host_kernel(k)[0], set()).add(T.panels_of(k, T.host_kernel(k)[1]))
        if k % 2 == 0:
            kinds = {T.claimed_kernel(k, e, o)[0][:3] for e, o in T.EVEN_LAYOUTS}
            assert kinds == {"vec", "sca"}, k
    assert set(seen) == {"vec_u4", "vec_u2", "scalar_32", "scalar_64"}
    assert {n for n, _ in seen["scalar_32"]} == {1} and (1, 1) in seen["scalar_32"]
    assert {n for n, _ in seen["scalar_64"]} == {1, 2, 3, 5} and (2, 1) in seen["scalar_64"]
    assert (5, 1) in seen["scalar_64"] and (3, 1) in seen["scalar_64"]
    assert {n for n, _ in seen["vec_u4"]} == {1} and {n for n, _ in seen["vec_u2"]} == {1, 2}
    assert (2, 2) in seen["vec_u2"]
    # full panels too
    assert (1, 64) in seen["vec_u4"] and (1, 128) in seen["vec_u2"] and (2, 64) in seen["scalar_64"]


# ---------------------------------------------------------------- seams
@pytest.mark.parametrize("P", PASSES)
def test_cases_reach_their_seams(P):
    case = T.seam_case(P)
    T.assert_seam_case(case)
    # with U = 4 and U = 2, the last batch of the seam rows takes every residue
    for U in (4, 2):
        res = {(L % T.WINDOW or T.WINDOW) % U for L in T.SEAM_LENS if L}
        assert res == set(range(U)), U
    hub = T.hub_case(P)
    assert hub.lens[5] == 0 and hub.lens[P + 5] == T.BIG_HUB and hub.lens[6] == T.HUB
    assert (P + 5) // P == 1 and hub.n < 2 * P


def test_case_costs():
    """The H100 seam case stays small: C at k = 257 is under 300 MB."""
    case = T.seam_case(T.H100_P)
    assert case.n * max(T.KS) * 8 < 300e6 and case.ip[-1] < 500_000


# ---------------------------------------------------------------- order models
def products(case, b, rows, pos):
    j = case.ip[rows].astype(np.int64) + pos
    return case.data[j][:, None] * b[case.ind[j]]


def model(case, b, c0, mode, U=4):
    """out = c0 + A b with each row's terms taken in `mode`'s order, one IEEE operation at a
    time: "reference" (storage order), "batch_reverse", "batch_sum", "c_last", "window_reverse".
    Batches are U consecutive terms from the row's start (32 is a multiple of U, so no batch
    crosses a window)."""
    lens = case.lens
    acc = c0.copy()
    top = int(lens.max())
    if mode in ("reference", "batch_reverse", "window_reverse"):
        for t in range(top):
            rows = np.flatnonzero(lens > t)
            g = U if mode == "batch_reverse" else T.WINDOW
            s = (t // g) * g
            pos = t if mode == "reference" else s + np.minimum(s + g, lens[rows]) - 1 - t
            acc[rows] = acc[rows] + products(case, b, rows, pos)
    elif mode == "batch_sum":
        for s in range(0, top, U):
            rows = np.flatnonzero(lens > s)
            part = products(case, b, rows, s)
            for u in range(1, U):
                sel = lens[rows] > s + u
                part[sel] = part[sel] + products(case, b, rows[sel], s + u)
            acc[rows] = acc[rows] + part
    elif mode == "c_last":
        rows = np.flatnonzero(lens > 0)
        part = products(case, b, rows, 0)
        for t in range(1, top):
            sel = lens[rows] > t
            part[sel] = part[sel] + products(case, b, rows[sel], t)
        acc[rows] = c0[rows] + part
    else:
        raise ValueError(mode)
    return acc


MODELS = [("batch_reverse", 4, 64), ("batch_sum", 4, 64), ("batch_reverse", 2, 130),
          ("batch_sum", 2, 130), ("c_last", 1, 33), ("window_reverse", 1, 33)]


@pytest.fixture(scope="module")
def medium():
    return T.seam_case(T.EMU_P)


@pytest.mark.parametrize("mode,U,k", MODELS)
def test_orders_are_told_apart(O, medium, mode, U, k):
    """On the emulator-sized seam case, accumulating onto a random C0 as the GPU tests do: the
    model's storage order is the oracle's, and each other order changes at least 15 % of the
    outputs of rows with three or more terms."""
    case = medium
    rng = np.random.default_rng(700 + k)
    b = case.b(rng, k)
    c0 = T.real_values(rng, (case.n, k))
    want = case.oracle(O, b, c0)
    ref = model(case, b, c0, "reference")
    assert np.array_equal(ref.view(np.uint64), want.view(np.uint64))
    three = case.lens >= 3
    assert np.count_nonzero(three) >= 100
    alt = model(case, b, c0, mode, U)
    changed = alt.view(np.uint64) != want.view(np.uint64)
    share = np.count_nonzero(changed[three]) / changed[three].size
    assert share >= MIN_SHARE, (mode, U, share)
