"""tests/gen_model.py, the host model of the benchmark inputs, pinned without a GPU: its hash is
splitmix64, its constants are the ones csrc/gen.cu, csrc/common.cuh and sprs_b200/generate.py use
(read from their source, so a change there fails here, not as a silent change of every benchmark
matrix), its R-MAT quadrants come up as often as the quantised (a, b, c, d) say, and its pipeline
keeps the promises generate.py's docstring makes."""
import math
import os

import numpy as np
import pytest

import gen_model as M
from conftest import ROOT


def source(*parts):
    return open(os.path.join(ROOT, *parts)).read()


# ---------------------------------------------------------------- the hash
def splitmix64(seed, n):
    """Vigna's splitmix64 generator, Python integers: state += golden ratio, then mix."""
    out, s = [], seed
    for _ in range(n):
        s = (s + 0x9E3779B97F4A7C15) & M.MASK64
        z = s
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M.MASK64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M.MASK64
        out.append(z ^ (z >> 31))
    return out


def test_mix64_is_splitmix64():
    assert M.mix64_int(0) == 0xE220A8397B1DCDAF
    assert splitmix64(0, 5) == [0xE220A8397B1DCDAF, 0x6E789E6AA1B965F4, 0x06C45D188009454F,
                                0xF88BB8A8724C81EC, 0x1B39896A51A8749B]
    # output k of seed s is mix64(s + k * golden ratio), in Python integers and vectorised
    for seed in (0, 1, 0x5EED0005, M.MASK64):
        want = splitmix64(seed, 1000)
        z = [(seed + k * M.MIX_GAMMA) & M.MASK64 for k in range(1000)]
        assert [M.mix64_int(v) for v in z] == want
        assert M.mix64(np.array(z, np.uint64)).tolist() == want


def test_unmix64_inverts_mix64():
    rng = np.random.default_rng(5)
    for z in [0, 1, M.MASK64, 1 << 63] + [int(v) for v in rng.integers(0, 1 << 63, 200, np.uint64)]:
        assert M.unmix64_int(M.mix64_int(z)) == z
    for seed, h in ((0x5EED1002, 1 << 62), (3, M.MASK64), (0, 0)):
        k = M.key_with_h1(seed, h)
        assert M.mix64_int(seed ^ M.mix64_int(k)) == h
        k = M.key_with_h2(seed, h)
        assert M.mix64_int((M.mix64_int(seed ^ M.mix64_int(k)) + M.GAMMA) & M.MASK64) == h


def test_mulhi64_matches_python_integers():
    rng = np.random.default_rng(6)
    h = np.concatenate([rng.integers(0, 1 << 63, 2000, np.uint64) * np.uint64(2) + np.uint64(1),
                        np.array([0, 1, M.MASK64, 1 << 63, (1 << 32) - 1, 1 << 32], np.uint64)])
    for n in (1, 2, 3, 1000, 10 ** 7, (1 << 31) + 1, (1 << 32) - 1):
        assert M.mulhi64(h, n).tolist() == [(int(v) * n) >> 64 for v in h]


# ---------------------------------------------------------------- constants read from the source
def test_hash_constants_match_the_source():
    mix = source("sprs_b200", "csrc", "common.cuh")
    body = mix[mix.index("uint64_t mix64(uint64_t z)"):]
    body = body[:body.index("}")]
    assert "z += 0x%Xull;" % M.MIX_GAMMA in body
    assert "z = (z ^ (z >> %d)) * 0x%Xull;" % (M.MIX_SHIFTS[0], M.MIX_M1) in body
    assert "z = (z ^ (z >> %d)) * 0x%Xull;" % (M.MIX_SHIFTS[1], M.MIX_M2) in body
    assert "return z ^ (z >> %d);" % M.MIX_SHIFTS[2] in body


def test_kernel_constants_match_the_source():
    """The words, digits, thresholds, uniform mapping, value formation, hash width, launch shape
    and argument checks of csrc/gen.cu, as the model and tests/test_gpu_gen_bits.py take them."""
    src = source("sprs_b200", "csrc", "gen.cu")
    g = "0x%Xull" % M.GAMMA
    assert src.count(g) == 3  # R-MAT words, uniform h2, value h2
    rmat = src[src.index("__global__ void rmat_keys_kernel"):src.index("__global__ void uniform_keys_kernel")]
    assert "const uint64_t base = mix64(seed ^ mix64(e));" in rmat
    assert "if ((l & 3) == 0) w = mix64(base + (uint64_t)(l >> 2) * %s);" % g in rmat
    assert "const uint32_t u = (uint32_t)(w >> (16 * (l & 3))) & 0xffffu;" in rmat
    assert M.DIGIT_BITS == 16 and M.DIGITS_PER_WORD == 4
    assert "const uint32_t rbit = u >= tab;" in rmat
    assert "const uint32_t cbit = (u >= ta && u < tab) || (u >= tabc);" in rmat
    assert "row = (row << 1) | rbit;" in rmat and "col = (col << 1) | cbit;" in rmat
    assert "keys[i] = (row < n_rows && col < n_cols) ? ((row << 32) | col) : ~0ull;" in rmat
    for name, p in (("ta", "a"), ("tab", "(a + b)"), ("tabc", "(a + b + c)")):
        assert "const uint32_t %s = (uint32_t)(%s * 65536.0 + 0.5);" % (name, p) in src
    uni = src[src.index("__global__ void uniform_keys_kernel"):src.index("__global__ void normal_from_keys")]
    assert "const uint64_t h1 = mix64(seed ^ mix64(e));" in uni
    assert "const uint64_t h2 = mix64(h1 + %s);" % g in uni
    assert "const uint64_t row = __umul64hi(h1, n_rows);" in uni
    assert "const uint64_t col = __umul64hi(h2, n_cols);" in uni
    nrm = src[src.index("__global__ void normal_from_keys"):src.index("__global__ void split_keys")]
    assert "const uint64_t key = keys ? keys[i] : i;" in nrm
    for h in ("u1", "u2"):
        assert ("const double %s = ((double)(h%s >> 11) + 0.5) * (1.0 / 9007199254740992.0);"
                % (h, h[1])) in nrm
    assert "out[i] = sqrt(-2.0 * log(u1)) * cospi(2.0 * u2);" in nrm
    assert "out[i] = mix64(seed ^ mix64(keys[i])) >> 1;" in src
    # one thread per candidate, 256 per block; the argument checks the tests exercise
    assert "inline unsigned grid_for(uint64_t n) { return (unsigned)((n + 255) / 256); }" in src
    assert src.count("<<<grid_for(count), 256, 0, pick_stream(ctx, stream)>>>") == 5
    assert "scale < 1 || scale > 31 || a <= 0 || b < 0 || c < 0 || a + b + c >= 1.0" in src
    assert "if (count > 0x7fffffffull * 256)" in src
    assert "n_rows == 0 || n_cols == 0 || n_rows > 0xffffffffull || n_cols > 0xffffffffull" in src


def test_assembly_constants_match_the_source():
    src = source("sprs_b200", "generate.py")
    assert "seed ^ 0x%X," % M.VALUE_TWEAK in src and src.count("0x%X" % M.VALUE_TWEAK) == 1
    assert "seed ^ 0x%X," % M.HASH_TWEAK in src and src.count("0x%X" % M.HASH_TWEAK) == 1
    assert "def _collect(ctx, gen, n_candidates, chunk=1 << 27):" in src and M.CHUNK == 1 << 27
    assert "k = k[k != SENTINEL]" in src and "SENTINEL = -1" in src
    assert "over = target + max(%d, target // %d)" % (M.RAND_MIN_EXTRA, M.RAND_EXTRA_DIV) in src
    assert "factor = oversample or %s" % M.RMAT_FACTOR in src
    assert "over = int(over * %s)" % M.RMAT_GROWTH in src
    assert "factor *= %s" % M.RMAT_GROWTH in src and "for _ in range(%d):" % M.RMAT_PASSES in src
    assert "exact=keys.numel() <= (1 << 27)" in src and M.EXACT_THIN_MAX == 1 << 27
    assert "keep = h <= thr" in src and "torch.kthvalue(h, target)" in src
    assert "keep = h < int((target / n) * (1 << 63))" in src
    assert "target = int(math.ceil(nnz_per_row * rows))" in src
    assert "target = int(nnz_per_row * n)" in src
    assert "scale = max(1, int(math.ceil(math.log2(n))))" in src
    assert "abc=(0.57, 0.19, 0.19)" in src and M.GRAPH500 == (0.57, 0.19, 0.19)


# ---------------------------------------------------------------- R-MAT quadrants
def test_thresholds_round_half_up():
    assert M.thresholds(*M.GRAPH500) == (37356, 49807, 62259)
    # a * 65536 exactly k + 1/2 rounds up; one ulp below it rounds down
    a = 37355.5 / 65536
    assert M.thresholds(a, 0.1, 0.1)[0] == 37356
    assert M.thresholds(np.nextafter(a, 0), 0.1, 0.1)[0] == 37355


@pytest.mark.parametrize("abc", [M.GRAPH500, (0.25, 0.25, 0.25), (0.7, 0.0, 0.29)])
def test_quadrant_frequencies(abc):
    """10^6 candidates at scale 8 (two words): the quadrant drawn at each level comes up within
    6 standard deviations of the quantised probability."""
    n = 10 ** 6
    keys = M.rmat_keys(11, 8, 256, 256, *abc, 3, n)
    assert not np.any(keys == M.SENTINEL)
    row, col = M.split_keys(keys)
    ta, tab, tabc = M.thresholds(*abc)
    p = np.array([ta, tab - ta, tabc - tab, 65536 - tabc]) / 65536
    for level in range(8):
        q = ((row >> (7 - level)) & 1) * 2 + ((col >> (7 - level)) & 1)
        count = np.bincount(q, minlength=4)
        sd = np.sqrt(n * p * (1 - p))
        assert np.all(np.abs(count - n * p) <= 6 * sd + 1e-9), (level, count, n * p)


def test_rejection_and_shape():
    """Candidates outside an n_rows x n_cols shape are the sentinel; the rest lie inside."""
    keys = M.rmat_keys(2, 5, 20, 27, *M.GRAPH500, 0, 50000)
    inside = keys != M.SENTINEL
    row, col = M.split_keys(keys[inside])
    assert row.max() < 20 and col.max() < 27 and 0 < np.count_nonzero(~inside) < 50000


# ---------------------------------------------------------------- the pipeline's promises
@pytest.mark.parametrize("rows,cols,npr", [(1000, 1000, 32), (200, 50, 40), (300, 70, 70),
                                           (97, 13, 6.5)])
def test_rand_csr_has_the_promised_nnz(rows, cols, npr):
    """ceil(density * rows * cols) distinct cells, also where duplicates outnumber the first
    pass's slack (density 0.8) and at density 1."""
    indptr, indices, keys = M.rand_csr(rows, cols, npr, 9)
    assert keys.size == math.ceil(npr * rows) == indptr[-1]
    assert np.all(np.diff(keys.astype(np.float64)) > 0) and indices.max() < cols


def test_rand_csr_rejects_more_than_every_cell():
    with pytest.raises(ValueError):
        M.rand_csr(10, 10, 10.5, 1)


def test_rmat_passes():
    passes = []
    M.rmat_csr(1000, 16, 0x5EED0005, passes_out=passes)
    M.rmat_csr(64, 8, 0x5EED0005, passes_out=passes)
    M.rmat_csr(64, 30, 0x5EED0005, passes_out=passes)
    assert passes == [1, 2, 5]
    with pytest.raises(ValueError):
        M.rmat_csr(64, 60, 0x5EED0005)


def test_normal_model_accuracy():
    """The extended-precision values agree with float64 numpy to a few ulp, and cos(2 pi u2) is
    exactly zero only at u2 = 3/4 (the one multiple of 1/4 the formation of u2 can give)."""
    ex, u1, u2 = M.normal_values(5, 20000)
    approx = np.sqrt(-2 * np.log(u1)) * np.cos(2 * np.pi * u2)
    rel = np.abs(approx - ex.astype(np.float64)) / np.abs(ex.astype(np.float64))
    assert np.median(rel) < 2 ** -50
    assert float(M.normal_exact(np.array([0.5]), np.array([0.75]))[0]) == 0.0
    assert float(M.normal_exact(np.array([1.0]), np.array([0.1]))[0]) == 0.0
