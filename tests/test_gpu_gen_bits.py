"""The device generators of the benchmark inputs (csrc/gen.cu, sprs_b200/generate.py) BIT FOR BIT
against their host model, tests/gen_model.py, and the benchmark matrices pinned by digest.

  * keys: R-MAT candidates at `first` = 0, around the 2^27 chunk, 2^32 and 2^63 (the candidate
    number is 64-bit), at every scale that adds or drops a 64-bit word, with and without
    rejection, non-square; candidates built (by inverting mix64) to put a digit exactly on and
    just below each quantised threshold, and (a, b, c) whose products with 65536 sit on the
    rounding edge; uniform keys at n = 1 and n = 2^32 - 1; the hash and split kernels; the
    argument checks;
  * values: N(0,1) from keys and from indices within a bound derived below from the CUDA Math
    API's documented maximum errors, including u2 at and next to 1/4 and 3/4, where cos(2 pi u2)
    is zero, and u1 at both ends;
  * the pipeline: rand_csr and rmat_csr (also at density 0.8 and 1, an R-MAT that needs more than
    one oversampling pass, and shapes that cannot reach their target), _collect with chunks
    small enough that duplicates cross them, both branches of _thin;
  * full size (`*_full_size`): configs 2 and 4 whole against the model, config 5's nnz, row
    pointer and one 2^27 candidate chunk, normal_vector(10^7) within the bound, and SHA-256
    digests of every benchmark input (config 3 multiplies config 2's matrix).

The value bound.  The kernel computes y = sqrt(-2 log u1) * cospi(2 u2) in float64.  The CUDA
Math API documents a maximum error of 1 ulp for log and 2 ulp for cospi; sqrt and the product
are correctly rounded; -2 * and 2 * are exact.  With ulp(v) <= 2^-52 |v|, log contributes at most
2^-52 relative, halved by sqrt (1/2 * 2^-52); sqrt rounds (2^-53); cospi 2 * 2^-52; the product
rounds (2^-53): |y_dev - y| <= 3.5 * 2^-52 |y| up to second-order terms (bounded here by
2^-70 |y|).  Since |y| < 2^53 ulp(y), that is at most 7 ulp of y.  The tests report the largest
error they saw in ulp of the float64 of the exact value.  On the CPU emulator, whose cospi is a
plain cos(pi * x), the bound gains that function's absolute error (EMU_COSPI_ABS below).

Small cases run on the CPU emulator too (tests/test_emu_preflight.py); `*_full_size` need the H100."""
import hashlib
import math
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import gen_model as M

pytestmark = pytest.mark.gpu

REL_BOUND = 3.5 * 2.0 ** -52 + 2.0 ** -70
ULP_BOUND = 7
# CPU emulator (tests/emu): cospi(x) is std::cos(pi_d * x) with x in (0, 2]; the argument is off
# by at most 2 pi (2^-53 + 2^-54) < 9.5 * 2^-53 and glibc's cos adds at most 2^-53: |error| <
# 10.5 * 2^-53 < 6 * 2^-52 absolute (the value checks add it; the ulp ceiling is the GPU's)
EMU = os.environ.get("SPRS_B200_EMU") == "1"
EMU_COSPI_ABS = 6 * 2.0 ** -52

FIRSTS = (0, (1 << 27) - 301, (1 << 27) + 3, (1 << 32) - 257, (1 << 32) + 1, (1 << 63) - 300,
          (1 << 63) + 7)
SCALES = (1, 2, 3, 4, 5, 8, 16, 17, 24, 31)
COUNT = 600  # two full blocks of 256 and a partial one

# (name, generator call) of every benchmark input, and the SHA-256 digests of its indptr, indices
# and data bytes (of normal_vector(10^7) with its default seed), recorded on an H100: any change
# of a benchmark input fails here
CONFIGS = {
    "config2": ("rand", 1_000_000, 32, 0x5EED0002),
    "config4_a": ("rmat", 500_000, 16, 0x5EED0004),
    "config4_b": ("rmat", 500_000, 16, 0x5EED0004 ^ 0x1000),
    "config5": ("rmat", 10_000_000, 100, 0x5EED0005),
}
DIGESTS = {
    "config2": ["f77b324736c34d7dd85f89592167b4dc0cef19eee383955b5d7ab6368cf93c88",
                "6a778707aa1db6d59e812428e57ef2a6c9e6f6595f4b2ad426c0a1c08e6ad681",
                "f4a7d0b7b0061d04692643fa3456d0848da935dbd1ffebdbde05c58e8be3d5d1"],
    "config4_a": ["861d573a57214cf7837ecac83ac9480723c152ef393fe01f17f869c47eb231f3",
                  "c5860f84f43d6156c1ff61bf35fe0cf0300e8e1c19c03b885f922ec940c2f46a",
                  "1ab998a801605f73b74ee8b38da9cee0daa282d97a792bd7ff5cf8684cc69ad8"],
    "config4_b": ["298c2cbd03b523716005f814ea92ab5e068abfb90a90b6e05afb823973ccf9f9",
                  "5c2fedd65219a9446436683983cad15c8d7c4b993fb08def64e97de8fb823e7c",
                  "0462237086fc9bb9cfbf03376bafcfd60ec07bd77fa7c7fec0572aa3b879b2af"],
    "config5": ["3405701274884caef80fbce3e6f6c288c84a46c076b6bfcaa701b255ddf74648",
                "9256719ce0732fb1b542a48d389f61458ef6ba43f3c7abc1f4a43c1ac41d1609",
                "24d8175c248ff4a8f8b412c46986027007e9939ef8812499d6f8949cb28b874f"],
    "normal_vector": "db78eea53c5e72b2d5edcabf2b57ed38705b5b3ce37204e470c071d8c9e104a5",
}
CONFIG5_NNZ = 999_996_249


@pytest.fixture(scope="module")
def env():
    import torch
    import sprs_b200
    from sprs_b200 import generate as G
    ctx = sprs_b200.Context.default()  # raises without a GPU / without the .so: no fallback
    return ctx, G, torch


def _dev(env, n, dtype):
    ctx, G, torch = env
    return torch.empty(n, dtype=dtype, device=G._device(ctx))


def _upload(env, a):
    ctx, G, torch = env
    return torch.from_numpy(np.ascontiguousarray(a)).to(G._device(ctx))


def _host(t, dtype):
    return t.cpu().numpy().view(dtype)


def dev_rmat(env, seed, scale, n_rows, n_cols, abc, first, count):
    ctx, G, torch = env
    out = _dev(env, count, torch.int64)
    ctx.check(ctx.lib.sprs_b200_gen_rmat_keys(ctx.h, seed, scale, n_rows, n_cols, *abc, first, count,
                                              G._dptr(out), G._stream_ptr()))
    G._sync()
    return _host(out, np.uint64)


def dev_uniform(env, seed, n_rows, n_cols, first, count):
    ctx, G, torch = env
    out = _dev(env, count, torch.int64)
    ctx.check(ctx.lib.sprs_b200_gen_uniform_keys(ctx.h, seed, n_rows, n_cols, first, count,
                                                 G._dptr(out), G._stream_ptr()))
    G._sync()
    return _host(out, np.uint64)


def dev_normal(env, seed, keys=None, count=None):
    """the value kernel on uint64 keys (host array or device int64 tensor), or on indices"""
    ctx, G, torch = env
    if keys is not None and isinstance(keys, np.ndarray):
        keys = _upload(env, keys.view(np.int64))
    n = count if keys is None else keys.numel()
    out = _dev(env, n, torch.float64)
    ctx.check(ctx.lib.sprs_b200_gen_normal_from_keys(ctx.h, seed, None if keys is None else G._dptr(keys),
                                                     n, G._dptr(out), G._stream_ptr()))
    G._sync()
    return out


def check_values(got, exact, u1):
    """got (float64) within REL_BOUND of exact, and within ULP_BOUND ulp of it on a GPU; returns
    the largest error in ulp of exact.  The emulator's cospi is cos(pi * x) in float64, whose
    error is absolute (EMU_COSPI_ABS) rather than relative near the zeros, so there the bound
    gains that error times sqrt(-2 log u1)."""
    ex = exact.astype(np.float64)
    err = np.abs(got.astype(exact.dtype) - exact)
    bound = REL_BOUND * np.abs(exact)
    if EMU:
        bound = bound + EMU_COSPI_ABS * np.sqrt(-2 * np.log(u1.astype(exact.dtype)))
    bad = np.flatnonzero(~(err <= bound))
    assert bad.size == 0, [(int(i), got[i], ex[i]) for i in bad[:5]]
    nz = ex != 0  # an exact zero must come out zero (bound 0 on a GPU); it has no ulp to count in
    ulp = np.spacing(np.abs(ex[nz]))
    worst = float(np.max((err[nz] / ulp.astype(exact.dtype)).astype(np.float64))) if nz.any() else 0.0
    assert EMU or worst <= ULP_BOUND
    print("normal values: %d checked, largest error %.3f ulp (GPU bound %d)" % (got.size, worst, ULP_BOUND))
    return worst


def edge_shapes(scale):
    """(n_rows, n_cols): powers of two (nothing rejected), and non-square shapes that reject"""
    p = 1 << scale
    return ((p, p), (max(1, p - p // 4 + 1), max(1, p // 2 + 1)), (max(1, p - 1), p))


# ---------------------------------------------------------------- keys
@pytest.mark.parametrize("scale", SCALES)
def test_rmat_keys_bits(env, scale):
    seed = 0x5EED0005 + scale
    for n_rows, n_cols in edge_shapes(scale):
        for first in FIRSTS:
            got = dev_rmat(env, seed, scale, n_rows, n_cols, M.GRAPH500, first, COUNT)
            want = M.rmat_keys(seed, scale, n_rows, n_cols, *M.GRAPH500, first, COUNT)
            assert np.array_equal(got, want), (n_rows, n_cols, first, np.flatnonzero(got != want)[:5])
            if (n_rows, n_cols) == (1 << scale, 1 << scale):
                assert not np.any(want == M.SENTINEL)
            elif n_cols == (1 << scale) // 2 + 1 and scale >= 2:
                assert np.any(want == M.SENTINEL)


def _candidate_with_digit(seed, level, digit):
    """the candidate number e whose digit at `level` is `digit` (found by inverting mix64)"""
    j, d = divmod(level, M.DIGITS_PER_WORD)
    w = (0x0123456789ABCDEF & ~(0xFFFF << (16 * d))) | (digit << (16 * d))
    base = (M.unmix64_int(w) - j * M.GAMMA) & M.MASK64
    return M.unmix64_int(M.unmix64_int(base) ^ seed)


@pytest.mark.parametrize("abc", [M.GRAPH500, (0.1, 0.3, 0.5)])
def test_rmat_digits_on_the_thresholds(env, abc):
    """A digit equal to a threshold belongs to the next quadrant, one below it to this one: at
    each of the four digits of a word, in the first and second word."""
    seed, scale = 0x5EED0004, 8
    n = 1 << scale
    for t in M.thresholds(*abc):
        for level in (0, 1, 2, 3, 4, 7):
            for digit in (t - 1, t):
                e = _candidate_with_digit(seed, level, digit)
                got = dev_rmat(env, seed, scale, n, n, abc, e, 1)
                want = M.rmat_keys(seed, scale, n, n, *abc, e, 1)
                assert np.array_equal(got, want), (t, level, digit)


def test_rmat_thresholds_at_the_rounding_edge(env):
    """(a, b, c) whose products with 65536, and those of a + b and a + b + c, are k + 1/2 exactly
    (rounded up) and just below it (down): the keys follow the model's thresholds, which differ by
    one between the two."""
    seed, scale, n = 0x5EED0003, 4, 16
    exact = (23456.5 / 65536, 9000 / 65536, 20000 / 65536)
    below = (np.nextafter(exact[0], 0), exact[1], np.nextafter(exact[2], 0))
    assert np.subtract(M.thresholds(*exact), M.thresholds(*below)).tolist() == [1, 1, 1]
    for abc in (exact, below):
        for level in range(scale):
            for t in M.thresholds(*abc):
                for digit in (t - 1, t):
                    e = _candidate_with_digit(seed, level, digit)
                    got = dev_rmat(env, seed, scale, n, n, abc, e, 1)
                    assert np.array_equal(got, M.rmat_keys(seed, scale, n, n, *abc, e, 1))
        got = dev_rmat(env, seed, scale, n, n, abc, 5, 4000)
        assert np.array_equal(got, M.rmat_keys(seed, scale, n, n, *abc, 5, 4000))


@pytest.mark.parametrize("n_rows,n_cols", [(1, 1), (1, (1 << 32) - 1), ((1 << 32) - 1, 3),
                                           (1_000_000, 999_983), (7, (1 << 31) + 1)])
def test_uniform_keys_bits(env, n_rows, n_cols):
    for first in FIRSTS:
        got = dev_uniform(env, 0x5EED0002, n_rows, n_cols, first, COUNT)
        assert np.array_equal(got, M.uniform_keys(0x5EED0002, n_rows, n_cols, first, COUNT)), first


def test_hash_and_split_keys_bits(env):
    ctx, G, torch = env
    rng = np.random.default_rng(3)
    keys = np.concatenate([rng.integers(0, 1 << 63, 1000, np.uint64),
                           np.array([0, 1, (1 << 63) - 1, (5 << 32) | 7], np.uint64)])
    d = _upload(env, keys.view(np.int64))
    h = _dev(env, keys.size, torch.int64)
    ctx.check(ctx.lib.sprs_b200_gen_hash_keys(ctx.h, 0x5EED0002 ^ M.HASH_TWEAK, G._dptr(d), keys.size,
                                              G._dptr(h), G._stream_ptr()))
    G._sync()
    assert np.array_equal(_host(h, np.uint64), M.hash_keys(0x5EED0002 ^ M.HASH_TWEAK, keys))
    assert _host(h, np.uint64).max() < (1 << 63)
    want_r, want_c = M.split_keys(keys)
    for with_rows in (False, True):
        rows = _dev(env, keys.size, torch.int32)
        rows.fill_(-7)
        cols = _dev(env, keys.size, torch.int32)
        ctx.check(ctx.lib.sprs_b200_gen_split_keys(ctx.h, G._dptr(d), keys.size,
                                                   G._dptr(rows) if with_rows else None, G._dptr(cols),
                                                   G._stream_ptr()))
        G._sync()
        assert np.array_equal(_host(cols, np.uint32), want_c)
        if with_rows:
            assert np.array_equal(_host(rows, np.uint32), want_r)
        else:
            assert np.all(rows.cpu().numpy() == -7)


def test_argument_errors(env):
    ctx, G, torch = env
    from sprs_b200 import _lib
    out = _dev(env, 4, torch.int64)
    lib, s = ctx.lib, G._stream_ptr()
    for scale, abc in ((0, M.GRAPH500), (32, M.GRAPH500), (5, (0.5, 0.3, 0.2)), (5, (0.6, 0.3, 0.2)),
                       (5, (0.0, 0.3, 0.2)), (5, (0.5, -0.1, 0.2))):
        assert lib.sprs_b200_gen_rmat_keys(ctx.h, 1, scale, 8, 8, *abc, 0, 4, G._dptr(out), s) == \
            _lib.ERR_ARGUMENT, (scale, abc)
    assert lib.sprs_b200_gen_rmat_keys(ctx.h, 1, 5, 8, 8, *M.GRAPH500, 0, 0x7FFFFFFF * 256 + 1,
                                       G._dptr(out), s) == _lib.ERR_ARGUMENT
    for n_rows, n_cols in ((0, 5), (5, 0), (1 << 32, 5), (5, 1 << 32)):
        assert lib.sprs_b200_gen_uniform_keys(ctx.h, 1, n_rows, n_cols, 0, 4, G._dptr(out), s) == \
            _lib.ERR_ARGUMENT, (n_rows, n_cols)
    # nothing was written, and the largest legal scale still runs
    got = dev_rmat(env, 1, 31, 1 << 31, 1 << 31, M.GRAPH500, 0, 4)
    assert np.array_equal(got, M.rmat_keys(1, 31, 1 << 31, 1 << 31, *M.GRAPH500, 0, 4))


# ---------------------------------------------------------------- values
def edge_value_keys(seed):
    """keys whose u2 sits at and next to 1/4 and 3/4 (cospi(2 u2) near zero; exactly 3/4 gives
    cospi(1.5) = 0), and whose u1 is at its ends (2^-54, and 1 - 2^-53 rounded up to 1.0)"""
    keys = []
    for m in [(1 << 51) + k for k in range(-3, 4)] + [3 * (1 << 51) + k for k in range(-3, 4)]:
        keys.append(M.key_with_h2(seed, (m << 11) | 0x5A5))
    for m in (0, 1, (1 << 52) + 1, (1 << 53) - 2, (1 << 53) - 1):
        keys.append(M.key_with_h1(seed, (m << 11) | 0x3C3))
    return np.array(keys, np.uint64)


def test_normal_values_within_the_bound(env):
    seed = 0x5EED0002 ^ M.VALUE_TWEAK
    rng = np.random.default_rng(4)
    keys = np.concatenate([edge_value_keys(seed), rng.integers(0, 1 << 63, 3000, np.uint64)])
    ex, u1, u2 = M.normal_values(seed, keys)
    assert np.count_nonzero(np.abs(u2[:14] * 4 - np.round(u2[:14] * 4)) < 1e-14) == 14
    assert u2[10] == 0.75 and u1[18] == 1.0 and u1[14] == 2.0 ** -54
    got = dev_normal(env, seed, keys).cpu().numpy()
    check_values(got, ex, u1)
    assert got[18] == 0 and (EMU or got[10] == 0)  # cospi(1.5) is 0 on a GPU, not in cos(pi * 1.5)


def test_normal_vector_within_the_bound(env):
    ctx, G, torch = env
    n = 5000
    got = G.normal_vector(ctx, n)
    G._sync()
    ex, u1, _ = M.normal_values(0x5EED1002, n)
    check_values(got.cpu().numpy(), ex, u1)


# ---------------------------------------------------------------- the pipeline
def check_csr(env, a, want, seed):
    """DeviceCsr a equals the model's (indptr, indices, keys); data bit for bit the value kernel
    on the model's keys under seed ^ VALUE_TWEAK"""
    indptr, indices, keys = want
    ip, ind, data = a.to_host()
    assert a.nnz == keys.size
    assert np.array_equal(ip.astype(np.int64), indptr)
    assert np.array_equal(ind, indices)
    vals = dev_normal(env, seed ^ M.VALUE_TWEAK, keys).cpu().numpy()
    assert np.array_equal(data.view(np.uint64), vals.view(np.uint64))


@pytest.mark.parametrize("rows,cols,npr", [(1000, 1000, 8), (200, 50, 40), (300, 70, 70),
                                           (97, 13, 6.5)])
def test_rand_csr_bits(env, rows, cols, npr):
    """(1000, 1000, 8): one pass; (200, 50, 40): density 0.8, where the first pass has fewer
    distinct cells than the target; (300, 70, 70): every cell; (97, 13, 6.5): ceil of the target"""
    ctx, G, torch = env
    seed = 0x5EED0002 + rows
    a = G.rand_csr(ctx, rows, cols, npr, seed=seed)
    assert a.nnz == math.ceil(npr * rows)
    check_csr(env, a, M.rand_csr(rows, cols, npr, seed), seed)


def test_rand_csr_rejects_more_than_every_cell(env):
    ctx, G, torch = env
    with pytest.raises(ValueError):
        G.rand_csr(ctx, 10, 10, 10.5)


@pytest.mark.parametrize("n,npr,passes", [(1000, 16, 1), (64, 8, 2), (64, 30, 5)])
def test_rmat_csr_bits(env, n, npr, passes):
    ctx, G, torch = env
    seed = 0x5EED0005
    got = []
    want = M.rmat_csr(n, npr, seed, passes_out=got)
    assert got == [passes]
    check_csr(env, G.rmat_csr(ctx, n, npr, seed=seed), want, seed)


def test_rmat_csr_rejects_an_unreachable_target(env):
    """64 x 64 with 60 per row: six passes of candidates never reach 3840 distinct cells"""
    ctx, G, torch = env
    with pytest.raises(ValueError):
        M.rmat_csr(64, 60, 0x5EED0005)
    with pytest.raises(ValueError):
        G.rmat_csr(ctx, 64, 60, seed=0x5EED0005)


def test_collect_across_chunks(env):
    """small chunks, so that duplicates cross them and the last one is partial"""
    ctx, G, torch = env
    seed, scale, n = 0x5EED0004, 7, 100

    def gen(first, cnt, out):
        ctx.check(ctx.lib.sprs_b200_gen_rmat_keys(ctx.h, seed, scale, n, n, *M.GRAPH500, first, cnt,
                                                  G._dptr(out), G._stream_ptr()))
    mgen = lambda f, c: M.rmat_keys(seed, scale, n, n, *M.GRAPH500, f, c)  # noqa: E731
    total, chunk = 5000, 777
    want = M.collect(mgen, total, chunk=chunk)
    parts = [M.sorted_unique(k[k != M.SENTINEL]) for k in (mgen(f, min(chunk, total - f)) for f in range(0, total, chunk))]
    assert sum(p.size for p in parts) > want.size  # duplicates across chunks
    got = G._collect(ctx, gen, total, chunk=chunk)
    G._sync()
    assert np.array_equal(_host(got, np.uint64), want)


@pytest.mark.parametrize("exact", [True, False])
def test_thin_bits(env, exact):
    ctx, G, torch = env
    seed = 0x5EED0002
    keys = M.collect(lambda f, c: M.uniform_keys(seed, 3000, 3000, f, c), 20000)
    for target in (1, 4321, keys.size - 1, keys.size, keys.size + 5):
        got = G._thin(ctx, _upload(env, keys.view(np.int64)), target, seed, exact)
        G._sync()
        want = M.thin(keys, target, seed, exact)
        assert np.array_equal(_host(got, np.uint64), want), target
        if exact:
            assert want.size == min(target, keys.size)


# ---------------------------------------------------------------- full size
def sha256_of(t, chunk=1 << 27):
    """SHA-256 of a device tensor's bytes, downloaded in chunks"""
    h = hashlib.sha256()
    flat = t.reshape(-1)
    for i in range(0, flat.numel(), chunk):
        h.update(flat[i:i + chunk].cpu().numpy().tobytes())
    return h.hexdigest()


def make_config(env, name):
    ctx, G, torch = env
    kind, n, npr, seed = CONFIGS[name]
    if kind == "rand":
        return G.rand_csr(ctx, n, n, npr, seed=seed)
    return G.rmat_csr(ctx, n, npr, seed=seed)


def digests_of(a):
    return [sha256_of(a.indptr), sha256_of(a.indices), sha256_of(a.data)]


@pytest.mark.parametrize("name", ["config2", "config4_a", "config4_b"])
def test_config_matrix_full_size(env, name):
    kind, n, npr, seed = CONFIGS[name]
    a = make_config(env, name)
    want = M.rand_csr(n, n, npr, seed) if kind == "rand" else M.rmat_csr(n, npr, seed)
    check_csr(env, a, want, seed)
    assert digests_of(a) == DIGESTS[name]


def test_config5_full_size(env, monkeypatch):
    """nnz and the row pointer; every candidate of the last 2^27 chunk that survives the
    approximate thinning is in the matrix; the digests."""
    ctx, G, torch = env
    kind, n, npr, seed = CONFIGS["config5"]
    seen = []
    thin = G._thin

    def spy(ctx_, keys, target, seed_, exact):
        seen.append((keys.numel(), target, exact))
        return thin(ctx_, keys, target, seed_, exact)
    monkeypatch.setattr(G, "_thin", spy)
    a = make_config(env, "config5")
    monkeypatch.undo()
    (n_unique, target, exact), = seen
    assert a.nnz == CONFIG5_NNZ and not exact and target == n * npr
    ip = a.indptr.to(torch.int64) & 0xFFFFFFFF
    assert int(ip[0]) == 0 and int(ip[-1]) == a.nnz and bool(torch.all(ip[1:] >= ip[:-1]))
    # the last chunk of the first pass: candidates [first, total)
    total = int(target * M.RMAT_FACTOR)
    first = (total - 1) // M.CHUNK * M.CHUNK
    thr = int((target / n_unique) * (1 << 63))
    rows_of = torch.repeat_interleave(torch.arange(n, device=ip.device, dtype=torch.int64), ip[1:] - ip[:-1])
    rows_of <<= 32
    rows_of |= a.indices.to(torch.int64) & 0xFFFFFFFF
    dev_keys = rows_of
    del rows_of, ip
    step = 1 << 22

    def kept_keys(f):  # the model's candidates [f, f + step) that survive the thinning
        k = M.rmat_keys(seed, M.rmat_scale(n), n, n, *M.GRAPH500, f, min(step, total - f))
        k = k[k != M.SENTINEL]
        return M.sorted_unique(k[M.hash_keys(seed ^ M.HASH_TWEAK, k).astype(np.int64) < thr])
    kept = 0
    with ThreadPoolExecutor(max(1, min(8, os.cpu_count() or 1))) as pool:  # numpy releases the GIL
        for f, k in zip(range(first, total, step), pool.map(kept_keys, range(first, total, step))):
            q = _upload(env, k.view(np.int64))
            pos = torch.searchsorted(dev_keys, q).clamp_(max=dev_keys.numel() - 1)
            assert bool(torch.all(dev_keys[pos] == q)), f
            kept += k.size
    assert kept > 0.5 * (total - first)
    del dev_keys
    assert digests_of(a) == DIGESTS["config5"]


def test_normal_vector_full_size(env):
    ctx, G, torch = env
    n = 10_000_000
    x = G.normal_vector(ctx, n)
    G._sync()
    got = x.cpu().numpy()
    for i in range(0, n, 1 << 21):
        ex, u1, _ = M.normal_values(0x5EED1002, np.arange(i, min(n, i + (1 << 21)), dtype=np.uint64))
        check_values(got[i:i + ex.size], ex, u1)
    assert sha256_of(x) == DIGESTS["normal_vector"]
