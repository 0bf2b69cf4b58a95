"""Host model of the synthetic benchmark inputs (csrc/gen.cu, sprs_b200/generate.py), written
from their definition in numpy so that tests can compare the device generators with it bit for bit.

  * hash: the splitmix64 finaliser `mix64` on uint64 (and its inverse, to build keys whose
    hashes land where a test wants them);
  * R-MAT keys: candidate e of `seed` draws one 16-bit digit per level, four digits from each
    64-bit word w_j = mix64(mix64(seed ^ mix64(e)) + j * GAMMA), the lowest digit first.  The
    digit u picks a quadrant against the quantised thresholds ta <= tab <= tabc (a: u < ta,
    b: u < tab, c: u < tabc, d: otherwise), whose row and column bits are appended below the
    ones already drawn; a candidate outside the shape is the all-ones SENTINEL;
  * uniform keys: row = hi64(h1 * n_rows), col = hi64(h2 * n_cols) with h2 = mix64(h1 + GAMMA);
  * hash keys (`>> 1`: 63 bits), split keys;
  * normal values: u1, u2 formed in float64 exactly as the kernel forms them, then
    sqrt(-2 log u1) * cos(2 pi u2) in extended precision with the argument of cos reduced exactly;
  * the assembly of generate.py: collect (drop the sentinel, unique per chunk, unique overall),
    thin (exact: the `target` smallest hashes; approximate: hashes below target / n * 2^63),
    the R-MAT oversampling loop, and the CSR of the sorted unique keys.

Keys are row << 32 | col as uint64."""
import math
import sys

import numpy as np

assert sys.byteorder == "little"  # rmat_keys reads a word's digits as its uint16s

U64 = np.uint64
MASK64 = (1 << 64) - 1
SENTINEL = U64(MASK64)

# splitmix64
MIX_GAMMA = 0x9E3779B97F4A7C15
MIX_M1, MIX_M2 = 0xBF58476D1CE4E5B9, 0x94D049BB133111EB
MIX_SHIFTS = (30, 27, 31)
# the increment between a candidate's words (R-MAT) and from h1 to h2 (uniform keys, values)
GAMMA = 0xD1B54A32D192ED03
DIGIT_BITS = 16
DIGITS_PER_WORD = 4
# seed tweaks of generate.py: values of a matrix, hashes of its thinning
VALUE_TWEAK = 0xDA7A
HASH_TWEAK = 0x7417
# generate.py's assembly
CHUNK = 1 << 27
RAND_MIN_EXTRA, RAND_EXTRA_DIV = 4096, 512
RMAT_FACTOR, RMAT_GROWTH, RMAT_PASSES = 1.6, 1.5, 6
EXACT_THIN_MAX = 1 << 27
GRAPH500 = (0.57, 0.19, 0.19)


def _u64(x):
    return np.asarray(x, dtype=U64)


# ---------------------------------------------------------------- hash
def mix64_int(z):
    """splitmix64's finaliser of z + golden ratio, Python integers."""
    z = (z + MIX_GAMMA) & MASK64
    z = ((z ^ (z >> MIX_SHIFTS[0])) * MIX_M1) & MASK64
    z = ((z ^ (z >> MIX_SHIFTS[1])) * MIX_M2) & MASK64
    return z ^ (z >> MIX_SHIFTS[2])


def mix64(z):
    z = _u64(z)
    with np.errstate(over="ignore"):
        z = z + U64(MIX_GAMMA)
        z = (z ^ (z >> U64(MIX_SHIFTS[0]))) * U64(MIX_M1)
        z = (z ^ (z >> U64(MIX_SHIFTS[1]))) * U64(MIX_M2)
    return z ^ (z >> U64(MIX_SHIFTS[2]))


def _unxorshift(z, s):
    x = z
    for _ in range(64 // s + 1):
        x = z ^ (x >> s)
    return x


def unmix64_int(h):
    """The z with mix64_int(z) == h."""
    z = _unxorshift(h, MIX_SHIFTS[2])
    z = (z * pow(MIX_M2, -1, 1 << 64)) & MASK64
    z = _unxorshift(z, MIX_SHIFTS[1])
    z = (z * pow(MIX_M1, -1, 1 << 64)) & MASK64
    z = _unxorshift(z, MIX_SHIFTS[0])
    return (z - MIX_GAMMA) & MASK64


def key_with_h1(seed, h1):
    """The key whose value hashes give h1 = mix64(seed ^ mix64(key)) (hence h2 too)."""
    return unmix64_int(unmix64_int(h1) ^ seed)


def key_with_h2(seed, h2):
    return key_with_h1(seed, (unmix64_int(h2) - GAMMA) & MASK64)


def hash_keys(seed, keys):
    return mix64(U64(seed) ^ mix64(keys)) >> U64(1)


def split_keys(keys):
    keys = _u64(keys)
    return (keys >> U64(32)).astype(np.uint32), (keys & U64(0xFFFFFFFF)).astype(np.uint32)


# ---------------------------------------------------------------- keys
def thresholds(a, b, c):
    """The digit thresholds of quadrants a, a+b and a+b+c: each probability times 2^16, rounded
    half up (truncation of x + 0.5 in float64)."""
    return tuple(int(p * 65536.0 + 0.5) for p in (a, a + b, a + b + c))


def _words(seed, e, j):
    with np.errstate(over="ignore"):
        return mix64(mix64(U64(seed) ^ mix64(e)) + U64((j * GAMMA) & MASK64))


def rmat_keys(seed, scale, n_rows, n_cols, a, b, c, first, count):
    ta, tab, tabc = thresholds(a, b, c)
    u = np.arange(1 << DIGIT_BITS)
    quadrant = ((u >= ta).astype(np.uint8) + (u >= tab) + (u >= tabc)).astype(np.uint8)  # 0 a .. 3 d
    e = np.arange(count, dtype=U64) + U64(first)
    row = np.zeros(count, np.uint32)  # scale <= 31
    col = np.zeros(count, np.uint32)
    for level in range(scale):
        j, d = divmod(level, DIGITS_PER_WORD)
        if d == 0:  # digit d of a word is its d-th uint16, the lowest first (little-endian)
            digits = _words(seed, e, j).view(np.uint16).reshape(count, DIGITS_PER_WORD)
        q = quadrant[digits[:, d]]
        row = (row << np.uint32(1)) | (q >> 1)
        col = (col << np.uint32(1)) | (q & 1)
    inside = (row < U64(n_rows)) & (col < U64(n_cols))
    return np.where(inside, (row.astype(U64) << U64(32)) | col, SENTINEL)


def mulhi64(h, n):
    """hi64(h * n) for uint64 h and n < 2^32, from 32-bit halves."""
    h = _u64(h)
    n = U64(n)
    hi, lo = h >> U64(32), h & U64(0xFFFFFFFF)
    return (hi * n + ((lo * n) >> U64(32))) >> U64(32)


def uniform_keys(seed, n_rows, n_cols, first, count):
    e = np.arange(count, dtype=U64) + U64(first)
    h1 = mix64(U64(seed) ^ mix64(e))
    with np.errstate(over="ignore"):
        h2 = mix64(h1 + U64(GAMMA))
    return (mulhi64(h1, n_rows) << U64(32)) | mulhi64(h2, n_cols)


# ---------------------------------------------------------------- normal values
def uniforms(seed, keys):
    """(u1, u2) in float64 as the kernel forms them: ((h >> 11) + 0.5) * 2^-53, the addition
    rounded to nearest even (it rounds once h >> 11 >= 2^52)."""
    h1 = mix64(U64(seed) ^ mix64(keys))
    with np.errstate(over="ignore"):
        h2 = mix64(h1 + U64(GAMMA))
    half = np.float64(0.5)
    u1 = ((h1 >> U64(11)).astype(np.float64) + half) * np.float64(2.0 ** -53)
    u2 = ((h2 >> U64(11)).astype(np.float64) + half) * np.float64(2.0 ** -53)
    return u1, u2


def _cospi_ext(x):
    """cos(pi x) for float64 x in [0, 2], in extended precision with the argument reduced exactly:
    x' = min(x, 2 - x) and r = 1/2 - x' are exact, and cos(pi x') = sin(pi r)."""
    x = np.asarray(x, np.float64).astype(np.longdouble)
    xr = np.minimum(x, np.longdouble(2) - x)
    r = np.longdouble(0.5) - xr
    return np.sin(PI_EXT * r)


def _pi_ext():
    if np.finfo(np.longdouble).nmant < 63:
        return None
    # pi to the longdouble's precision: the float64 pi plus its remainder
    return np.longdouble(math.pi) + np.longdouble(1.2246467991473532e-16)


PI_EXT = _pi_ext()


def normal_exact(u1, u2):
    """sqrt(-2 log u1) * cos(2 pi u2), relative error far below 2^-53: numpy's long double when it
    carries >= 63 mantissa bits, mpmath at 40 digits otherwise."""
    u1 = np.asarray(u1, np.float64)
    u2 = np.asarray(u2, np.float64)
    if PI_EXT is not None:
        r = np.sqrt(np.longdouble(-2) * np.log(u1.astype(np.longdouble))) * _cospi_ext(2.0 * u2)
        return r
    import mpmath
    mpmath.mp.dps = 40
    out = np.empty(u1.shape, dtype=object)
    for i, (a, b) in enumerate(zip(u1.ravel(), u2.ravel())):
        out.flat[i] = mpmath.sqrt(-2 * mpmath.log(mpmath.mpf(float(a)))) * mpmath.cospi(2 * mpmath.mpf(float(b)))
    return out


def normal_values(seed, keys):
    """(exact, u1, u2): the extended-precision normal values of keys (indices 0.. when keys is an
    int count) and the uniforms they come from."""
    if isinstance(keys, (int, np.integer)):
        keys = np.arange(int(keys), dtype=U64)
    u1, u2 = uniforms(seed, keys)
    return normal_exact(u1, u2), u1, u2


# ---------------------------------------------------------------- assembly (generate.py)
def sorted_unique(k):
    k = np.sort(k)
    return k[np.concatenate(([True], k[1:] != k[:-1]))] if k.size else k


def collect(gen, n_candidates, chunk=CHUNK):
    """gen(first, count) -> uint64 keys; the sorted unique keys that are not the sentinel."""
    parts = []
    for first in range(0, n_candidates, chunk):
        k = gen(first, min(chunk, n_candidates - first))
        parts.append(sorted_unique(k[k != SENTINEL]))
    if not parts:
        return np.zeros(0, U64)
    return sorted_unique(np.concatenate(parts))


def thin(keys, target, seed, exact):
    """Keep `target` of the keys, chosen by their hash under seed ^ HASH_TWEAK."""
    n = keys.size
    if n <= target:
        return keys
    h = hash_keys(seed ^ HASH_TWEAK, keys).astype(np.int64)
    if exact:
        keep = h <= np.partition(h, target - 1)[target - 1]
    else:
        keep = h < int((target / n) * (1 << 63))
    return keys[keep]


def keys_to_csr(keys, rows):
    """(indptr int64, indices uint32) of sorted unique keys."""
    r, c = split_keys(keys)
    indptr = np.zeros(rows + 1, np.int64)
    np.cumsum(np.bincount(r, minlength=rows), out=indptr[1:])
    return indptr, c


def rand_keys(rows, cols, nnz_per_row, seed):
    target = int(math.ceil(nnz_per_row * rows))
    if target > rows * cols:
        raise ValueError("more non-zeros than cells")
    over = target + max(RAND_MIN_EXTRA, target // RAND_EXTRA_DIV)
    gen = lambda f, n: uniform_keys(seed, rows, cols, f, n)  # noqa: E731
    keys = collect(gen, over)
    while keys.size < target:
        over = int(over * RMAT_GROWTH)
        keys = collect(gen, over)
    return thin(keys, target, seed, exact=True)


def rmat_scale(n):
    return max(1, int(math.ceil(math.log2(n))))


def rmat_keys_pipeline(n, nnz_per_row, seed, abc=GRAPH500, oversample=None, passes_out=None):
    scale = rmat_scale(n)
    target = int(nnz_per_row * n)
    gen = lambda f, cnt: rmat_keys(seed, scale, n, n, *abc, f, cnt)  # noqa: E731
    factor = oversample or RMAT_FACTOR
    for p in range(RMAT_PASSES):
        keys = collect(gen, int(target * factor))
        if keys.size >= target:
            break
        factor *= RMAT_GROWTH
    else:
        raise ValueError("R-MAT candidates short of the target")
    if passes_out is not None:
        passes_out.append(p + 1)
    return thin(keys, target, seed, exact=keys.size <= EXACT_THIN_MAX)


def rand_csr(rows, cols, nnz_per_row, seed):
    """(indptr, indices, keys) of generate.rand_csr."""
    keys = rand_keys(rows, cols, nnz_per_row, seed)
    return keys_to_csr(keys, rows) + (keys,)


def rmat_csr(n, nnz_per_row, seed, **kw):
    keys = rmat_keys_pipeline(n, nnz_per_row, seed, **kw)
    return keys_to_csr(keys, n) + (keys,)
