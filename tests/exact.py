"""Integer-valued test data: every product result is EXACT in f64, so it has one right answer.

With small integer inputs every partial sum is an integer below 2^53 and therefore exact, so
every summation order -- trees, carries between tiles, atomics in any arrival order, chunked
fix-ups -- gives the same bits, and a device result must equal the oracle's bit for bit on every
output.  Values are never 0, so a dropped or doubled product always changes a result, and x
differs between columns, so a misrouted gather almost always does too.

Values are a hash of the position, computed identically from numpy (host) and torch (device):
  mat_values    A / B entries in {+-1 .. +-8}
  x_values      x_j in [-2^20, 2^20] \\ {0}, distinct for j < 2^21
  y0_values     integer starting values of the accumulating forms, |y0| <= 2^20
Positions must be below 2^31 (every intermediate then fits an int64 without wrapping).

Test helper, not part of the package."""
import numpy as np

EXACT_LIMIT = 2.0 ** 53


def _hash32(pos, seed):
    """32-bit mix of a non-negative int64 array / tensor (< 2^31); same bits in numpy and torch."""
    h = (pos * 0x9E3779B1 + (seed & 0x7FFFFFFF)) & 0xFFFFFFFF
    h = ((h ^ (h >> 15)) * 0x2C1B3C6D) & 0xFFFFFFFF
    h = ((h ^ (h >> 12)) * 0x297A2D39) & 0xFFFFFFFF
    return h ^ (h >> 15)


def _signed(mag, h, bit):
    return mag * (1 - 2 * ((h >> bit) & 1))


def mat_values(pos, seed):
    """+-1 .. +-8 for positions `pos` (int64 numpy array or torch tensor); float64."""
    h = _hash32(pos, seed)
    v = _signed((h & 7) + 1, h, 3)
    return v.double() if hasattr(v, "double") else v.astype(np.float64)


def x_values(cols, seed):
    """x_j for column indices `cols`: a bijection of j mod 2^21 onto [-2^20, 2^20] \\ {0}."""
    m = ((cols & 0x1FFFFF) * 0x9E3779 + (seed & 0x1FFFFF)) & 0x1FFFFF  # odd multiplier: bijective
    v = _signed((m >> 1) + 1, m, 0)
    return v.double() if hasattr(v, "double") else v.astype(np.float64)


def y0_values(n, seed):
    """Integer starting values for y += A x, |y0| <= 2^20 (numpy)."""
    h = _hash32(np.arange(n, dtype=np.int64), seed ^ 0x5A5A)
    return _signed((h & 0xFFFFF).astype(np.int64), h, 20).astype(np.float64)


def int_csr_data(indptr, seed):
    """numpy: integer values for a host CSR's non-zeros (position = offset from indptr[0])."""
    ip = np.asarray(indptr).astype(np.int64)
    return mat_values(np.arange(int(ip[-1] - ip[0]), dtype=np.int64), seed)


def device_int_data(n, seed, device, chunk=1 << 26):
    """torch: the same values as int_csr_data for n non-zeros, built on `device` in chunks
    (a full-size matrix has 1e9 of them: no 8 GB temporaries)."""
    import torch
    out = torch.empty(n, dtype=torch.float64, device=device)
    for s in range(0, n, chunk):
        e = min(n, s + chunk)
        out[s:e] = mat_values(torch.arange(s, e, dtype=torch.int64, device=device), seed)
    return out


def device_int_csr(ctx, a, seed):
    """A second generate.DeviceCsr over a's indptr / indices with integer data."""
    from sprs_b200 import generate as G
    return G.DeviceCsr(ctx, a.rows, a.cols, a.indptr, a.indices,
                       device_int_data(a.nnz, seed, a.indices.device))


def device_x(ctx, n, seed):
    import torch
    from sprs_b200 import generate as G
    dev = G._device(ctx)
    x = torch.empty(n, dtype=torch.float64, device=dev)
    for s in range(0, n, 1 << 26):
        e = min(n, s + (1 << 26))
        x[s:e] = x_values(torch.arange(s, e, dtype=torch.int64, device=dev), seed)
    return x


def assert_exact_budget(O, indptr, indices, data, x, y0=None):
    """Every output of y (+)= A x is exact: the oracle's product on |A| and |x| (itself exact
    below 2^53), plus |y0|, stays below 2^53 on every row."""
    bound = np.abs(y0) if y0 is not None else np.zeros(len(indptr) - 1)
    bound = np.ascontiguousarray(bound, dtype=np.float64)
    O.mul_acc_mat_vec_csr(indptr, indices, np.abs(data), np.abs(x), bound)
    assert float(bound.max(initial=0.0)) < EXACT_LIMIT, "inputs too large for exact sums"


def assert_spgemm_budget(O, a_shape, a, b_shape, b):
    _, _, bound = O.mul_csr_csr(a_shape, (a[0], a[1], np.abs(a[2])), b_shape,
                                (b[0], b[1], np.abs(b[2])), threads=1)
    assert float(np.max(bound, initial=0.0)) < EXACT_LIMIT, "inputs too large for exact sums"


def assert_bits(got, ref, what=""):
    """Bit-equality of two f64 arrays; a failure names the first differing entry (row of a
    vector, (row, column) of a matrix) and the difference -- with the value scheme above, the
    difference of a dropped / doubled product is +-a_ij * x_j."""
    got, ref = np.asarray(got), np.asarray(ref)
    assert got.shape == ref.shape, "%s: shape %s, want %s" % (what, got.shape, ref.shape)
    g = np.ascontiguousarray(got, dtype=np.float64).view(np.uint64)
    r = np.ascontiguousarray(ref, dtype=np.float64).view(np.uint64)
    bad = g != r
    if bad.any():
        i = np.unravel_index(int(np.flatnonzero(bad.ravel())[0]), bad.shape)
        i = i[0] if len(i) == 1 else i
        raise AssertionError("%s: %d entries differ; first at %s: got %r, want %r (difference %r)"
                             % (what, int(bad.sum()), i, float(got[i]), float(ref[i]),
                                float(got[i]) - float(ref[i])))


def assert_same_class(got, ref, what=""):
    """Outputs with one non-finite term: NaN where the oracle has NaN (any payload / sign),
    the same infinity where it has one, the same bits everywhere else."""
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan), "%s: NaN at %s, want at %s" % (
        what, np.flatnonzero(np.isnan(got).ravel())[:5], np.flatnonzero(nan.ravel())[:5])
    assert_bits(np.where(nan, 0.0, got), np.where(nan, 0.0, ref), what)


def assert_csr_bits(got, ref, what=""):
    """(indptr, indices, data) triples: the structure exactly, the values bit for bit."""
    for name, g, r in zip(("indptr", "indices"), got[:2], ref[:2]):
        g, r = np.asarray(g).astype(np.int64), np.asarray(r).astype(np.int64)
        assert g.shape == r.shape, "%s: %s length %d, want %d" % (what, name, g.size, r.size)
        if not np.array_equal(g, r):
            i = int(np.flatnonzero(g != r)[0])
            raise AssertionError("%s: %s[%d] = %d, want %d" % (what, name, i, g[i], r[i]))
    assert_bits(got[2], ref[2], what + ": data")
