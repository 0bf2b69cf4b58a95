"""The SpMV BIT FOR BIT against the host model of its summation order (tests/spmv_model.py), with
real-valued inputs: N(0,1), and N(0,1) * 2^k with k uniform in [-20, 20], where almost any
re-association changes a bit.

The integer-valued suite (test_gpu_exact.py) makes every partial sum exact, so it cannot see an
FMA, a changed lane stride, carries added in another order, a moved tiny-row threshold or y0
entering the sum elsewhere; the N(0,1) parity checks allow 1e-6 * sum|terms|.  Here every output
of every SpMV entry must equal the model's bits (NaN by class), and on the rows the kernel sums in
storage order (tiny rows no tile carries) the accumulating forms must also equal the oracle's
mul_acc_mat_vec_csr -- y0 = -0.0 on an empty row stays -0.0.

Matrices: the seam matrix of test_gpu_exact.py (rows of 8, 9, 16G and 16G + 1 non-zeros in a
tile of each G, cut rows, carry runs of 1, 2 and > 100 tiles), runs of empty rows, hub rows over
more than 64 tiles, a hypersparse matrix, and a 1M R-MAT in child processes under every switch of
the SpMV, including the cut constants (SPRS_B200_SPMV_VARIANT): the model follows them."""
import ctypes as C
import os
import subprocess
import sys
import types

import numpy as np
import pytest

import exact
import solver_model as SM
import spmv_model as M
from test_gpu_exact import SEAM_COLS, _csr_from_lens, seam_matrix

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SPECIALS = (-0.0, np.inf, -np.inf, np.nan, 0.0)


@pytest.fixture(scope="module")
def sp():
    import sprs_b200
    sprs_b200.Context.default()  # raises without a GPU / without the .so: no fallback
    return sprs_b200


@pytest.fixture(scope="module")
def O():
    from oracle import oracle
    return oracle


# ---------------------------------------------------------------- matrices and values
def structure(sp, name):
    """(indptr u32, indices u32, cols) of a named test matrix."""
    w = sp.SPMV_TILE
    if name == "seam":  # built for the default cut whatever the cut constants are
        ip, ind, _ = seam_matrix(types.SimpleNamespace(SPMV_TILE=1024, SPMV_ROW_COST=16))
        return ip, ind, SEAM_COLS
    rng = np.random.default_rng(sum(map(ord, name)))
    if name == "empty_runs":  # runs of 1 .. 300 empty rows between short and medium rows
        lens = []
        while len(lens) < 6000:
            lens += [0] * int(rng.integers(1, 300)) + list(rng.choice([1, 2, 5, 8, 9, 20, 40], 3))
        cols = 4000
    elif name == "hubs":  # two hub rows over > 64 tiles each, tiny rows around them
        lens = [3] * 50 + [70 * w] + [0] * 5 + [2, 9] + [66 * w + 5] + [1] * 100 + [8] * 40
        cols = 200_000
    elif name == "hypersparse":  # 200k rows, ~1% of them with 1-3 non-zeros, 1M columns
        lens = np.zeros(200_000, dtype=np.int64)
        hit = rng.choice(200_000, 2000, replace=False)
        lens[hit] = rng.integers(1, 4, 2000)
        cols = 1_000_000
    elif name == "random":
        lens = rng.poisson(12, 3000)
        cols = 2000
    elif name == "skewed":
        lens = np.minimum((rng.pareto(1.2, 3000) * 4).astype(np.int64), 2000)
        cols = 2000
    else:
        raise KeyError(name)
    ip, ind = _csr_from_lens(rng, lens, cols)
    return ip, ind, cols


MATRICES = ["seam", "empty_runs", "hubs", "hypersparse"]


def values(n, kind, seed):
    """N(0,1), or N(0,1) * 2^k, k uniform in [-20, 20] ("wide")."""
    rng = np.random.default_rng(seed)
    v = rng.standard_normal(n)
    return np.ldexp(v, rng.integers(-20, 21, n)) if kind == "wide" else v


def start_values(ip, kind, seed):
    """y0: `values`, with -0.0, +-inf, NaN and +0.0 in turn on the empty rows."""
    y0 = values(len(ip) - 1, kind, seed)
    empty = np.flatnonzero(np.diff(ip.astype(np.int64)) == 0)
    for i, v in enumerate(SPECIALS):
        y0[empty[i::len(SPECIALS)]] = v
    return y0


def same(got, want, what):
    """Bits; where `want` is NaN, any NaN."""
    exact.assert_same_class(got, want, what)


# ---------------------------------------------------------------- shape
def test_spmv_bits_matrices_shape(sp):
    """Every path of the model's seam report occurs in the matrices of this file."""
    reached = {}
    for name in MATRICES:
        for k, n in M.seams(structure(sp, name)[0]).items():
            reached[k] = reached.get(k, 0) + n
    missing = [k for k in M.ALL_SEAMS if not reached.get(k)]
    assert not missing, "no matrix reaches: %s" % missing
    print("seams reached: %s" % reached)


# ---------------------------------------------------------------- every entry
def _device(sp, a):
    from sprs_b200 import generate as G
    return G._device(a.context())


def _dev_spmv(sp, a, x, y0, accumulate):
    import torch
    from sprs_b200 import generate as G
    ctx = a.context()
    dev = _device(sp, a)
    yt = torch.from_numpy(np.array(y0, dtype=np.float64)).to(dev)
    G.spmv(ctx, a.device(), torch.from_numpy(x).to(dev), yt, accumulate=accumulate)
    G._sync()
    return yt.cpu().numpy()


def _allgather(sp, a, x, y0, accumulate, n_targets):
    """sprs_b200_spmv_allgather_dev into n_targets buffers on this device (target 0 holds y0)."""
    import torch
    from sprs_b200 import generate as G
    ctx = a.context()
    dev = _device(sp, a)
    rows, pad = a.shape[0], 2
    bufs = [torch.full((rows + 2 * pad,), -7.0, dtype=torch.float64, device=dev) for _ in range(n_targets)]
    bufs[0][pad:pad + rows] = torch.from_numpy(np.array(y0, dtype=np.float64)).to(dev)
    xt = torch.from_numpy(x).to(dev)
    ptrs = (C.c_void_p * n_targets)(*[b.data_ptr() + 8 * pad for b in bufs])
    G._sync()
    ctx.check(ctx.lib.sprs_b200_spmv_allgather_dev(ctx.h, a.device().h, C.c_void_p(xt.data_ptr()), 0,
                                                  n_targets, ptrs, int(accumulate), G._stream_ptr()))
    G._sync()
    out = [b.cpu().numpy() for b in bufs]
    for b in out:
        assert np.all(b[:pad] == -7.0) and np.all(b[pad + rows:] == -7.0), "written outside y"
    return [b[pad:pad + rows] for b in out]


def check_entries(sp, O, ip, ind, data, cols, x, y0, what):
    """Every SpMV entry on one matrix, fresh and accumulating, against the model."""
    rows = len(ip) - 1
    fresh = M.spmv(ip, ind, data, x)
    acc = M.spmv(ip, ind, data, x, y0)
    a = sp.CsMat.new((rows, cols), ip, ind, data)
    same(a * x, fresh, what + ": a * x")
    y = y0.copy()
    sp.prod.mul_acc_mat_vec_csr(a, x, y)
    same(y, acc, what + ": mul_acc_mat_vec_csr")
    # the rows summed in storage order carry the reference's bits, y0 = -0.0 / inf / NaN included
    so = M.storage_order_rows(ip)
    with np.errstate(all="ignore"):
        ref = O.mul_acc_mat_vec_csr(ip, ind, data, x, y0.copy())
    same(y[so], ref[so], what + ": mul_acc_mat_vec_csr vs the oracle on storage-order rows")
    same(fresh[so], O.mul_acc_mat_vec_csr(ip, ind, data, x, np.zeros(rows))[so],
         what + ": model vs the oracle on storage-order rows")
    # CSC operand: the device runs its CSR form, whose rows are sorted like ip's
    cip, cind, cdat = O.convert_mat_storage(rows, cols, ip, ind, data)
    y = y0.copy()
    sp.prod.mul_acc_mat_vec_csc(sp.CsMat.new_csc((rows, cols), cip, cind, cdat), x, y)
    same(y, acc, what + ": mul_acc_mat_vec_csc")
    # k = 3 < 8 columns: one accumulating SpMV per column
    b = np.asfortranarray(np.stack([np.roll(x, 7 * j) for j in range(3)], axis=1))
    out0 = np.asfortranarray(np.stack([np.roll(y0, 5 * j) for j in range(3)], axis=1))
    got = out0.copy(order="F")
    sp.prod.csr_mulacc_dense_colmaj(a, b, got)
    for j in range(3):
        same(got[:, j], M.spmv(ip, ind, data, b[:, j], out0[:, j]), what + ": colmaj column %d" % j)
    same(_dev_spmv(sp, a, x, np.full(rows, -3.0), False), fresh, what + ": spmv_dev")
    same(_dev_spmv(sp, a, x, y0, True), acc, what + ": spmv_dev accumulate")
    for nt in (2, 3):
        for accumulate, want in ((False, fresh), (True, acc)):
            for q, t in enumerate(_allgather(sp, a, x, y0, accumulate, nt)):
                same(t, want, "%s: allgather %d targets, accumulate %d, target %d" % (what, nt, accumulate, q))
    # a row slice (indptr[0] != 0): its own partition
    lo, hi = 41, rows - 37
    part = a.slice_outer(lo, hi)
    same(part * x, M.spmv(part.indptr, part.indices, part.data, x), what + ": row slice")
    return fresh, acc


@pytest.mark.parametrize("kind", ["normal", "wide"])
@pytest.mark.parametrize("name", MATRICES)
def test_spmv_model_bits(sp, O, name, kind):
    """a * x, mul_acc_mat_vec_csr / _csc (y0 with -0.0, +-inf and NaN on empty rows), the
    column-major product with k = 3, spmv_dev plain and accumulating, spmv_allgather_dev with 2
    and 3 targets (plain and accumulating) and a row slice: every output equals the model's."""
    ip, ind, cols = structure(sp, name)
    seed = 100 + MATRICES.index(name)
    data = values(len(ind), kind, seed)
    x = values(cols, kind, seed + 1)
    check_entries(sp, O, ip, ind, data, cols, x, start_values(ip, kind, seed + 2), "%s/%s" % (name, kind))


def test_spmv_model_bits_nonfinite_x(sp, O):
    """NaN, +Inf and -Inf in x at columns that long, cut and tiny rows use: every output by class
    (the model meets them in the kernel's order, so an inf - inf NaN lands where it does there)."""
    ip, ind, cols = structure(sp, "seam")
    rng = np.random.default_rng(12)
    data = values(len(ind), "normal", 13)
    x = values(cols, "normal", 14)
    used = np.unique(ind)
    bad = rng.choice(used, 150, replace=False)
    x[bad[0::3]], x[bad[1::3]], x[bad[2::3]] = np.nan, np.inf, -np.inf
    fresh, acc = check_entries(sp, O, ip, ind, data, cols, x, start_values(ip, "normal", 15), "non-finite x")
    assert np.isnan(fresh).sum() > 10 and np.isinf(fresh).sum() > 10 and np.isfinite(fresh).sum() > len(fresh) // 2


def test_spmv_model_bits_bicgstab(sp):
    """The device BiCGSTAB against tests/solver_model.py with the SpMV MODEL as its matvec (no
    device SpMV in the reference) and the solver's reduction order: new, 6 steps, the restarts
    and a solve, bit for bit."""
    ctx = sp.Context.default()
    n = M.WARP * 1000 + 3
    csr, x0, b = SM.dominant_system(n, 4242, max_off=40)
    a = sp.CsMat((n, n), *csr)
    dev = sp.linalg.BiCGSTAB(a, x0, b)
    mod = SM.Model(SM.model_matvec(*csr), SM.device(SM.grid_for(n, ctx.sm_count)), x0, b)
    SM.assert_same_state(dev, mod, "new")
    for it in range(1, 7):
        dev.step()
        mod.step()
        SM.assert_same_state(dev, mod, "step %d" % it)
    dev.soft_restart()
    mod.soft_restart()
    dev.hard_restart()
    mod.hard_restart()
    SM.assert_same_state(dev, mod, "restarts")
    from sprs_b200.linalg import NotConverged
    try:
        dev.run(1e-9, 300)
        ok = True
    except NotConverged:
        ok = False
    assert ok and mod.run(1e-9, 300)
    SM.assert_same_state(dev, mod, "solve")


# ---------------------------------------------------------------- switches (child processes)
def _child_cases(out_path):
    """(child) the seam matrix (N(0,1)) and a 1M R-MAT through the SpMV entries."""
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import sprs_b200 as sp
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    res = {}
    ip, ind, cols = structure(sp, "seam")
    data, x = values(len(ind), "wide", 1), values(cols, "wide", 2)
    y0 = start_values(ip, "wide", 3)
    a = sp.CsMat.new((len(ip) - 1, cols), ip, ind, data)
    res["seam/host"] = a * x
    y = y0.copy()
    sp.prod.mul_acc_mat_vec_csr(a, x, y)
    res["seam/host_acc"] = y
    res["seam/dev_acc"] = _dev_spmv(sp, a, x, y0, True)
    n = 1_000_000
    r = G.rmat_csr(ctx, n, 16, seed=23)
    x = G.normal_vector(ctx, n, 6)
    y = torch.empty(n, dtype=torch.float64, device="cuda")
    G.spmv(ctx, r, x, y)
    res["rmat/dev"] = y.cpu().numpy()
    y = G.normal_vector(ctx, n, 7)
    res["rmat/y0"] = y.cpu().numpy()
    G.spmv(ctx, r, x, y, accumulate=True)
    res["rmat/dev_acc"] = y.cpu().numpy()
    hx, hy = x.cpu().numpy(), np.empty(n)
    ctx.check(ctx.lib.sprs_b200_mul_mat_vec(ctx.h, r.mirror.h, hx.ctypes.data_as(C.c_void_p), n,
                                            hy.ctypes.data_as(C.c_void_p), n))
    res["rmat/host"] = hy
    res["rmat/x"] = hx
    res["rmat/indptr"], res["rmat/indices"], res["rmat/data"] = r.to_host()
    np.savez(out_path, **res)


CONFIGS = {
    "hot_off": dict(SPRS_B200_SPMV_HOT="0"),
    "hot_1023": dict(SPRS_B200_SPMV_HOT="1023"),
    "hot_24576": dict(SPRS_B200_SPMV_HOT="24576"),
    "force_indptr64": dict(SPRS_B200_FORCE_INDPTR64="1"),
    "variant_512_8": dict(SPRS_B200_SPMV_VARIANT="512,8"),
    "variant_2048_4": dict(SPRS_B200_SPMV_VARIANT="2048,4"),
    "chunked_host_path": dict(SPRS_B200_E2E_CHUNKS="5", SPRS_B200_E2E_MIN_TILES="1"),
}


@pytest.mark.parametrize("config", sorted(CONFIGS))
def test_spmv_model_configuration_child_process(tmp_path, monkeypatch, config):
    """The seam matrix (wide values) and a 1M R-MAT (N(0,1)) under each switch of the SpMV (read
    once per process): hot set off / K = 1023 / K = 24576, 64-bit indptr, the cut constants
    512,8 and 2048,4, and the chunked host path (tile ranges + their carries).  The model runs
    with the child's cut constants; every y equals it bit for bit."""
    sys.path.insert(0, ROOT)
    import sprs_b200 as sp
    env = {k: v for k, v in os.environ.items() if not k.startswith("SPRS_B200_")}
    env.update(CONFIGS[config])
    out = os.path.join(str(tmp_path), config + ".npz")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), out], capture_output=True,
                       text=True, timeout=900, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    got = dict(np.load(out))
    if "SPRS_B200_SPMV_VARIANT" in CONFIGS[config]:
        w, rc = CONFIGS[config]["SPRS_B200_SPMV_VARIANT"].split(",")
        monkeypatch.setattr(sp, "SPMV_TILE", int(w))
        monkeypatch.setattr(sp, "SPMV_ROW_COST", int(rc))
    ip, ind, cols = structure(sp, "seam")
    data, x = values(len(ind), "wide", 1), values(cols, "wide", 2)
    y0 = start_values(ip, "wide", 3)
    same(got["seam/host"], M.spmv(ip, ind, data, x), config + ": seam a * x")
    acc = M.spmv(ip, ind, data, x, y0)
    same(got["seam/host_acc"], acc, config + ": seam mul_acc")
    same(got["seam/dev_acc"], acc, config + ": seam spmv_dev accumulate")
    hip, hind, hdat, hx = got["rmat/indptr"], got["rmat/indices"], got["rmat/data"], got["rmat/x"]
    fresh = M.spmv(hip, hind, hdat, hx)
    same(got["rmat/dev"], fresh, config + ": R-MAT spmv_dev")
    same(got["rmat/host"], fresh, config + ": R-MAT host path")
    same(got["rmat/dev_acc"], M.spmv(hip, hind, hdat, hx, got["rmat/y0"]), config + ": R-MAT accumulate")


# ---------------------------------------------------------------- full size
def _full_size(sp, a, x_seed):
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    n = a.rows
    x = G.normal_vector(ctx, n, x_seed)
    import torch
    y = torch.empty(n, dtype=torch.float64, device="cuda")
    G.spmv(ctx, a, x, y)
    G._sync()
    got = y.cpu().numpy()
    del y
    hip, hind, hdat = a.to_host()
    same(got, M.spmv(hip, hind, hdat, x.cpu().numpy()), "y = A x")


def test_spmv_model_rand_1m_full_size(sp):
    """BASELINE config 2 (1M x 1M sprs-rand, 32 non-zeros per row, N(0,1)): the whole y."""
    from sprs_b200 import generate as G
    _full_size(sp, G.rand_csr(sp.Context.default(), 1_000_000, 1_000_000, 32, seed=0x5EED0002), 0x5EED1002)


def test_spmv_model_rmat_10m_full_size(sp):
    """BASELINE config 5 (10M x 10M R-MAT, ~1e9 non-zeros, N(0,1), the hot set at `auto`): the
    whole y."""
    from sprs_b200 import generate as G
    _full_size(sp, G.rmat_csr(sp.Context.default(), 10_000_000, 100, seed=0x5EED0005), 0x5EED1005)


if __name__ == "__main__":
    _child_cases(sys.argv[1])
