"""tests/spmv_model.py pinned on the CPU: the vectorised model against its lane-by-lane
transcription, against the oracle on the rows the kernel sums in storage order, and against
math.fsum within the error bound of its own tree depth."""
import numpy as np
import pytest

import exact
import spmv_model as M
from test_gpu_zzz_spmv_bits import SPECIALS, start_values, structure, values

CUTS = [None, (512, 8), (2048, 4)]


@pytest.fixture(scope="module")
def O():
    from oracle import oracle
    return oracle


@pytest.fixture
def sp(request, monkeypatch):
    import sprs_b200
    cut = getattr(request, "param", None)
    if cut:
        monkeypatch.setattr(sprs_b200, "SPMV_TILE", cut[0])
        monkeypatch.setattr(sprs_b200, "SPMV_ROW_COST", cut[1])
    return sprs_b200


def _case(sp, name, kind, seed=1):
    ip, ind, cols = structure(sp, name)
    return ip, ind, values(len(ind), kind, seed), values(cols, kind, seed + 1), start_values(ip, kind, seed + 2)


@pytest.mark.parametrize("sp", CUTS, indirect=True, ids=["default", "512,8", "2048,4"])
@pytest.mark.parametrize("name", ["seam", "random", "skewed", "hypersparse", "hubs", "empty_runs"])
def test_vectorised_model_matches_literal(sp, name):
    """The vectorised model equals the loop transcription of rows_direct + the fix-up bit for bit,
    fresh and accumulating (wide values; y0 with -0.0, +-inf and NaN on empty rows)."""
    ip, ind, data, x, y0 = _case(sp, name, "wide")
    exact.assert_same_class(M.spmv(ip, ind, data, x), M.literal(ip, ind, data, x), name + " fresh")
    exact.assert_same_class(M.spmv(ip, ind, data, x, y0), M.literal(ip, ind, data, x, y0), name + " acc")


@pytest.mark.parametrize("name", ["seam", "skewed", "empty_runs", "hypersparse"])
def test_model_matches_oracle_on_storage_order_rows(sp, O, name):
    """Tiny rows no tile carries are summed in storage order: the oracle's bits, fresh and
    accumulating, with y0 = +-0.0, +-inf and NaN on empty rows (kept as they are)."""
    ip, ind, data, x, y0 = _case(sp, name, "normal")
    so = M.storage_order_rows(ip)
    assert so.sum() > 100
    want = O.mul_acc_mat_vec_csr(ip, ind, data, x, np.zeros(len(y0)))
    exact.assert_bits(M.spmv(ip, ind, data, x)[so], want[so], name + " fresh")
    with np.errstate(all="ignore"):
        want = O.mul_acc_mat_vec_csr(ip, ind, data, x, y0.copy())
    got = M.spmv(ip, ind, data, x, y0)
    exact.assert_same_class(got[so], want[so], name + " accumulating")
    empty = np.flatnonzero(np.diff(ip.astype(np.int64)) == 0)
    keep = empty[so[empty]]  # (an empty row that starts a tile is the previous tile's carry row)
    assert len(keep) >= len(SPECIALS)
    exact.assert_same_class(got[keep], y0[keep], name + ": empty rows keep y0")


@pytest.mark.parametrize("name", ["seam", "skewed", "hubs"])
def test_model_within_its_tree_bound(sp, name):
    """|y - fsum| <= gamma_d * sum|terms| per row, d = the model's tree depth for the row: the
    model is a summation of the row's terms and y0, whatever its order."""
    ip, ind, data, x, _ = _case(sp, name, "wide")
    y0 = values(len(ip) - 1, "wide", 9)
    for start in (None, y0):
        got = M.spmv(ip, ind, data, x, start)
        ref, mag = M.fsum_rows(ip, ind, data, x, start)
        bound = M.gamma(M.tree_depth(ip)) * mag
        bad = np.abs(got - ref) > bound
        assert not bad.any(), (np.flatnonzero(bad)[:5], (got - ref)[bad][:5], bound[bad][:5])


def test_one_shot_and_tile_range_forms_agree(sp):
    """The tile-range form (each range's kernel, then the carries of the rows ending in it)
    gives the one-shot bits for cuts through carry runs and at single tiles."""
    for name in ("seam", "hubs"):
        ip, ind, data, x, y0 = _case(sp, name, "wide")
        n = M.n_tiles(ip)
        rng = np.random.default_rng(3)
        for ranges in ([0, 1, n], [0, n - 1, n], [0] + sorted(rng.choice(np.arange(1, n), 6, replace=False).tolist()) + [n]):
            for start in (None, y0):
                exact.assert_same_class(M.spmv(ip, ind, data, x, start, tile_ranges=ranges),
                                        M.spmv(ip, ind, data, x, start), "%s %s" % (name, ranges))


def test_model_chunks_by_tile_range(sp, monkeypatch):
    """A small CHUNK_NNZ (the model then holds a few tiles at a time) changes no bit."""
    ip, ind, data, x, y0 = _case(sp, "seam", "wide")
    want = M.spmv(ip, ind, data, x, y0)
    monkeypatch.setattr(M, "CHUNK_NNZ", 3000)
    exact.assert_same_class(M.spmv(ip, ind, data, x, y0), want, "chunked model")
