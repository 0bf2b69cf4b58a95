"""The row-partitioned SpMV, its peer exchanges and the distributed BiCGSTAB checked BIT FOR BIT,
at the seams of the partition.

Two references, both exact:
  * integer values (tests/exact.py): every partial sum is exact, so the oracle's
    mul_acc_mat_vec_csr on the WHOLE matrix is the only right answer, whatever the block cut;
    a row that is dropped, doubled, misplaced or stale fails;
  * N(0,1) values: the concatenation over blocks g of sprs_b200_spmv_dev on the block mirror
    rows [b_g, b_g+1).  Every exchange runs that same mirror's kernel, so the bits must match for
    any values.

Part 1 (single process, all targets on one device; these also run on the emulator): the put
kernel behind every exchange (sprs_b200_peer_push_dev) and the chunked push
(sprs_b200_spmv_chunked_push_dev), each target a buffer with sentinels before and after the
written range.

Part 2 (test_comm_*: one spawned process per rank, rank r on device r % n_devices, so a one-GPU
box runs every rank on device 0 through CUDA IPC): CommSpMV over explicit bounds sets -- empty
first / last blocks, a 1-row block at an odd offset, a block of empty rows, cuts beside a hub row
whose carry spans many tiles, world 8 -- in every exchange mode, with and without multicast, as
one call and as the compute() + exchange() split, with two different x on two reps and y
poisoned to NaN before each; CommHostSpMV with uneven x slices; the hot-set kernel and 64-bit
indptr in child processes; and row_partitioned_bicgstab against the host model of
tests/solver_model.py.  Ranks agree with each other through Comm.allgather of a digest."""
import ctypes as C
import hashlib
import os
import sys
import traceback

import numpy as np
import pytest

import exact
import solver_model as M
from test_gpu_exact import SEAM_COLS, _csr_from_lens, seam_matrix

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SENTINEL = -7.25
PAD = 8                 # sentinel doubles before and after every target's range (16-byte aligned)
PUSH_THREADS = 256      # csrc/peer.cu: threads per block of peer_push_kernel
PUSH_UNROLL = 4         # pairs per thread and sweep step


@pytest.fixture(scope="module")
def sp():
    import sprs_b200
    sprs_b200.Context.default()  # raises without a GPU / without the .so: no fallback
    return sprs_b200


@pytest.fixture(scope="module")
def O():
    from oracle import oracle
    return oracle


def _ptrs(tensors):
    return (C.c_void_p * max(len(tensors), 1))(*[t.data_ptr() for t in tensors])


def _filled(dev, n, value=SENTINEL):
    import torch
    return torch.full((n,), value, dtype=torch.float64, device=dev)


def _assert_target(buf, lo, want, what):
    """buf[lo : lo + len(want)] holds want's bits, everything else the sentinel."""
    got = buf.cpu().numpy()
    exact.assert_bits(got[lo:lo + len(want)], want, what + ": written range")
    outside = np.concatenate([got[:lo], got[lo + len(want):]])
    exact.assert_bits(outside, np.full(outside.size, SENTINEL), what + ": sentinels")


# ================================================================ 1. single process
def _push(sp, src, offset, count, peers):
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    st = ctx.lib.sprs_b200_peer_push_dev(ctx.h, C.c_void_p(src.data_ptr()), offset, count,
                                         len(peers), _ptrs(peers) if peers else None,
                                         G._stream_ptr())
    G._sync()
    return st


def _check_push(sp, offset, count, n_peers, what):
    import torch
    from sprs_b200 import generate as G
    dev = G._device(sp.Context.default())
    length = offset + count + PAD
    src = torch.from_numpy(np.random.default_rng(count * 31 + offset).standard_normal(length)).to(dev)
    before = src.cpu().numpy().copy()
    peers = [_filled(dev, length) for _ in range(n_peers)]
    assert _push(sp, src, offset, count, peers) == 0, what
    for q, buf in enumerate(peers):
        _assert_target(buf, offset, before[offset:offset + count], "%s peer %d" % (what, q))
    exact.assert_bits(src.cpu().numpy(), before, what + ": source changed")


@pytest.mark.parametrize("n_peers", [0, 1, 2, 7, 8])
def test_peer_push_small_counts_bits(sp, n_peers):
    """Counts 0-3 from an even and an odd row offset: the scalar head (odd offset) and the scalar
    tail (odd count after the head) are taken or not, alone or around one pair."""
    for offset in (PAD, PAD + 1):
        for count in (0, 1, 2, 3):
            _check_push(sp, offset, count, n_peers, "offset %d count %d" % (offset, count))


def _push_blocks(sm_count, count):
    """peer_push_launch: one block per 1024 pairs, at most 2 * sm_count."""
    return max(1, min((count // 2 + 1023) // 1024, 2 * sm_count))


@pytest.mark.parametrize("n_peers", [1, 8])
def test_peer_push_sweep_seams_bits(sp, n_peers):
    """Counts on the put kernel's grid-stride seams: a sweep is 4 * blocks * 256 pairs with
    blocks = min(ceil(floor(count / 2) / 1024), 2 * sm_count).  At the block cap: exactly one sweep, one
    sweep and one pair, and more than two full sweeps -- each with and without a head."""
    sm = sp.Context.default().sm_count
    cap = 2 * sm
    sweep = PUSH_UNROLL * PUSH_THREADS * cap  # pairs of one sweep at the cap
    for head in (0, 1):
        offset = PAD + head
        for pairs, tail in ((sweep, 0), (sweep + 1, 1), (2 * sweep + sweep // 2 + 3, 1)):
            count = head + 2 * pairs + tail
            blocks = _push_blocks(sm, count)
            assert blocks == cap, (count, blocks)
            _check_push(sp, offset, count, n_peers, "head %d pairs %d tail %d" % (head, pairs, tail))


def test_peer_push_contract(sp):
    """n_peers outside 0..8, a null peer or a peer whose 16-byte parity differs from the
    source's: ARGUMENT, and nothing is launched or written."""
    from sprs_b200 import _lib
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    dev = G._device(ctx)
    n = 64
    src = _filled(dev, n + 2 * PAD, 1.5)
    peers = [_filled(dev, n + 2 * PAD) for _ in range(9)]
    launches = ctx.launches
    for n_peers in (-1, 9):
        st = ctx.lib.sprs_b200_peer_push_dev(ctx.h, C.c_void_p(src.data_ptr()), PAD, n, n_peers,
                                             _ptrs(peers), G._stream_ptr())
        assert st == _lib.ERR_ARGUMENT, (n_peers, st)
    for bad in (1, 2):  # one peer off by one double, at either position
        arr = (C.c_void_p * 3)(*[p.data_ptr() for p in peers[:3]])
        arr[bad] = peers[bad].data_ptr() + 8
        for count in (0, n):
            st = ctx.lib.sprs_b200_peer_push_dev(ctx.h, C.c_void_p(src.data_ptr()), PAD, count, 3,
                                                 arr, G._stream_ptr())
            assert st == _lib.ERR_ARGUMENT, (bad, count, st)
    arr = (C.c_void_p * 2)(peers[0].data_ptr(), None)
    st = ctx.lib.sprs_b200_peer_push_dev(ctx.h, C.c_void_p(src.data_ptr()), PAD, n, 2, arr,
                                         G._stream_ptr())
    assert st == _lib.ERR_ARGUMENT, st
    G._sync()
    assert ctx.launches == launches
    for buf in peers:
        _assert_target(buf, 0, np.zeros(0), "untouched peer")


# ---------------------------------------------------------------- chunked push
MAX_CHUNKS = 8  # SPRS_E2E_MAX_CHUNKS


def _chunk_tiles(sp, ip, n_chunks):
    """csmat_chunk_table(taper=True) restated: the tile cut of each chunk of the tile stream, and
    the tile partition (tile_row, tile_nnz) it cuts."""
    _, tr, tk = sp.spmv_rows_cut_by_tiles(np.asarray(ip), tiles=True)
    n_tiles = len(tr) - 1
    n = max(1, min(n_chunks, MAX_CHUNKS, n_tiles))
    wsum = n * (n + 1) // 2
    tiles, acc = [], 0
    for c in range(n):
        tiles.append(n_tiles * acc // wsum)
        acc += n - c
    tiles.append(n_tiles)
    for c in range(1, n):
        tiles[c] = max(tiles[c], tiles[c - 1] + 1)
    for c in range(n - 1, 0, -1):
        tiles[c] = min(tiles[c], tiles[c + 1] - 1)
    return tiles, tr, tk


def _chunk_rows(sp, ip, n_chunks):
    """The row cut of each chunk (rows [cut[c], cut[c+1]) are final after chunk c) and n_tiles."""
    tiles, tr, _ = _chunk_tiles(sp, ip, n_chunks)
    return [int(tr[t]) for t in tiles], len(tr) - 1


def _rows_across_cuts(sp, ip, n_chunks):
    """Rows that a chunk cut splits: their carries from one chunk are added after the next."""
    tiles, tr, tk = _chunk_tiles(sp, ip, n_chunks)
    ip = np.asarray(ip).astype(np.int64)
    rows = len(ip) - 1
    return {int(tr[t]) for t in tiles[1:-1] if ip[tr[t]] < tk[t] < ip[min(tr[t] + 1, rows)]}


HUB_ROW = 2500


def _hub_matrix():
    """N(0,1) values; row HUB_ROW (60000 non-zeros, about a third of the tiles) is split by a
    chunk cut at every chunk count from 2 to 8 (test_hub_matrix_rows_across_cuts), so its carries
    reach the rows of a later chunk; row 100 (20000) is long but stays inside the first chunk;
    empty rows at both ends belong to the first / last chunk."""
    rng = np.random.default_rng(32)
    rows, cols = 5000, 120000
    lens = rng.poisson(12, rows)
    lens[rng.random(rows) < 0.3] = 0
    lens[:40] = 0
    lens[-55:] = 0
    lens[100] = 20000
    lens[HUB_ROW] = 60000
    ip, ind = _csr_from_lens(rng, lens, cols)
    return ip, ind, rng.standard_normal(len(ind)), cols


def test_hub_matrix_rows_across_cuts(sp):
    """The hub row of the chunked-push matrix is split by a chunk cut at every chunk count the
    chunked-push tests use, so the carry across chunks is always exercised."""
    ip = _hub_matrix()[0]
    missing = [n for n in range(2, MAX_CHUNKS + 2) if HUB_ROW not in _rows_across_cuts(sp, ip, n)]
    assert not missing, "no chunk cut inside the hub row at %s chunks" % missing


def _small_matrix():
    """Fewer tiles than chunks."""
    rng = np.random.default_rng(33)
    ip, ind = _csr_from_lens(rng, rng.integers(1, 6, 100), 500)
    return ip, ind, rng.standard_normal(len(ind)), 500


def _matrix(sp, name):
    if name == "seam_int":
        ip, ind, data = seam_matrix(sp)
        return ip, ind, data, SEAM_COLS
    return {"hub_normal": _hub_matrix, "few_tiles": _small_matrix}[name]()


def _chunked(sp, mirror, x, offset, bufs, accumulate, n_chunks):
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    st = ctx.lib.sprs_b200_spmv_chunked_push_dev(ctx.h, mirror.h, C.c_void_p(x.data_ptr()), offset,
                                                 len(bufs), _ptrs(bufs), accumulate,
                                                 n_chunks, G._stream_ptr())
    G._sync()
    return st


def _spmv_dev(sp, mirror, x, y0, accumulate):
    import torch
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    y = torch.from_numpy(y0.copy()).to(G._device(ctx))
    G.spmv(ctx, mirror, x, y, accumulate=bool(accumulate))
    G._sync()
    return y.cpu().numpy()


def _check_chunked(sp, ip, mirror, x, n_chunks, accumulate, n_targets, offset, what, want_chunks=None):
    """Every target holds spmv_dev's bits in rows [offset, offset + rows), sentinels elsewhere,
    and the call issued one put per non-empty chunk of the table for `want_chunks`."""
    import torch
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    dev = G._device(ctx)
    rows = mirror.rows
    y0 = exact.y0_values(rows, 9) if accumulate else np.full(rows, SENTINEL)
    want = _spmv_dev(sp, mirror, x, y0, accumulate)
    length = offset + rows + PAD

    def bufs():
        out = [_filled(dev, length) for _ in range(n_targets)]
        out[0][offset:offset + rows] = torch.from_numpy(y0).to(dev)
        return out

    b1 = bufs()[:1]
    assert _chunked(sp, mirror, x, offset, b1, accumulate, n_chunks) == 0, what
    _assert_target(b1[0], offset, want, what + " (1 target)")
    l0 = ctx.launches  # the launches of the chunks alone, once the chunk table exists
    assert _chunked(sp, mirror, x, offset, bufs()[:1], accumulate, n_chunks) == 0, what
    alone = ctx.launches - l0
    bn = bufs()
    l0 = ctx.launches
    assert _chunked(sp, mirror, x, offset, bn, accumulate, n_chunks) == 0, what
    puts = ctx.launches - l0 - (alone if n_targets > 1 else 0)
    for q, b in enumerate(bn):
        _assert_target(b, offset, want, "%s target %d of %d" % (what, q, n_targets))
    if n_targets > 1 and want_chunks is not None:
        cut, _ = _chunk_rows(sp, ip, want_chunks)
        expect = sum(1 for c in range(len(cut) - 1) if cut[c + 1] > cut[c])
        assert puts == expect, "%s: %d puts, want one per non-empty chunk of %d: %d" % (
            what, puts, want_chunks, expect)
    return want


CHUNK_CASES = [(0, 0, 8, 5), (1, 1, 2, 8), (2, 0, 1, 8), (5, 1, 8, 3), (8, 0, 2, 3), (9, 1, 8, 8)]


@pytest.mark.parametrize("name", ["seam_int", "hub_normal", "few_tiles"])
def test_chunked_push_bits(sp, O, name):
    """n_chunks 0 (the default 4), 1, 2, 5, 8 and 9 (clamped to 8), and more chunks than the
    mirror has tiles, each with accumulate 0 / 1, 1, 2 or 8 targets and an odd or an even row
    offset: every target equals spmv_dev, one put per non-empty chunk.  With integer values the
    result must also equal the oracle."""
    import torch
    from sprs_b200 import generate as G
    ip, ind, data, cols = _matrix(sp, name)
    rows = len(ip) - 1
    a = sp.CsMat.new((rows, cols), ip, ind, data)
    mirror = a.device()
    dev = G._device(sp.Context.default())
    integer = name.endswith("_int")
    xh = exact.x_values(np.arange(cols, dtype=np.int64), 4) if integer else \
        np.random.default_rng(4).standard_normal(cols)
    x = torch.from_numpy(xh).to(dev)
    _, n_tiles = _chunk_rows(sp, ip, 1)
    if name == "few_tiles":
        assert n_tiles < 5, n_tiles
    for n_chunks, acc, nt, offset in CHUNK_CASES:
        want_chunks = 4 if n_chunks == 0 else n_chunks
        got = _check_chunked(sp, ip, mirror, x, n_chunks, acc, nt, offset,
                             "%s chunks %d acc %d" % (name, n_chunks, acc), want_chunks)
        if integer:
            y0 = exact.y0_values(rows, 9) if acc else np.zeros(rows)
            exact.assert_bits(got, O.mul_acc_mat_vec_csr(ip, ind, data, xh, y0.copy()), name + " oracle")


def test_chunked_push_env_and_table_cache(sp, monkeypatch):
    """SPRS_B200_PUSH_CHUNKS overrides n_chunks on every call; the cached chunk table of a
    mirror is rebuilt when the chunk count changes (4, then 2, then 4 on one mirror)."""
    import torch
    from sprs_b200 import generate as G
    ip, ind, data, cols = _hub_matrix()
    rows = len(ip) - 1
    mirror = sp.CsMat.new((rows, cols), ip, ind, data).device()
    x = torch.from_numpy(np.random.default_rng(8).standard_normal(cols)).to(G._device(sp.Context.default()))
    first = _check_chunked(sp, ip, mirror, x, 4, 0, 2, 3, "4 chunks", 4)
    for n in (2, 4, 3, 4):
        exact.assert_bits(_check_chunked(sp, ip, mirror, x, n, 0, 2, 3, "%d chunks" % n, n), first,
                          "chunk count %d" % n)
    monkeypatch.setenv("SPRS_B200_PUSH_CHUNKS", "6")
    for n in (0, 2):
        _check_chunked(sp, ip, mirror, x, n, 0, 8, 3, "env 6, argument %d" % n, 6)
    monkeypatch.setenv("SPRS_B200_PUSH_CHUNKS", "1")
    _check_chunked(sp, ip, mirror, x, 5, 0, 2, 4, "env 1", 1)


def test_chunked_push_empty_mirrors(sp):
    """Rows without non-zeros: every target gets +0.0 (accumulate: y0 unchanged); 0 rows:
    nothing is written."""
    import torch
    from sprs_b200 import generate as G
    dev = G._device(sp.Context.default())
    x = torch.from_numpy(np.arange(1.0, 41.0)).to(dev)
    empty = sp.CsMat.new((300, 40), np.zeros(301, np.uint32), np.zeros(0, np.uint32), np.zeros(0)).device()
    ip = np.zeros(301, np.uint32)
    for acc in (0, 1):
        got = _check_chunked(sp, ip, empty, x, 3, acc, 8, 5, "empty rows acc %d" % acc, 3)
        exact.assert_bits(got, exact.y0_values(300, 9) if acc else np.zeros(300), "empty rows")
    none = sp.CsMat.new((0, 40), np.zeros(1, np.uint32), np.zeros(0, np.uint32), np.zeros(0)).device()
    bufs = [_filled(dev, 2 * PAD) for _ in range(3)]
    assert _chunked(sp, none, x, PAD, bufs, 0, 4) == 0
    for b in bufs:
        _assert_target(b, 0, np.zeros(0), "0-row mirror")


def test_chunked_push_contract(sp):
    """A CSC mirror: STORAGE.  A null target, or a target whose 16-byte parity differs from
    d_y_bufs[0]: ARGUMENT, before anything is launched or written."""
    import torch
    from sprs_b200 import _lib
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    dev = G._device(ctx)
    ip, ind, data, cols = _small_matrix()
    rows = len(ip) - 1
    x = torch.from_numpy(np.ones(cols)).to(dev)
    csr = sp.CsMat.new((rows, cols), ip, ind, data)
    csc = csr.to_other_storage().device()
    bufs = [_filled(dev, rows + 2 * PAD) for _ in range(3)]
    launches = ctx.launches
    assert _chunked(sp, csc, x, PAD, bufs, 0, 4) == _lib.ERR_STORAGE
    mirror = csr.device()
    for bad in (1, 2):
        arr = (C.c_void_p * 3)(*[b.data_ptr() for b in bufs])
        arr[bad] = bufs[bad].data_ptr() + 8
        st = ctx.lib.sprs_b200_spmv_chunked_push_dev(ctx.h, mirror.h, C.c_void_p(x.data_ptr()), PAD, 3,
                                                     arr, 0, 4, G._stream_ptr())
        assert st == _lib.ERR_ARGUMENT, (bad, st)
        arr[bad] = None
        st = ctx.lib.sprs_b200_spmv_chunked_push_dev(ctx.h, mirror.h, C.c_void_p(x.data_ptr()), PAD, 3,
                                                     arr, 0, 4, G._stream_ptr())
        assert st == _lib.ERR_ARGUMENT, (bad, st)
    G._sync()
    assert ctx.launches == launches
    for b in bufs:
        _assert_target(b, 0, np.zeros(0), "untouched target")


# ================================================================ 2. multi-rank
def _n_devices():
    import torch
    return torch.cuda.device_count()


def _bounds_sets(sp, world, ip):
    """Named row cuts of the seam matrix for `world` ranks."""
    from sprs_b200.dist import nnz_balanced_bounds
    n = len(ip) - 1
    lens = np.diff(ip.astype(np.int64))
    hub = int(np.argmax(lens))
    assert lens[hub] > 64 * sp.SPMV_TILE  # its carry runs over many tiles
    if world == 2:
        return [("balanced rc8", nnz_balanced_bounds(ip, 2, row_cost=8.0)),
                ("empty first", [0, 0, n]), ("empty last", [0, n, n]),
                ("cut after hub", [0, hub + 1, n])]
    if world == 3:
        k = next(r for r in range(n // 2 | 1, n, 2) if lens[r] > 0)
        empty = np.flatnonzero(lens == 0)
        runs = np.split(empty, np.flatnonzero(np.diff(empty) != 1) + 1)
        run = max(runs, key=len)
        return [("1 row at odd %d" % k, [0, k, k + 1, n]),
                ("empty rows %d..%d" % (run[0], run[-1] + 1), [0, int(run[0]), int(run[-1]) + 1, n]),
                ("hub alone", [0, hub, hub + 1, n])]
    nb = nnz_balanced_bounds(ip, 6)
    return [("balanced", nnz_balanced_bounds(ip, 8)),
            ("two empty", [nb[0], nb[1], nb[1], nb[2], nb[3], nb[4], nb[4], nb[5], nb[6]])]


X_BOUNDS = {2: [[0, 3], [0, 0]], 3: [[0, 0, 7], [0, 1001, 1001]],
            8: [[0, 0, 3, 1001, 50001, 50001, 99999, 120000]]}


class _Rank:
    """A rank's check log: failures are collected (never raised) so every rank keeps making the
    same collective calls in the same order."""

    def __init__(self, sp, ctx, comm, dev):
        self.sp, self.ctx, self.comm, self.dev = sp, ctx, comm, dev
        self.failures, self.arms, self.cases = [], set(), 0

    def check(self, fn, *args):
        try:
            fn(*args)
        except AssertionError as e:
            self.failures.append(str(e)[:400])

    def agree(self, arr, what):
        """Every rank holds the same bits (digest all-gather through the communicator)."""
        self.cases += 1
        d = hashlib.sha256(np.ascontiguousarray(arr).tobytes()).digest()
        ds = self.comm.allgather(d)
        if len(set(ds)) != 1:
            self.failures.append("%s: ranks disagree (%s)" % (what, [x[:4].hex() for x in ds]))


def _block_mirrors(a, bounds):
    return [a.slice_outer(bounds[g], bounds[g + 1]).device() for g in range(len(bounds) - 1)]


def _per_block(ctx, mirrors, x):
    return np.concatenate([M.device_matvec(ctx, m)(x) for m in mirrors])


def _spmv_job(R, world, rank):
    """CommSpMV and CommHostSpMV over every bounds set of this world size."""
    import torch
    from oracle import oracle as O
    from sprs_b200.dist import CommHostSpMV, CommSpMV
    sp, ctx, comm, dev = R.sp, R.ctx, R.comm, R.dev
    ip, ind, dint = seam_matrix(sp)
    rows, cols = len(ip) - 1, SEAM_COLS
    dnorm = np.random.default_rng(3).standard_normal(len(ind))
    mats = {"int": sp.CsMat.new((rows, cols), ip, ind, dint),
            "normal": sp.CsMat.new((rows, cols), ip, ind, dnorm)}
    jc = np.arange(cols, dtype=np.int64)
    xs = {"int": [exact.x_values(jc, 5), exact.x_values(jc, 6)],
          "normal": [np.random.default_rng(s).standard_normal(cols) for s in (11, 12)]}
    for x in xs["int"]:
        exact.assert_exact_budget(O, ip, ind, dint, x)
    int_ref = [O.mul_acc_mat_vec_csr(ip, ind, dint, x, np.zeros(rows)) for x in xs["int"]]
    xd = {k: [torch.from_numpy(x).to(dev) for x in v] for k, v in xs.items()}
    for i, (bname, bounds) in enumerate(_bounds_sets(sp, world, ip)):
        r0, r1 = bounds[rank], bounds[rank + 1]
        blocks = {k: _block_mirrors(m, bounds) for k, m in mats.items()}
        refs = {"int": int_ref,
                "normal": [_per_block(ctx, blocks["normal"], x) for x in xs["normal"]]}
        for x, ref in zip(xs["int"], refs["int"]):  # the per-block concatenation is the whole product
            R.check(exact.assert_bits, _per_block(ctx, blocks["int"], x), ref, bname + " blocks vs oracle")
        for mode in ("fused", "push", "auto"):
            for mc in (False, True):
                for kind in ("int", "normal"):
                    op = CommSpMV(comm, blocks[kind][rank], bounds, rows, dev, exchange=mode, multicast=mc)
                    arm = mode + ("+mc" if op.multicast else "")
                    R.arms.add(arm)
                    for split in (False, True):
                        for rep in (0, 1):
                            what = "%s %s %s %s rep %d" % (bname, arm, kind, "split" if split else "step", rep)
                            op.y.fill_(float("nan"))  # a row never delivered, or stale, fails
                            torch.cuda.synchronize()
                            comm.barrier_host()
                            if split:  # bench.py's timed form
                                op.compute(xd[kind][rep])
                                op.exchange()
                            else:
                                op.step(xd[kind][rep])
                            comm.check()
                            got = op.y.cpu().numpy()
                            R.check(exact.assert_bits, got, refs[kind][rep], what)
                            R.agree(got, what)
                            comm.barrier_host()
                    op.close()
        # host vectors: x uploaded in uneven slices, one of them empty, one at an odd column
        xb = X_BOUNDS[world][i % len(X_BOUNDS[world])] + [cols]
        for kind in ("int", "normal"):
            hop = CommHostSpMV(comm, blocks[kind][rank], bounds, cols, multicast=True, x_bounds=xb)
            for rep in (0, 1):
                hx = torch.from_numpy(xs[kind][rep][xb[rank]:xb[rank + 1]].copy()).pin_memory()
                hy = torch.full((max(r1 - r0, 1),), float("nan"), dtype=torch.float64).pin_memory()
                hop.step(hx.data_ptr(), hy.data_ptr())
                what = "%s host %s x %s rep %d" % (bname, kind, xb, rep)
                got = hy[:r1 - r0].numpy().copy()
                R.check(exact.assert_bits, got, refs[kind][rep][r0:r1], what)
                R.cases += 1
            hop.close()
        del blocks
    # contract cases: every rank makes the same failing call; nothing is launched
    from sprs_b200 import _lib
    from sprs_b200.dist import _stream_ptr
    bounds = _bounds_sets(sp, world, ip)[0][1]
    op = CommSpMV(comm, _block_mirrors(mats["int"], bounds)[rank], bounds, rows, dev)
    launches = ctx.launches
    x0 = C.c_void_p(xd["int"][0].data_ptr())
    st = ctx.lib.sprs_b200_spmv_rowpart(comm.h, op.mirror.h, x0, op.buf.h, op.bounds[rank], 3,
                                        _stream_ptr(dev))
    if st != _lib.ERR_ARGUMENT:
        R.failures.append("unknown exchange mode: status %d, want ARGUMENT" % st)
    st = ctx.lib.sprs_b200_spmv_rowpart(comm.h, op.mirror.h, x0, op.buf.h, rows + 3, 1, _stream_ptr(dev))
    if st != _lib.ERR_DIMENSION:
        R.failures.append("row block past y: status %d, want DIMENSION" % st)
    if ctx.launches != launches:
        R.failures.append("contract cases launched %d kernels" % (ctx.launches - launches))
    op.close()


def _bicgstab_job(R, world, rank):
    """row_partitioned_bicgstab over two alternating CommSpMV (fused, then push) against the host
    model with the per-block device matvec and the solver's reduction order."""
    import torch
    from sprs_b200.dist import CommSpMV, nnz_balanced_bounds, row_partitioned_bicgstab
    from sprs_b200.linalg import NotConverged
    sp, ctx, comm, dev = R.sp, R.ctx, R.comm, R.dev
    sm = ctx.sm_count
    full = M.CHUNK * M.RED_THREADS * M.grid_cap(sm)
    n = 2 * full + 3  # tail of 3, every thread 2+ chunks, all of the grid's partials
    need = {"tail of 3", "thread with 2+ chunks"} | ({"more than 256 partials"}
                                                      if M.grid_cap(sm) > M.RED_THREADS else set())
    if not need <= M.seams(n, sm):
        R.failures.append("n = %d misses %s" % (n, need - M.seams(n, sm)))
    csr, x0, b = M.dominant_system(n, 17 + world)
    a = sp.CsMat.new((n, n), *csr)
    if world == 2:
        bounds = nnz_balanced_bounds(csr[0], 2)
        bounds[1] |= 1  # an odd offset
    else:
        cut = nnz_balanced_bounds(csr[0], 2)[1]
        bounds = [0, cut, cut, n]
    blocks = _block_mirrors(a, bounds)
    ops = [CommSpMV(comm, blocks[rank], bounds, n, dev, exchange=ex) for ex in ("fused", "push")]
    solver = row_partitioned_bicgstab(ctx, ops, n, x0, b, dev)
    model = None
    if rank == 0:
        model = M.Model(lambda v: _per_block(ctx, blocks, v), M.device(M.grid_for(n, sm)), x0, b)

    def compare(what):
        state = [solver.x(), solver.r(), solver.rhat(), solver.p(),
                 np.array([solver.err(), solver.rho()]),
                 np.array([solver.iteration_count(), solver.soft_restart_count(),
                           solver.hard_restart_count()], dtype=np.float64)]
        if model is not None:
            R.check(M.assert_same_state, solver, model, what)
        R.agree(np.concatenate(state), what)

    compare("new")
    for it in range(1, 11):
        solver.step()
        if model is not None:
            model.step()
        compare("step %d" % it)
    solver.soft_restart()
    if model is not None:
        model.soft_restart()
    compare("soft restart")
    solver.hard_restart()
    if model is not None:
        model.hard_restart()
    compare("hard restart")
    try:
        solver.run(1e-9, 300)
        ok = True
    except NotConverged:
        ok = False
    if model is not None:
        ok_model = model.run(1e-9, 300)
        if not (ok and ok_model):
            R.failures.append("solve: device Ok=%s, model Ok=%s" % (ok, ok_model))
    compare("solve")
    solver.free()
    torch.cuda.synchronize()
    for op in ops:
        op.close()


JOBS = {"spmv": _spmv_job, "bicgstab": _bicgstab_job}


def _rank_main(rank, world, q_id, q_out, ndev, job):
    sys.path.insert(0, ROOT)
    try:
        import torch
        import sprs_b200 as sp
        from sprs_b200.dist import Comm
        device = rank % ndev
        torch.cuda.set_device(device)
        ctx = sp.Context.default(device)
        comm = Comm(ctx, q_id.get(timeout=120), rank, world)
        R = _Rank(sp, ctx, comm, torch.device("cuda", device))
        JOBS[job](R, world, rank)
        report = {"failures": R.failures, "arms": sorted(R.arms), "cases": R.cases,
                  "multicast_supported": comm.multicast}
        comm.close()
        q_out.put((rank, report))
    except BaseException as e:  # report instead of leaving the parent to time out
        q_out.put((rank, {"error": repr(e), "trace": traceback.format_exc()[-2000:]}))


def _run_ranks(world, job, timeout=900):
    import torch.multiprocessing as mp
    from sprs_b200.dist import Comm
    ndev = max(1, _n_devices())
    mpc = mp.get_context("spawn")
    q_id, q_out = mpc.Queue(), mpc.Queue()
    cid = Comm.unique_id()
    for _ in range(world):
        q_id.put(cid)
    procs = [mpc.Process(target=_rank_main, args=(r, world, q_id, q_out, ndev, job)) for r in range(world)]
    res = {}
    try:
        for p in procs:
            p.start()
        for _ in procs:
            r, rep = q_out.get(timeout=timeout)
            res[r] = rep
        for p in procs:
            p.join(timeout=60)
    finally:
        for p in procs:
            p.kill()
            p.join()
    for r in range(world):
        assert "error" not in res[r], (r, res[r])
        assert not res[r]["failures"], (r, res[r]["failures"][:10])
        assert res[r]["cases"] > 0
    # the multicast arm must really run where the communicator supports it
    if job == "spmv" and ndev >= 2 and res[0]["multicast_supported"]:
        assert any(a.endswith("+mc") for a in res[0]["arms"]), res[0]["arms"]
    print("world %d, %d devices, arms %s, %d checked cases per rank"
          % (world, ndev, res[0]["arms"], res[0]["cases"]))
    return res


@pytest.mark.parametrize("world", [2, 3, 8])
def test_comm_rowpart_bounds_sets_bits(world):
    """Every bounds set x exchange mode x multicast x (step | compute + exchange) x integer /
    N(0,1) values, two different x: each rank's whole y bit-exact and equal across ranks; then
    CommHostSpMV with uneven x slices and the contract cases."""
    _run_ranks(world, "spmv")


@pytest.mark.parametrize("env", [("SPRS_B200_SPMV_HOT", "24576", 2),
                                 ("SPRS_B200_FORCE_INDPTR64", "1", 3)], ids=["hot", "indptr64"])
def test_comm_rowpart_variants_child_process(env, monkeypatch):
    """The same with the multi-target hot-set kernel forced (a hot set of 24576 columns) and with
    64-bit indptr mirrors; the switches are read once per process, so the ranks start with them.
    The library has no accessor for a mirror's hot set, so this does not check that one was built:
    a block without non-zeros never gets one, and a build that cannot allocate its buffers leaves
    the mirror on the plain multi-target kernel."""
    name, value, world = env
    monkeypatch.setenv(name, value)
    _run_ranks(world, "spmv")


@pytest.mark.parametrize("world", [2, 3])
def test_comm_rowpart_bicgstab_bits(world):
    """row_partitioned_bicgstab with two alternating CommSpMV (world 2 cut at an odd row, world 3
    with an empty block): after new, each of 10 steps, the restarts and a solve ending Ok, every
    rank's x, r, rhat, p, err, rho and counters equal the host model and each other."""
    _run_ranks(world, "bicgstab")
