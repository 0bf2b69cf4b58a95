"""Host model of the SpMV's summation order (csrc/spmv.cu), so that y = A x and y += A x can be
compared BIT FOR BIT with the device for any values, not only integer ones.

The order depends only on indptr and the two cut constants (sprs_b200.SPMV_TILE, SPMV_ROW_COST):
not on the grid, the hot set, the number of targets or the indptr width.  The partition is
sprs_b200.spmv_rows_cut_by_tiles; the rest restates rows_direct, sink_row, spmv_fixup_kernel and
apply_carries_ending_in:

  segments  tile t owns rows tile_row[t] .. r_last (r_last = tile_row[t+1] if that is < rows, else
            rows - 1), each clamped to [tile_k[t], tile_k[t+1]);
  G         once per tile from cnt = k1 - k0 and nr = r_last - r0 + 1: 4 lanes per row if
            cnt <= 24 nr, 8 if <= 48 nr, 16 if <= 96 nr, else 32;
  tiny      a segment of at most 2U = 8 non-zeros (empty ones included) is summed by one lane in
            storage order from +0.0 -- or, accumulating, from y[r] when no tile carries the row
            (every row of the tile but r0, and r0 in tile 0), which is then stored as is;
  long      G < 32 and more than 4 G U = 16 G non-zeros: the whole warp takes the segment;
  lanes     with L lanes (G, or 32 for a long segment), lane l sums elements s + l, s + l + L, ...
            in order from +0.0, then the xor butterfly L/2, ..., 1 combines them;
  sink      a row r < tile_row[t+1] is stored as the sum, or y0 + sum under accumulate (tiny rows
            that started from y excepted); the segment of row tile_row[t+1] is carry[t] (an empty
            one stores +0.0);
  fix-up    each run of tiles with the same carry row is summed in tile order from the run's head,
            then y[row] = y[row] + that sum.  The tile-range form (spmv_launch_tile_range) adds the
            carries of the rows that end in each range after it, in the same order.

So the accumulating forms carry the reference's bits ((y0 + p0) + p1) + ... on every tiny row no
tile carries; longer rows and carried rows are y0 + partial (+ carries).

Every product and every sum is one numpy operation on float64 arrays (one rounding each; numpy
never fuses), with masks wherever a lane has nothing to add: a running sum that may start from
y0 = -0.0 must not meet a +0.0 pad.  No np.sum / np.dot / `@`.  Indices, data and the gathered x
are taken one tile range at a time, so a matrix of 1e9 non-zeros needs no 8 GB temporaries.

`literal` is a lane-by-lane loop transcription of the same kernels for small inputs; the test
suite pins the vectorised model to it.

Test helper, not part of the package."""
import math

import numpy as np

U = 4                          # SPMV_LOADS_IN_FLIGHT: loads of each kind in flight per lane
TINY = 2 * U                   # sweep 1: segments of at most 8 non-zeros, one lane each
G_LIMITS = ((24, 4), (48, 8), (96, 16))   # cnt <= f * nr -> G lanes per row; otherwise 32
LONG = 4 * U                   # G < 32 and a segment longer than LONG * G: the whole warp
WARP = 32
BLOCK_ROWS = 31                # rows_direct: row boundaries come 31 rows at a time
CHUNK_NNZ = 1 << 24            # non-zeros per tile range the vectorised model holds at once


def partition(indptr):
    """(ip, tile_row, tile_k), int64, ip rebased to start at 0."""
    import sprs_b200 as sp
    ip = np.asarray(indptr).astype(np.int64)
    ip = ip - ip[0]
    _, tr, tk = sp.spmv_rows_cut_by_tiles(ip, tiles=True)
    return ip, tr, tk


def tile_lanes(cnt, nr):
    """G of each tile."""
    g = np.full(np.shape(cnt), WARP, dtype=np.int64)
    for f, lanes in reversed(G_LIMITS):
        g = np.where(cnt <= f * nr, lanes, g)
    return g


class _Segments:
    """Every (tile, row) segment of tiles [t0, t1)."""

    def __init__(self, ip, tr, tk, t0, t1):
        rows = len(ip) - 1
        r0, r1 = tr[t0:t1], tr[t0 + 1:t1 + 1]
        r_last = np.where(r1 < rows, r1, r1 - 1)
        nr = r_last - r0 + 1
        g = tile_lanes(tk[t0 + 1:t1 + 1] - tk[t0:t1], nr)
        self.tile = np.repeat(np.arange(t0, t1, dtype=np.int64), nr)
        start = np.cumsum(nr) - nr
        self.row = np.repeat(r0, nr) + (np.arange(int(nr.sum()), dtype=np.int64) - np.repeat(start, nr))
        k0, k1 = tk[self.tile], tk[self.tile + 1]
        self.s = np.maximum(ip[self.row], k0)
        self.e = np.maximum(np.minimum(ip[self.row + 1], k1), self.s)
        n = self.e - self.s
        self.g = np.repeat(g, nr)
        self.lanes = np.where(n <= TINY, 1, np.where((self.g < WARP) & (n > LONG * self.g), WARP, self.g))
        self.carry = self.row >= tr[self.tile + 1]             # the tile's carry row
        # row r0 of every tile but tile 0 is the previous tile's carry row
        self.carried = self.carry | ((self.row == tr[self.tile]) & (self.tile > 0))


def _lane_sums(prod, base, s, e, L, start):
    """Sums of segments [s, e) (absolute non-zero positions; prod holds base ..) over L lanes of
    stride L, lane sums from `start` (lane 0; +0.0 elsewhere), then the xor butterfly."""
    m = len(s)
    if m == 0:
        return np.zeros(0)
    n = e - s
    order = np.argsort(-n, kind="stable")
    ns, ss = n[order], s[order] - base
    acc = np.zeros((m, L))
    acc[:, 0] = start[order]
    neg = -ns
    lane = np.arange(L, dtype=np.int64)
    for j in range(-(-int(ns[0]) // L)):
        p = int(np.searchsorted(neg, -j * L, side="left"))      # segments with more than j*L
        off = j * L + lane
        mask = off[None, :] < ns[:p, None]
        sub = acc[:p]
        sub[mask] = sub[mask] + prod[(ss[:p, None] + off[None, :])[mask]]
    o = L // 2
    while o:
        acc[:, :o] = acc[:, :o] + acc[:, o:2 * o]
        o //= 2
    out = np.empty(m)
    out[order] = acc[:, 0]
    return out


def _run_sums(carry, heads, lens):
    """carry[h] + carry[h+1] + ... (len terms, in tile order) for every run."""
    acc = carry[heads].copy()
    if len(heads) == 0:
        return acc
    order = np.argsort(-lens, kind="stable")
    hs, ls = heads[order], lens[order]
    neg = -ls
    s = acc[order]
    for j in range(1, int(ls[0])):
        p = int(np.searchsorted(neg, -j, side="left"))        # runs longer than j
        s[:p] = s[:p] + carry[hs[:p] + j]
    acc[order] = s
    return acc


def _kernel(ip, indices, data, x, tr, tk, t0, t1, y, carry, accumulate):
    """spmv_rows_kernel over tiles [t0, t1): y rows and carry[t0:t1], in place."""
    ta = t0
    while ta < t1:  # tile ranges of at most CHUNK_NNZ non-zeros (at least one tile)
        tb = int(np.searchsorted(tk, tk[ta] + CHUNK_NNZ, side="right")) - 1
        tb = min(max(tb, ta + 1), t1)
        seg = _Segments(ip, tr, tk, ta, tb)
        base, end = int(tk[ta]), int(tk[tb])
        cols = np.asarray(indices[base:end]).astype(np.int64)
        prod = np.asarray(data[base:end], dtype=np.float64) * x[cols]
        from_y = (seg.lanes == 1) & ~seg.carried if accumulate else np.zeros(len(seg.row), bool)
        sums = np.empty(len(seg.row))
        for L in (1, 4, 8, 16, WARP):
            sel = np.flatnonzero(seg.lanes == L)
            start = np.where(from_y[sel], y[seg.row[sel]], 0.0)
            sums[sel] = _lane_sums(prod, base, seg.s[sel], seg.e[sel], L, start)
        own = ~seg.carry
        r = seg.row[own]
        if accumulate:
            sums[own] = np.where(from_y[own], sums[own], y[r] + sums[own])
        y[r] = sums[own]
        carry[seg.tile[seg.carry]] = sums[seg.carry]
        ta = tb


def _fixup(tr, carry, y, n_tiles):
    """spmv_fixup_kernel: the runs of equal carry rows tile_row[t+1], t < n_tiles - 1."""
    if n_tiles < 2:
        return
    cr = tr[1:n_tiles]
    heads = np.flatnonzero(np.concatenate(([True], cr[1:] != cr[:-1])))
    lens = np.diff(np.concatenate((heads, [len(cr)])))
    rows = cr[heads]
    y[rows] = y[rows] + _run_sums(carry, heads, lens)


def _carries_ending_in(tr, carry, y, u0, u1):
    """spmv_fixup_range_kernel: rows tile_row[u] that end in tile u, u in [max(u0, 1), u1)."""
    u = np.arange(max(u0, 1), u1, dtype=np.int64)
    u = u[tr[u + 1] != tr[u]]
    if len(u) == 0:
        return
    row = tr[u]
    f = np.searchsorted(tr[1:], row, side="left") + 1          # first f >= 1 with tile_row[f] >= row
    y[row] = y[row] + _run_sums(carry, f - 1, u - f + 1)


def spmv(indptr, indices, data, x, y0=None, tile_ranges=None):
    """y = A x (y0 None) or y = y0 + A x in the SpMV's order.  tile_ranges = [0, t1, ..., n_tiles]:
    the tile-range form (each range's kernel, then the carries of the rows that end in it).
    indptr may be a row slice's (not starting at 0): indices / data hold the slice's non-zeros,
    entry k of the slice at k - indptr[0], as sprs stores a view."""
    ip, tr, tk = partition(indptr)
    rows = len(ip) - 1
    y = np.zeros(rows) if y0 is None else np.array(y0, dtype=np.float64)
    if rows == 0:
        return y
    x = np.asarray(x, dtype=np.float64)
    n_tiles = len(tr) - 1
    carry = np.zeros(n_tiles)
    with np.errstate(all="ignore"):
        if tile_ranges is None:
            _kernel(ip, indices, data, x, tr, tk, 0, n_tiles, y, carry, y0 is not None)
            _fixup(tr, carry, y, n_tiles)
        else:
            assert tile_ranges[0] == 0 and tile_ranges[-1] == n_tiles
            for a, b in zip(tile_ranges[:-1], tile_ranges[1:]):
                _kernel(ip, indices, data, x, tr, tk, a, b, y, carry, y0 is not None)
                _carries_ending_in(tr, carry, y, a, b)
    return y


def n_tiles(indptr):
    return len(partition(indptr)[1]) - 1


def storage_order_rows(indptr):
    """Rows the kernel sums in storage order from their start value (+0.0, or y0 under
    accumulate): the tiny rows no tile carries.  They carry the reference's bits."""
    ip, tr, tk = partition(indptr)
    seg = _Segments(ip, tr, tk, 0, len(tr) - 1)
    out = np.zeros(len(ip) - 1, dtype=bool)
    out[seg.row[(seg.lanes == 1) & ~seg.carried]] = True
    return out


def tree_depth(indptr):
    """Per row, an upper bound on the additions any one term passes through in the model's order
    (lane steps + butterfly + the y0 add + the carries of its run + the fix-up's add)."""
    ip, tr, tk = partition(indptr)
    rows = len(ip) - 1
    seg = _Segments(ip, tr, tk, 0, len(tr) - 1)
    n = seg.e - seg.s
    d = -(-n // seg.lanes) + np.log2(seg.lanes).astype(np.int64)
    depth = np.zeros(rows, dtype=np.int64)
    np.maximum.at(depth, seg.row, d)
    runs = np.bincount(seg.row[seg.carry], minlength=rows)
    return depth + runs + 2


# ---------------------------------------------------------------- literal transcription
def literal(indptr, indices, data, x, y0=None):
    """rows_direct + sink_row + spmv_fixup_kernel, lane by lane, with Python floats (IEEE double,
    one rounding per operation).  Small inputs only."""
    ip, tr, tk = partition(indptr)
    ip, tr, tk = ip.tolist(), tr.tolist(), tk.tolist()
    rows = len(ip) - 1
    accumulate = y0 is not None
    y = [0.0] * rows if y0 is None else [float(v) for v in y0]
    if rows == 0:
        return np.array(y)
    ind = np.asarray(indices).astype(np.int64)[:ip[-1]].tolist()
    dat = np.asarray(data, dtype=np.float64)[:ip[-1]].tolist()
    xs = np.asarray(x, dtype=np.float64).tolist()
    n_t = len(tr) - 1
    carry = [0.0] * n_t

    def p(q):
        return dat[q] * xs[ind[q]]

    def butterfly(acc):
        o = len(acc) // 2
        while o:
            acc = [acc[i] + acc[i ^ o] for i in range(len(acc))]
            o //= 2
        return acc[0]

    for t in range(n_t):
        r0, r1, k0, k1 = tr[t], tr[t + 1], tk[t], tk[t + 1]

        def sink(r, total, from_y=False):
            if r < r1:
                y[r] = y[r] + total if accumulate and not from_y else total
            else:
                carry[t] = total

        r_last = r1 if r1 < rows else r1 - 1
        cnt, nr = k1 - k0, r_last - r0 + 1
        G = 4 if cnt <= 24 * nr else 8 if cnt <= 48 * nr else 16 if cnt <= 96 * nr else 32
        for rbase in range(r0, r_last + 1, BLOCK_ROWS):
            b = [ip[rbase + L] if rbase + L <= r_last + 1 else 0 for L in range(WARP)]
            nrows = min(r_last - rbase + 1, BLOCK_ROWS)
            tiny = [False] * WARP
            for lane in range(nrows):  # sweep 1
                ms, me = max(b[lane], k0), min(b[lane + 1], k1)
                me = max(me, ms)
                tiny[lane] = me - ms <= TINY
                if not tiny[lane]:
                    continue
                rl = rbase + lane
                from_y = accumulate and rl < r1 and (rl > r0 or (r0 == 0 and k0 == 0))
                acc = y[rl] if from_y else 0.0
                for q in range(ms, me):
                    acc = acc + p(q)
                sink(rl, acc, from_y)
            todo = [j for j in range(nrows) if not tiny[j]]
            while todo:  # sweeps 2 and 3: 32 / G rows per pass, lowest lane first
                batch, todo = todo[:WARP // G], todo[WARP // G:]
                longs = []
                for j in batch:
                    s, e = max(b[j], k0), min(b[j + 1], k1)
                    e = max(e, s)
                    if G < WARP and e - s > LONG * G:
                        longs.append((j, s, e))
                        continue
                    acc = [0.0] * G
                    for gl in range(G):
                        for q in range(s + gl, e, G):
                            acc[gl] = acc[gl] + p(q)
                    sink(rbase + j, butterfly(acc))
                for j, s, e in longs:
                    acc = [0.0] * WARP
                    for lane in range(WARP):
                        for q in range(s + lane, e, WARP):
                            acc[lane] = acc[lane] + p(q)
                    sink(rbase + j, butterfly(acc))
    for t in range(n_t - 1):  # spmv_fixup_kernel
        row = tr[t + 1]
        if t > 0 and tr[t] == row:
            continue
        end = t + 1
        while tr[end + 1] <= row:
            end += 1
        total = carry[t]
        for u in range(t + 1, end):
            total = total + carry[u]
        y[row] = y[row] + total
    return np.array(y)


# ---------------------------------------------------------------- seams
ALL_SEAMS = ("tiny row from y", "tiny segment of a carried row", "G=4 rows", "G=8 rows",
             "G=16 rows", "G=32 rows", "whole-warp row", "cut row with a tiny tail",
             "row starting on a cut", "carry run of 1", "carry run of 2", "carry run of > 64")


def seams(indptr):
    """How many segments / runs of the matrix take each path of ALL_SEAMS."""
    ip, tr, tk = partition(indptr)
    seg = _Segments(ip, tr, tk, 0, len(tr) - 1)
    tiny = seg.lanes == 1
    first = ~seg.carry & seg.carried                          # row r0 of a tile t > 0
    out = {"tiny row from y": int((tiny & ~seg.carried).sum()),
           "tiny segment of a carried row": int((tiny & seg.carried).sum())}
    for G in (4, 8, 16, 32):
        out["G=%d rows" % G] = int(((seg.lanes == G) & (seg.g == G)).sum())
    out["whole-warp row"] = int(((seg.lanes == WARP) & (seg.g < WARP)).sum())
    out["cut row with a tiny tail"] = int((first & tiny & (ip[seg.row] < tk[seg.tile])).sum())
    out["row starting on a cut"] = int((first & (ip[seg.row] == tk[seg.tile])).sum())
    n_t = len(tr) - 1
    cr = tr[1:n_t]
    runs = np.diff(np.flatnonzero(np.concatenate(([True], cr[1:] != cr[:-1], [True])))) \
        if n_t > 1 else np.zeros(0, np.int64)
    out["carry run of 1"] = int((runs == 1).sum())
    out["carry run of 2"] = int((runs == 2).sum())
    out["carry run of > 64"] = int((runs > 64).sum())
    return out


def gamma(n):
    """Higham's gamma_n = n u / (1 - n u), u = 2^-53."""
    nu = np.asarray(n, dtype=np.float64) * 2.0 ** -53
    return nu / (1.0 - nu)


def fsum_rows(indptr, indices, data, x, y0=None):
    """Per row: math.fsum of the products (and y0) -- the correctly rounded sum -- and the sum
    of their magnitudes."""
    ip = np.asarray(indptr).astype(np.int64)
    ip = ip - ip[0]
    prod = np.asarray(data, dtype=np.float64)[:ip[-1]] * \
        np.asarray(x)[np.asarray(indices).astype(np.int64)[:ip[-1]]]
    rows = len(ip) - 1
    exact, mag = np.zeros(rows), np.zeros(rows)
    for r in range(rows):
        terms = prod[ip[r]:ip[r + 1]].tolist() + ([float(y0[r])] if y0 is not None else [])
        exact[r] = math.fsum(terms)
        mag[r] = math.fsum(abs(t) for t in terms)
    return exact, mag
