"""CPU model (NOT a measurement) of the x-gather locality of BASELINE config 5.

Samples row blocks of this repo's R-MAT definition (sprs_b200/generate.py: Graph500
a,b,c,d = .57,.19,.19,.05, scale 24, n = 1e7, ~100 nnz/row), walks the non-zeros the way the
SpMV kernel does (32 consecutive non-zeros per warp gather instruction) and counts, per
non-zero, the distinct 128-byte lines (L1TEX wavefronts) and 32-byte sectors (L2->SM traffic)
the x gathers touch -- with and without a cache of the K most frequent columns.
The no-cache figures can be checked against ncu's L1TEX / L2 sector counts of the SpMV kernel.
"""
import sys

import numpy as np

SCALE, N, NNZ = 24, 10_000_000, 1.0e9
A, B, C_, D = 0.57, 0.19, 0.19, 0.05


def sample_rows(rng, n_blocks, block_rows):
    out = []
    for _ in range(n_blocks):
        # blocks are drawn UNIFORMLY over the rows: each row's weight is its own non-zero count
        # below (drawing blocks with R-MAT's row bias as well would count that bias twice and
        # understate the share of the hot columns)
        r0 = int(rng.integers(0, N // block_rows)) * block_rows
        for r in range(r0, min(r0 + block_rows, N)):
            rb = np.array([(r >> (SCALE - 1 - i)) & 1 for i in range(SCALE)], dtype=bool)
            k = int(rb.sum())
            p_r = (A + B) ** (SCALE - k) * (C_ + D) ** k
            lam = NNZ * 1.06 * p_r
            cnt = rng.poisson(lam)
            if cnt == 0:
                out.append(np.zeros(0, dtype=np.int64))
                continue
            pc = np.where(rb, D / (C_ + D), B / (A + B))          # P(col bit = 1 | row bit)
            cols = np.zeros(cnt, dtype=np.int64)
            for i in range(SCALE):
                cols = (cols << 1) | (rng.random(cnt) < pc[i])
            cols = np.unique(cols[cols < N])
            out.append(cols)
    return out


def popcount(v):
    v = v.copy()
    c = np.zeros_like(v)
    while np.any(v):
        c += v & 1
        v >>= 1
    return c


def main():
    rng = np.random.default_rng(int(sys.argv[1]) if len(sys.argv) > 1 else 1)
    rows = sample_rows(rng, n_blocks=int(sys.argv[2]) if len(sys.argv) > 2 else 400, block_rows=16)
    stream = np.concatenate(rows)
    nnz = len(stream)
    pad = (-nnz) % 32
    grp = np.concatenate([stream, np.full(pad, -1, dtype=np.int64)]).reshape(-1, 32)
    valid = grp >= 0
    pc = popcount(np.where(valid, grp, 0))
    print(f"sampled {len(rows)} rows, {nnz} nnz, mean row {nnz / len(rows):.1f}")

    def distinct(keys, mask):
        big = np.where(mask, keys, -1 - np.arange(32)[None, :] * 0)  # masked lanes -> -1
        s = np.sort(big, axis=1)
        d = (s[:, 1:] != s[:, :-1]) & (s[:, 1:] >= 0)
        first = s[:, 0] >= 0
        return d.sum() + first.sum()

    base_lines = distinct(grp >> 4, valid)
    base_sect = distinct(grp >> 2, valid)
    print(f"no cache      : {base_lines / nnz:.3f} lines/nnz  {base_sect / nnz:.3f} sectors/nnz "
          f"-> L2->SM bytes/nnz = {12 + 32 * base_sect / nnz:.1f}")
    # hot set = columns with popcount <= kmax (the K most probable columns, up to ties)
    from math import comb
    for kmax in (2, 3, 4, 5):
        K = sum(comb(SCALE, j) for j in range(kmax + 1))
        hot = valid & (pc <= kmax)
        cold = valid & ~hot
        lines = distinct(grp >> 4, cold)
        sect = distinct(grp >> 2, cold)
        # shared-memory side: wavefronts ~ max lanes per bank pair (8-byte words, 32 x 4-byte banks:
        # 16 distinct 8-byte bank slots per half... model: one wavefront per 16 hot lanes at best,
        # conflicts counted as the max multiplicity of (slot mod 16) among hot lanes
        print(f"hot popcount<={kmax} (K={K:6d}, {K * 8 / 1024:6.1f} KB): hot share {hot.sum() / nnz:.3f}  "
              f"cold {lines / nnz:.3f} lines/nnz {sect / nnz:.3f} sectors/nnz "
              f"-> L2->SM bytes/nnz = {12 + 32 * sect / nnz:.1f}")


if __name__ == "__main__":
    main()
