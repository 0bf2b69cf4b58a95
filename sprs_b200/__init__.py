"""sprs_b200 -- H100-native (sm_90a) implementation of the sprs sparse-product hot
path (SpMV / SpMM / SpGEMM) behind sprs's operator API.  See DESIGN.md.

Nothing here computes on the CPU: every product is a call into libsprs_b200.so
(hand-written CUDA).  Importing works without a GPU (so the ABI can be inspected);
creating a Context without one raises ThirdPartyError.
"""
from . import _lib, construct, io, ldl, linalg
from .construct import bmat, hstack, kronecker_product, vstack
from .ldl import is_symmetric
from .sparse import (CSC, CSR, Context, CsMat, CsVec, DeviceCsMat, SingularMatrix, SprsPanic,
                     ThirdPartyError, assign_to_dense, binop, csmat_mul_csmat, prod, smmp)

__all__ = ["CSC", "CSR", "Context", "CsMat", "CsVec", "DeviceCsMat", "SingularMatrix", "SprsPanic",
           "ThirdPartyError", "assign_to_dense", "binop", "bmat", "construct", "csmat_mul_csmat", "hstack",
           "is_symmetric", "kronecker_product", "prod", "smmp", "vstack", "_lib", "io", "ldl",
           "linalg"]
CONSTRUCT_TILE = 2048  # output entries per warp tile of the construction kernels (csrc/construct.cu)
DENSE_TILE = 4096      # positions per warp tile of the dense-boundary kernels (csrc/transpose.cu)
SCATTER_TILE = 256     # stored entries per warp tile of assign_to_dense (csrc/transpose.cu)
__version__ = "0.1.0"
import os as _os

_v = (_os.environ.get("SPRS_B200_SPMV_VARIANT", "") + ",").split(",")   # "w,row_cost" (csrc/spmv.cu)
SPMV_TILE = int(_v[0]) if _v[0] else 1024      # cost units per SpMV warp tile
SPMV_ROW_COST = int(_v[1]) if _v[1] else 16    # cost of one row end, in non-zeros


def spmv_rows_cut_by_tiles(indptr, tiles=False):
    """Boolean mask of the rows a merge-path tile boundary of the SpMV cuts (csrc/spmv.cu
    tile_cut_kernel restated in numpy): the cut of tile t is where nnz + SPMV_ROW_COST * rows
    reaches t * SPMV_TILE.  Tests use it: a cut row adds two partial sums, so only the rows it
    spares carry the storage-order (bit-exact) promise for rows of at most 8 non-zeros.
    tiles=True also returns the kernel's partition arrays (tile_row, tile_k), n_tiles + 1 entries
    each (int64): tile t covers non-zeros [tile_k[t], tile_k[t+1]) and rows tile_row[t] ..
    tile_row[t+1], the last one only up to tile_k[t+1] (its carry row when that is < rows)."""
    import numpy as np
    ip = np.asarray(indptr).astype(np.int64)
    ip = ip - ip[0]
    rows = len(ip) - 1
    f = ip + SPMV_ROW_COST * np.arange(rows + 1)
    total = int(f[-1])
    d = np.arange(0, total, SPMV_TILE, dtype=np.int64)[1:]       # cuts 1 .. n_tiles-1
    r = np.searchsorted(f, d, side="right") - 1                     # largest r with f[r] <= d
    k = np.minimum(d - SPMV_ROW_COST * r, ip[np.minimum(r + 1, rows)])
    inside = (k > ip[r]) & (k < ip[np.minimum(r + 1, rows)])        # strictly inside row r
    cut = np.zeros(rows, dtype=bool)
    cut[r[inside & (r < rows)]] = True
    if not tiles:
        return cut
    # cut 0 is the start of the path, cut n_tiles its end (n_tiles = 1 for an empty path)
    tile_row = np.concatenate([[0], r, [rows]]).astype(np.int64)
    tile_k = np.concatenate([[0], k, [int(ip[-1])]]).astype(np.int64)
    return cut, tile_row, tile_k


BINOP_TILE = 1024      # cost units per binop warp tile (csrc/binop.cu)
BINOP_LANE_COST = 32   # cost units per lane of a tile
BINOP_ROW_COST = 16    # cost of one outer dimension's end


def binop_cuts(a, b, d):
    """The binop's merge-path cuts (csrc/binop.cu cut_at restated in numpy, one cut per entry
    of the cost positions d): a, b = (indptr, indices) of the two operands.  Returns (r, ka, kb)
    int64 arrays: rows passed and entries of A / B consumed, the split snapped so that an equal
    pair A[ka-1] == B[kb] is never separated.  `snapped` (4th array) marks the cuts the snap
    moved.  Tests use it to assert that a matrix puts a cut where they want one."""
    import numpy as np
    ipa = np.asarray(a[0]).astype(np.int64)
    ipb = np.asarray(b[0]).astype(np.int64)
    ia, ib = np.asarray(a[1]).astype(np.int64), np.asarray(b[1]).astype(np.int64)
    outer = len(ipa) - 1
    w = ipa + ipb + BINOP_ROW_COST * np.arange(outer + 1)
    d = np.asarray(d, dtype=np.int64)
    r = np.searchsorted(w, d, side="right") - 1
    ka, kb, snapped = ipa[r].copy(), ipb[r].copy(), np.zeros(d.size, dtype=bool)
    for i in np.flatnonzero(r < outer):
        ri = r[i]
        ra, rb = ia[ipa[ri]:ipa[ri + 1]], ib[ipb[ri]:ipb[ri + 1]]
        k = min(int(d[i] - w[ri]), len(ra) + len(rb))
        # ja = A entries among the first k of the stable merge, A first on equal indices
        order = np.argsort(np.concatenate([ra * 2, rb * 2 + 1]), kind="stable")
        ja = int(np.count_nonzero(order[:k] < len(ra)))
        jb = k - ja
        if ja > 0 and jb < len(rb) and ra[ja - 1] == rb[jb]:
            jb += 1
            snapped[i] = True
        ka[i], kb[i] = ipa[ri] + ja, ipb[ri] + jb
    return r, ka, kb, snapped


def binop_tiles(a, b):
    """Every tile and lane boundary of the binop on (a, b): the cost positions (tile t starts at
    t * BINOP_TILE, lane l of it BINOP_LANE_COST * l later, the end of the path last) and their
    cuts (binop_cuts)."""
    import numpy as np
    outer = len(a[0]) - 1
    total = int(a[0][-1] - a[0][0]) + int(b[0][-1] - b[0][0]) + BINOP_ROW_COST * outer
    d = np.concatenate([np.arange(0, total, BINOP_LANE_COST, dtype=np.int64), [total]])
    return (d,) + binop_cuts(a, b, d)
