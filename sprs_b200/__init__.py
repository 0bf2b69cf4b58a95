"""sprs_b200 -- H100-native (sm_90a) implementation of the sprs sparse-product hot
path (SpMV / SpMM / SpGEMM) behind sprs's operator API.  See DESIGN.md.

Nothing here computes on the CPU: every product is a call into libsprs_b200.so
(hand-written CUDA).  Importing works without a GPU (so the ABI can be inspected);
creating a Context without one raises ThirdPartyError.
"""
from . import _lib, io, linalg
from .sparse import (CSC, CSR, Context, CsMat, CsVec, DeviceCsMat, SprsPanic, ThirdPartyError,
                     csmat_mul_csmat, prod, smmp)

__all__ = ["CSC", "CSR", "Context", "CsMat", "CsVec", "DeviceCsMat", "SprsPanic",
           "ThirdPartyError", "csmat_mul_csmat", "prod", "smmp", "_lib", "io", "linalg"]
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
