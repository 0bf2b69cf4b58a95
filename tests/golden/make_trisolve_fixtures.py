"""Writes tests/golden/trisolve_fixtures.json: the reference's trisolve KATs
(sprs/src/sparse/linalg/trisolve.rs:368-442) as data, each cross-checked with
scipy.sparse.linalg.spsolve_triangular before it is written.

    python tests/golden/make_trisolve_fixtures.py
"""
import json
import os

import numpy as np
import scipy.sparse as sps
from scipy.sparse.linalg import spsolve_triangular

KATS = {
    # trisolve.rs:368-384: |1    | |3|   |3|
    #                      |0 2  | |1| = |2|
    #                      |1 0 1| |1|   |4|
    "lsolve_csr": dict(form="lsolve_csr", storage="CSR", shape=[3, 3], indptr=[0, 1, 2, 4],
                       indices=[0, 1, 0, 2], data=[1, 2, 1, 1], b=[3, 2, 4], x=[3, 1, 1]),
    # trisolve.rs:386-406: |1    | |3|   |3|
    #                      |1 2  | |1| = |5|
    #                      |0 0 3| |1|   |3|
    "lsolve_csc": dict(form="lsolve_csc", storage="CSC", shape=[3, 3], indptr=[0, 2, 3, 4],
                       indices=[0, 1, 1, 2], data=[1, 1, 2, 3], b=[3, 5, 3], x=[3, 1, 1]),
    # trisolve.rs:408-424: |1 0 1| |3|   |4|
    #                      |  2 0| |1| = |2|
    #                      |    3| |1|   |3|
    "usolve_csc": dict(form="usolve_csc", storage="CSC", shape=[3, 3], indptr=[0, 1, 2, 4],
                       indices=[0, 1, 0, 2], data=[1, 2, 1, 3], b=[4, 2, 3], x=[3, 1, 1]),
    # trisolve.rs:426-442: |1 1 0| |3|   |4|
    #                      |  5 3| |1| = |8|
    #                      |    1| |1|   |1|
    "usolve_csr": dict(form="usolve_csr", storage="CSR", shape=[3, 3], indptr=[0, 2, 4, 5],
                       indices=[0, 1, 1, 2, 2], data=[1, 1, 5, 3, 1], b=[4, 8, 1], x=[3, 1, 1]),
}


def cross_check(k):
    cls = sps.csr_matrix if k["storage"] == "CSR" else sps.csc_matrix
    m = cls((np.array(k["data"], float), k["indices"], k["indptr"]), shape=k["shape"]).toarray()
    lower = k["form"].startswith("l")
    m = np.tril(m) if lower else np.triu(m)
    x = spsolve_triangular(sps.csr_matrix(m), np.array(k["b"], float), lower=lower)
    assert np.allclose(x, k["x"]), (k["form"], x)


def main():
    for k in KATS.values():
        cross_check(k)
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "trisolve_fixtures.json")
    with open(out, "w") as f:
        json.dump(KATS, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
