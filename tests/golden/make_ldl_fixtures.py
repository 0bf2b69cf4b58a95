"""Writes tests/golden/ldl_fixtures.json: the known-answer tests of the sprs-ldl crate
(sprs-ldl/src/lib.rs, `mod test`) as data.  The reference states its expected values with 17
significant digits, so each parses to the exact f64 the reference computed; they are kept as
those strings.  Each KAT is cross-checked with scipy before it is written: L D L^T equals
P A P^T within rounding, and the solves agree with a dense solve.

    python tests/golden/make_ldl_fixtures.py
"""
import json
import os

import numpy as np
import scipy.sparse as sps

# test_mat1 (CSC), test_vec1 and the expected_* vectors of lib.rs
MAT1 = dict(storage="CSC", shape=[10, 10],
            indptr=[0, 2, 5, 6, 7, 13, 14, 17, 20, 24, 28],
            indices=[0, 8, 1, 4, 9, 2, 3, 1, 4, 6, 7, 8, 9, 5, 4, 6, 9, 4, 7, 8, 0, 4, 7, 8, 1, 4,
                     6, 9],
            data=["1.7", "0.13", "1.", "0.02", "0.01", "1.5", "1.1", "0.02", "2.6", "0.16", "0.09",
                  "0.52", "0.53", "1.2", "0.16", "1.3", "0.56", "0.09", "1.6", "0.11", "0.13",
                  "0.52", "0.11", "1.4", "0.01", "0.53", "0.56", "3.1"],
            b=["0.287", "0.22", "0.45", "0.44", "2.486", "0.72", "1.55", "1.424", "1.621",
               "3.759"],
            l_colptr=[0, 1, 3, 3, 3, 7, 7, 10, 12, 13, 13],
            l_indices=[8, 4, 9, 6, 7, 8, 9, 7, 8, 9, 8, 9, 9],
            l_data=["0.076470588235294124", "0.02", "0.01", "0.061547930450838589",
                    "0.034620710878596701", "0.20003077396522542", "0.20380058470533929",
                    "-0.0042935346524025902", "-0.024807089102770519", "0.40878266366119237",
                    "0.05752526570865537", "-0.010068305077340346", "-0.071852278207562709"],
            d=["1.7", "1.", "1.5", "1.1000000000000001", "2.5996000000000001", "1.2",
               "1.290152331127866", "1.5968603527854308", "1.2799646117414738",
               "2.7695677698030283"],
            lsolve=["0.28699999999999998", "0.22", "0.45000000000000001", "0.44",
                    "2.4816000000000003", "0.71999999999999997", "1.3972626557931991",
                    "1.3440844395148306", "1.0599997771886431", "2.7695677698030279"],
            dsolve=["0.16882352941176471", "0.22", "0.29999999999999999", "0.39999999999999997",
                    "0.95460840129250657", "0.59999999999999998", "1.0830214557467768",
                    "0.84170443406044937", "0.82814772179243734", "0.99999999999999989"],
            x=["0.099999999999999992", "0.19999999999999998", "0.29999999999999999",
               "0.39999999999999997", "0.5", "0.59999999999999998", "0.70000000000000007",
               "0.79999999999999993", "0.90000000000000002", "0.99999999999999989"])

# permuted_ldl_solve: integer data in the reference (exact in f64), perm [0, 2, 1, 3]
PERMUTED = dict(storage="CSC", shape=[4, 4], indptr=[0, 2, 4, 6, 8],
                indices=[0, 3, 1, 2, 1, 2, 0, 3], data=["1", "2", "21", "6", "6", "2", "2", "8"],
                perm=[0, 2, 1, 3], b=["9", "60", "18", "34"], x=["1", "2", "3", "4"])

KATS = {"test_mat1": MAT1, "permuted_ldl_solve": PERMUTED}


def f(v):
    return np.array([float(s) for s in v])


def cross_check():
    m = sps.csc_matrix((f(MAT1["data"]), MAT1["indices"], MAT1["indptr"]), shape=MAT1["shape"])
    a = m.toarray()
    n = a.shape[0]
    strict = sps.csc_matrix((f(MAT1["l_data"]), MAT1["l_indices"], MAT1["l_colptr"]),
                            shape=(n, n)).toarray()
    lo = strict + np.eye(n)
    d = f(MAT1["d"])
    assert np.allclose(lo @ np.diag(d) @ lo.T, a, rtol=0, atol=1e-14)
    b = f(MAT1["b"])
    y = np.linalg.solve(lo, b)
    assert np.allclose(y, f(MAT1["lsolve"]), rtol=1e-14)
    assert np.allclose(y / d, f(MAT1["dsolve"]), rtol=1e-14)
    assert np.allclose(np.linalg.solve(a, b), f(MAT1["x"]), rtol=1e-14)
    p = PERMUTED
    a = sps.csc_matrix((f(p["data"]), p["indices"], p["indptr"]), shape=p["shape"]).toarray()
    pm = np.eye(4)[p["perm"]]
    pap = pm @ a @ pm.T
    assert np.allclose(pap, pap.T)
    assert np.allclose(np.linalg.solve(a, f(p["b"])), f(p["x"]), rtol=1e-14)


def main():
    cross_check()
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ldl_fixtures.json")
    with open(out, "w") as fh:
        json.dump(KATS, fh, indent=1, sort_keys=True)
        fh.write("\n")


if __name__ == "__main__":
    main()
