"""Writes tests/golden/binop_fixtures.json: the reference's binop known-answer data.

Transcribed as DATA (not code) from the reference's tests; each entry cites where it lives:

  sprs/src/sparse/binop.rs:488-510   mat1 + mat2, mat1 - mat2, mat1 .* mat2 (mul_mat_same_storage)
  sprs/src/test_data.rs:55-60        mat1 * 2.0
  sprs/src/sparse/binop.rs:523-531   test_add1: 3x3 operands with differing row patterns

The operands mat1 / mat2 are those of sprs_fixtures.json (test_data.rs).  scipy is used only as
an independent cross-check of the transcription: its `+`, `-` and `.multiply` also drop exact
zeros, and every expected result is recomputed and compared before the file is written.

Run:  python tests/golden/make_binop_fixtures.py
"""
import json
import os

import numpy as np
import scipy.sparse as sp

HERE = os.path.dirname(os.path.abspath(__file__))


def csmat(storage, shape, indptr, indices, data):
    return {"storage": storage, "shape": list(shape), "indptr": indptr,
            "indices": indices, "data": data}


F = {}
# ---- sprs/src/sparse/binop.rs:488-510
F["mat1_plus_mat2"] = csmat("CSR", (5, 5), [0, 5, 8, 9, 12, 15],
                            [0, 1, 2, 3, 4, 0, 3, 4, 2, 1, 2, 3, 1, 2, 3],
                            [6., 7., 6., 4., 3., 8., 11., 5., 5., 8., 2., 4., 4., 4., 7.])
F["mat1_minus_mat2"] = csmat("CSR", (5, 5), [0, 4, 7, 8, 11, 14],
                             [0, 1, 3, 4, 0, 3, 4, 2, 1, 2, 3, 1, 2, 3],
                             [-6., -7., 4., -3., -8., -7., 5., 5., 8., -2., -4., -4., -4., 7.])
F["mat1_times_mat2"] = csmat("CSR", (5, 5), [0, 1, 2, 2, 2, 2], [2, 3], [9., 18.])
# ---- sprs/src/test_data.rs:55-60
F["mat1_times_2"] = csmat("CSR", (5, 5), [0, 2, 4, 5, 6, 7], [2, 3, 3, 4, 2, 1, 3],
                          [6., 8., 4., 10., 10., 16., 14.])
# ---- sprs/src/sparse/binop.rs:523-531 (test_add1, second half)
F["add1_lhs"] = csmat("CSR", (3, 3), [0, 1, 1, 2], [0, 2], [1., 1.])
F["add1_rhs"] = csmat("CSR", (3, 3), [0, 1, 2, 2], [0, 1], [1., 1.])
F["add1_sum"] = csmat("CSR", (3, 3), [0, 1, 2, 3], [0, 1, 2], [2., 1., 1.])


def to_sp(m):
    cls = sp.csr_matrix if m["storage"] == "CSR" else sp.csc_matrix
    return cls((np.array(m["data"]), np.array(m["indices"]), np.array(m["indptr"])),
               shape=tuple(m["shape"]))


def check(got, want):
    got = got.tocsr() if want["storage"] == "CSR" else got.tocsc()
    got.sort_indices()
    assert got.indptr.tolist() == want["indptr"], (got.indptr, want["indptr"])
    assert got.indices.tolist() == want["indices"]
    assert got.data.tolist() == want["data"]


def main():
    with open(os.path.join(HERE, "sprs_fixtures.json")) as f:
        base = json.load(f)
    m1, m2 = to_sp(base["mat1"]), to_sp(base["mat2"])
    check(m1 + m2, F["mat1_plus_mat2"])
    check(m1 - m2, F["mat1_minus_mat2"])
    check(m1.multiply(m2), F["mat1_times_mat2"])
    check(m1 * 2.0, F["mat1_times_2"])
    check(to_sp(F["add1_lhs"]) + to_sp(F["add1_rhs"]), F["add1_sum"])
    with open(os.path.join(HERE, "binop_fixtures.json"), "w") as f:
        json.dump(F, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote %d fixtures" % len(F))


if __name__ == "__main__":
    main()
