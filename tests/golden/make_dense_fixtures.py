"""Writes tests/golden/dense_fixtures.json: the reference's known answers for the dense boundary,
transcribed from its unit tests and cross-checked here with numpy / scipy on the finite values.

  to_dense.rs:56-92      to_dense of eye (CSR and CSC), mat1 and mat3
  csmat.rs:2493-2539     csr_from_dense / csc_from_dense of eye(3) and of a 3 x 5 matrix, eps 1e-5
  binop.rs:600-718       csr_add_dense_rowmaj (add_dense_mat_same_ordering and `&a + &b`),
                         csr_mul_dense_rowmaj, mul_dense_strided in both layouts, and the
                         accepted standard and strided layouts of csmat_binop_dense_raw

Run: python tests/golden/make_dense_fixtures.py
"""
import json
import os

import numpy as np
import scipy.sparse as S

HERE = os.path.dirname(os.path.abspath(__file__))


def csr(m):
    m = S.csr_matrix(m)
    m.sort_indices()
    return {"storage": "CSR", "shape": list(m.shape), "indptr": m.indptr.tolist(),
            "indices": m.indices.tolist(), "data": m.data.tolist()}


def csc(m):
    m = S.csc_matrix(m)
    m.sort_indices()
    return {"storage": "CSC", "shape": list(m.shape), "indptr": m.indptr.tolist(),
            "indices": m.indices.tolist(), "data": m.data.tolist()}


def main():
    # sprs test_data.rs: mat1 (5 x 5 CSR) and mat3 (5 x 4 CSR), mat_dense1
    mat1 = {"storage": "CSR", "shape": [5, 5], "indptr": [0, 2, 4, 5, 6, 7],
            "indices": [2, 3, 3, 4, 2, 1, 3], "data": [3., 4., 2., 5., 5., 8., 7.]}
    mat3 = {"storage": "CSR", "shape": [5, 4], "indptr": [0, 2, 4, 5, 6, 7],
            "indices": [2, 3, 2, 3, 2, 1, 3], "data": [3., 4., 2., 5., 5., 8., 7.]}
    mat_dense1 = [[0., 1., 2., 3., 4.], [5., 6., 5., 4., 3.], [4., 5., 4., 3., 2.],
                  [3., 4., 3., 2., 1.], [1., 2., 1., 1., 0.]]
    to_dense_mat1 = [[0., 0., 3., 4., 0.], [0., 0., 0., 2., 5.], [0., 0., 5., 0., 0.],
                     [0., 8., 0., 0., 0.], [0., 0., 0., 7., 0.]]
    to_dense_mat3 = [[0., 0., 3., 4.], [0., 0., 2., 5.], [0., 0., 5., 0.], [0., 8., 0., 0.],
                     [0., 0., 0., 7.]]
    from_dense_in = [[1., 0., 2., 1e-7, 1.], [0., 0., 0., 1., 0.], [3., 0., 1., 0., 0.]]
    csr_from_dense_out = {"storage": "CSR", "shape": [3, 5], "indptr": [0, 3, 4, 6],
                          "indices": [0, 2, 4, 3, 0, 2], "data": [1., 2., 1., 1., 3., 1.]}
    csc_from_dense_out = {"storage": "CSC", "shape": [3, 5], "indptr": [0, 2, 2, 4, 5, 6],
                          "indices": [0, 2, 0, 2, 1, 0], "data": [1., 3., 2., 1., 1., 1.]}
    add_dense_out = [[0., 1., 5., 7., 4.], [5., 6., 5., 6., 8.], [4., 5., 9., 3., 2.],
                     [3., 12., 3., 2., 1.], [1., 2., 1., 8., 0.]]
    # cross-checks with scipy on the finite values
    m1 = S.csr_matrix((mat1["data"], mat1["indices"], mat1["indptr"]), shape=(5, 5))
    m3 = S.csr_matrix((mat3["data"], mat3["indices"], mat3["indptr"]), shape=(5, 4))
    assert np.array_equal(m1.toarray(), to_dense_mat1)
    assert np.array_equal(m3.toarray(), to_dense_mat3)
    fd = np.array(from_dense_in)
    assert csr(np.where(np.abs(fd) > 1e-5, fd, 0)) == csr_from_dense_out
    assert csc(np.where(np.abs(fd) > 1e-5, fd, 0)) == csc_from_dense_out
    assert np.array_equal(m1.toarray() + np.array(mat_dense1), add_dense_out)
    out = {
        "mat1": mat1, "mat3": mat3, "mat_dense1": mat_dense1,
        "eye3_csr": csr(np.eye(3)), "eye3_csc": csc(np.eye(3)), "eye3_dense": np.eye(3).tolist(),
        "to_dense_mat1": to_dense_mat1, "to_dense_mat3": to_dense_mat3,
        "from_dense_in": from_dense_in, "from_dense_eps": 1e-5,
        "csr_from_dense_out": csr_from_dense_out, "csc_from_dense_out": csc_from_dense_out,
        "add_dense_out": add_dense_out,
    }
    with open(os.path.join(HERE, "dense_fixtures.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
