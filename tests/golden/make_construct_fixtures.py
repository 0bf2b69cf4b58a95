"""Writes tests/golden/construct_fixtures.json: the reference's construction known-answer data.

Transcribed as DATA (not code) from the reference's tests:

  sprs/src/sparse/construct.rs, mod test   mat1_vstack_mat2 (vstack_trivial, hstack_trivial as
                                            its transpose, vstack_with_conversion), bmat_simple,
                                            both halves of bmat_complex, and the panic tests as
                                            (blocks, message) cases
  sprs/src/sparse/kronecker.rs             test_kronecker_product: a, b and the 16 expected
                                            entries, checked in all four storage combinations

mat1 .. mat4 are those of sprs_fixtures.json (test_data.rs).  scipy is used only as an
independent cross-check of the transcription: scipy.sparse.vstack / hstack / bmat / kron agree
with the reference where both are defined (bmat with equal block heights and widths, no empty
grids), and every expected result is recomputed and compared before the file is written.

Run:  python tests/golden/make_construct_fixtures.py
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
# ---- construct.rs mod test: mat1_vstack_mat2
F["mat1_vstack_mat2"] = csmat("CSR", (10, 5), [0, 2, 4, 5, 6, 7, 11, 13, 13, 15, 17],
                              [2, 3, 3, 4, 2, 1, 3, 0, 1, 2, 4, 0, 3, 2, 3, 1, 2],
                              [3., 4., 2., 5., 5., 8., 7., 6., 7., 3., 3., 8., 9., 2., 4., 4., 4.])
# bmat_simple: bmat([[eye(5), None], [None, eye(4)]])
F["bmat_simple"] = csmat("CSR", (9, 9), list(range(10)), list(range(9)), [1.] * 9)
# bmat_complex, first half: bmat([[mat1, mat2], [mat2, None]])
F["bmat_complex_1"] = csmat("CSR", (10, 10), [0, 6, 10, 11, 14, 17, 21, 23, 23, 25, 27],
                            [2, 3, 5, 6, 7, 9, 3, 4, 5, 8, 2, 1, 7, 8, 3, 6, 7, 0, 1, 2, 4,
                             0, 3, 2, 3, 1, 2],
                            [3., 4., 6., 7., 3., 3., 2., 5., 8., 9., 5., 8., 2., 4., 7., 4.,
                             4., 6., 7., 3., 3., 8., 9., 2., 4., 4., 4.])
# bmat_complex, second half: bmat([[mat3, mat1], [None, mat4]])
F["bmat_complex_2"] = csmat("CSR", (10, 9), [0, 4, 8, 10, 12, 14, 16, 18, 21, 23, 24],
                            [2, 3, 6, 7, 2, 3, 7, 8, 2, 6, 1, 5, 3, 7, 4, 5, 4, 8, 4, 7, 8,
                             5, 7, 4],
                            [3., 4., 3., 4., 2., 5., 2., 5., 5., 5., 8., 8., 7., 7., 6., 8.,
                             7., 4., 3., 2., 4., 9., 4., 3.])
# the panic tests: block grids by name ("mat1", "mat3", "mat4", null) and the message the
# reference's composition panics with
F["panics"] = [
    {"test": "same_storage_fast_stack_fail_empty_stacking_list", "stack": [],
     "message": "Empty stacking list"},
    {"test": "same_storage_fast_stack_fail_dim_mismatch", "stack": ["mat1", "mat3"],
     "message": "Dimension mismatch"},
    {"test": "bmat_fail_shapes", "blocks": [[None, None], [None]],
     "message": "Dimension mismatch"},
    {"test": "bmat_fail_empty_stacking_list", "blocks": [[]], "message": "Empty stacking list"},
    {"test": "bmat_fail_empty_bmat_row", "blocks": [[None, None], ["mat1", "mat3"]],
     "message": "Empty bmat row"},
    {"test": "bmat_fail_empty_bmat_col", "blocks": [["mat3", None], ["mat1", None]],
     "message": "Empty bmat col"},
]
# ---- kronecker.rs test_kronecker_product (i32 values in the reference; exact in f64)
F["kron_a"] = csmat("CSR", (2, 3), [0, 2, 4], [1, 2, 0, 2], [2., 3., 6., 8.])
F["kron_b"] = csmat("CSR", (3, 2), [0, 1, 2, 4], [0, 0, 0, 1], [1., 2., 3., -3.])
F["kron_entries"] = [[0, 2, 2], [0, 4, 3], [1, 2, 4], [1, 4, 6], [2, 2, 6], [2, 3, -6],
                     [2, 4, 9], [2, 5, -9], [3, 0, 6], [3, 4, 8], [4, 0, 12], [4, 4, 16],
                     [5, 0, 18], [5, 1, -18], [5, 4, 24], [5, 5, -24]]


def scipy_of(m):
    cls = sp.csr_matrix if m["storage"] == "CSR" else sp.csc_matrix
    return cls((m["data"], m["indices"], m["indptr"]), shape=tuple(m["shape"]))


def check():
    with open(os.path.join(HERE, "sprs_fixtures.json")) as f:
        base = json.load(f)
    m1, m2, m3, m4 = (scipy_of(base[k]) for k in ("mat1", "mat2", "mat3", "mat4"))

    def same(got, key):
        want = scipy_of(F[key])
        got = sp.csr_matrix(got)
        got.sort_indices()
        assert got.shape == want.shape, key
        assert np.array_equal(got.indptr, want.indptr), key
        assert np.array_equal(got.indices, want.indices), key
        assert np.array_equal(got.data, want.data), key

    same(sp.vstack([m1, m2]), "mat1_vstack_mat2")
    assert (sp.hstack([m1.T, m2.T]) != scipy_of(F["mat1_vstack_mat2"]).T).nnz == 0
    same(sp.block_diag([sp.eye(5), sp.eye(4)]), "bmat_simple")
    # scipy needs equal heights per block row and widths per block column: rows of
    # bmat_complex_1 are [mat1 mat2] and [mat2 0]; those of bmat_complex_2 [mat3 mat1], [0 mat4]
    same(sp.vstack([sp.hstack([m1, m2]), sp.hstack([m2, sp.csr_matrix((5, 5))])]),
         "bmat_complex_1")
    same(sp.vstack([sp.hstack([m3, m1]), sp.hstack([sp.csr_matrix((5, 4)), m4])]),
         "bmat_complex_2")
    # scipy's kron goes through a block format and stores the zeros of each block; the
    # reference keeps only products of stored entries
    c = sp.kron(scipy_of(F["kron_a"]), scipy_of(F["kron_b"])).tocsr()
    c.eliminate_zeros()
    c = c.tocoo()
    got = sorted((int(i), int(j), float(v)) for i, j, v in zip(c.row, c.col, c.data))
    assert got == sorted((i, j, float(v)) for i, j, v in F["kron_entries"])


if __name__ == "__main__":
    check()
    with open(os.path.join(HERE, "construct_fixtures.json"), "w") as f:
        json.dump(F, f, indent=1)
        f.write("\n")
    print("wrote construct_fixtures.json")
