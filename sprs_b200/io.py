"""MatrixMarket coordinate files -> triplets -> device CSR (SURVEY.md 8f rank 4).

Host-side mirror of sprs/src/io.rs: `read_matrix_market` / `read_matrix_market_from_bufread`
(io.rs:118-292) return a TriMat exactly like the reference (same triplet order, symmetric /
skew-symmetric / hermitian expansion, same errors); `TriMat.to_csr()` is the device
COO->CSR conversion (sprs_b200_csmat_from_triplets; reference: triplet_iter.rs:127-224).
`write_matrix_market` / `write_matrix_market_sym` follow io.rs:294-468.

The parser is plain host code (as it is in the reference); only real (f64) matrices can be
taken to the device -- integer files load into an int64 TriMat but `to_csr()` needs f64,
pattern / complex files are rejected the way `read_matrix_market::<f64, ..>` rejects them.
"""
import io as _io
import os

import numpy as np

GENERAL, HERMITIAN, SYMMETRIC, SKEW_SYMMETRIC = "general", "hermitian", "symmetric", "skew-symmetric"


class IoError(Exception):
    """sprs::io::IoError (io.rs:16-43)."""
    BAD_FILE = "BadMatrixMarketFile"
    MISMATCH = "MismatchedMatrixMarketRead"
    UNSUPPORTED = "UnsupportedMatrixMarketFormat"

    def __init__(self, kind, matrix_kind=None, file_kind=None):
        self.kind, self.matrix_kind, self.file_kind = kind, matrix_kind, file_kind
        if kind == self.MISMATCH:  # io.rs:35-40
            msg = "Tried to load %s file into %s matrix." % (file_kind, matrix_kind)
        else:                       # io.rs:31-33
            msg = "Bad matrix market file."
        super().__init__(msg)

    def __eq__(self, o):
        return (isinstance(o, IoError) and self.kind == o.kind and
                self.matrix_kind == o.matrix_kind and self.file_kind == o.file_kind)

    __hash__ = Exception.__hash__


class TriMat:
    """TriMatBase (sprs/src/sparse/triplet.rs): shape + parallel row / col / data arrays,
    duplicates allowed (they are summed by to_csr / to_csc)."""

    def __init__(self, shape, row_inds=(), col_inds=(), data=(), dtype=np.float64):
        self.shape = (int(shape[0]), int(shape[1]))
        self.row_inds = list(row_inds)
        self.col_inds = list(col_inds)
        self.data = list(data)
        self.dtype = np.dtype(dtype)
        if not (len(self.row_inds) == len(self.col_inds) == len(self.data)):
            raise AssertionError("all inputs should have the same length")
        for r, c in zip(self.row_inds, self.col_inds):
            if not (0 <= r < self.shape[0] and 0 <= c < self.shape[1]):
                raise AssertionError("triplet index out of bounds")

    @classmethod
    def from_triplets(cls, shape, row_inds, col_inds, data, dtype=np.float64):
        return cls(shape, row_inds, col_inds, data, dtype)

    def add_triplet(self, row, col, val):
        if not (0 <= row < self.shape[0] and 0 <= col < self.shape[1]):
            raise AssertionError("triplet index out of bounds")
        self.row_inds.append(row)
        self.col_inds.append(col)
        self.data.append(val)

    def rows(self):
        return self.shape[0]

    def cols(self):
        return self.shape[1]

    def nnz(self):
        return len(self.data)

    def __eq__(self, o):
        return (isinstance(o, TriMat) and self.shape == o.shape and
                self.row_inds == o.row_inds and self.col_inds == o.col_inds and
                self.data == o.data)

    def triplet_iter(self):
        return zip(self.data, zip(self.row_inds, self.col_inds))

    def to_csr(self, ctx=None):
        """TriMat::to_csr (triplet_iter.rs:115-124) on the device."""
        from .sparse import CsMat
        if self.dtype != np.float64:
            raise TypeError("the H100 path is f64 only; %s triplets stay on the host" % self.dtype)
        return CsMat.from_triplets(self.shape, self.row_inds, self.col_inds, self.data, ctx=ctx)

    def to_csc(self, ctx=None):
        return self.to_csr(ctx).to_other_storage()


_KIND_OF = {"integer": "integer", "real": "real", "complex": "complex", "pattern": "pattern"}


def _parse_header(header):
    """io.rs:84-111 (the header has already been lower-cased)."""
    if not header.startswith("%%matrixmarket matrix coordinate"):
        raise IoError(IoError.BAD_FILE)
    for tag in ("real", "integer", "complex", "pattern"):
        if tag in header:
            data_type = tag
            break
    else:
        raise IoError(IoError.BAD_FILE)
    if "general" in header:
        sym = GENERAL
    elif "skew-symmetric" in header:
        sym = SKEW_SYMMETRIC
    elif "symmetric" in header:
        sym = SYMMETRIC
    elif "hermitian" in header:
        sym = HERMITIAN
    else:
        raise IoError(IoError.BAD_FILE)
    return sym, data_type


def _parse_usize(tok):
    if tok.startswith("+"):
        tok = tok[1:]
    if not tok.isdigit():
        raise ValueError(tok)
    return int(tok)


def read_matrix_market_from_bufread(reader, dtype=np.float64):
    """io.rs:138-292.  `reader` is a text file object; dtype float64 <-> "real" files,
    int64 <-> "integer" files (N::num_kind() must match the file's, io.rs:165-168)."""
    dtype = np.dtype(dtype)
    matrix_kind = {"f": "real", "i": "integer", "u": "integer"}.get(dtype.kind)
    if matrix_kind is None:
        raise TypeError("dtype must be a float or integer type")
    header = reader.readline().lower()
    sym_mode, data_type = _parse_header(header)
    if matrix_kind != data_type:  # "any type can be converted to pattern" does not apply
        raise IoError(IoError.MISMATCH, matrix_kind, data_type)
    # the header is followed by any number of comment lines (io.rs:174-182; like the
    # reference, a blank line here is NOT skipped: it is taken for the size line and fails)
    while True:
        line = reader.readline()
        if line == "":
            raise IoError(IoError.BAD_FILE)  # EOF (the reference would spin here)
        if line.startswith("%"):
            continue
        break
    infos = []
    for s in line.split():
        try:
            infos.append(_parse_usize(s))
        except ValueError:
            pass  # filter_map(|s| s.parse().ok())
    if len(infos) != 3:
        raise IoError(IoError.BAD_FILE)
    rows, cols, entries = infos
    row_inds, col_inds, data = [], [], []
    for _ in range(entries):
        while True:  # skip all-whitespace lines, stop at EOF (io.rs:200-208)
            line = reader.readline()
            if line != "" and line.strip() == "":
                continue
            break
        entry = line.split()
        try:
            row = _parse_usize(entry[0])
            col = _parse_usize(entry[1])
        except (IndexError, ValueError):
            raise IoError(IoError.BAD_FILE) from None
        if row < 1 or col < 1:  # indices are 1-based (checked_sub)
            raise IoError(IoError.BAD_FILE)
        row, col = row - 1, col - 1
        try:
            tok = entry[2]
            val = float(tok) if matrix_kind == "real" else int(tok)
        except (IndexError, ValueError):
            raise IoError(IoError.BAD_FILE) from None
        row_inds.append(row)
        col_inds.append(col)
        data.append(val)
        if sym_mode != GENERAL and row != col:
            if sym_mode == HERMITIAN:
                # mm_conj() is None for every real and integer type
                # (num_matrixmarket.rs:158-177): only complex matrices can be hermitian
                raise IoError(IoError.UNSUPPORTED)
            row_inds.append(col)
            col_inds.append(row)
            data.append(-val if sym_mode == SKEW_SYMMETRIC else val)
        if sym_mode == SKEW_SYMMETRIC and row == col:
            raise IoError(IoError.BAD_FILE)
        if len(entry) > 3:  # all data must be consumed (io.rs:262-266)
            raise IoError(IoError.BAD_FILE)
    return TriMat((rows, cols), row_inds, col_inds, data, dtype)


def read_matrix_market(mm_file, dtype=np.float64):
    """io.rs:118-132."""
    with open(os.fspath(mm_file), "r") as f:
        return read_matrix_market_from_bufread(f, dtype)


def _triplets_of(mat):
    """(val, (row, col)) in the iteration order of the reference's IntoIterator impls:
    TriMat in insertion order, CsMat outer by outer."""
    from .sparse import CsMat
    if isinstance(mat, TriMat):
        return mat.shape, list(mat.triplet_iter()), mat.dtype
    if isinstance(mat, CsMat):
        ip = mat.indptr.astype(np.int64) - int(mat.indptr[0])
        out = []
        for o in range(mat.outer_dims()):
            for k in range(ip[o], ip[o + 1]):
                i = int(mat.indices[k])
                out.append((float(mat.data[k]), (o, i) if mat.is_csr() else (i, o)))
        return mat.shape, out, np.dtype(np.float64)
    raise TypeError("write_matrix_market takes a TriMat or a CsMat")


def _mm_display(v, dtype):
    return repr(float(v)) if dtype.kind == "f" else str(int(v))


def write_matrix_market_to_bufwrite(writer, mat):
    """io.rs:309-347."""
    (rows, cols), trips, dtype = _triplets_of(mat)
    writer.write("%%%%MatrixMarket matrix coordinate %s general\n" %
                 ("real" if dtype.kind == "f" else "integer"))
    writer.write("% written by sprs\n")
    writer.write("%d %d %d\n" % (rows, cols, len(trips)))
    for val, (row, col) in trips:
        writer.write("%d %d %s\n" % (row + 1, col + 1, _mm_display(val, dtype)))


def write_matrix_market(path, mat):
    """io.rs:294-308."""
    with open(os.fspath(path), "w") as f:
        write_matrix_market_to_bufwrite(f, mat)


def write_matrix_market_sym(path, mat, sym):
    """io.rs:361-468: only one triangle is written (r <= c; r < c for skew-symmetric); the
    entry count in the size line is patched afterwards, padded with spaces."""
    (rows, cols), trips, dtype = _triplets_of(mat)
    if sym == GENERAL:
        keep = trips
    elif sym == SKEW_SYMMETRIC:
        keep = [t for t in trips if t[1][0] < t[1][1]]
    else:
        keep = [t for t in trips if t[1][0] <= t[1][1]]
    buf = _io.StringIO()
    buf.write("%%%%MatrixMarket matrix coordinate %s %s\n" %
              ("real" if dtype.kind == "f" else "integer", sym))
    buf.write("% written by sprs\n")
    full = "%d %d %d" % (rows, cols, len(trips))
    new = "%d %d %d" % (rows, cols, len(keep))
    buf.write(new + " " * (len(full) - len(new)) + "\n")
    for val, (row, col) in keep:
        buf.write("%d %d %s\n" % (row + 1, col + 1, _mm_display(val, dtype)))
    with open(os.fspath(path), "w") as f:
        f.write(buf.getvalue())
