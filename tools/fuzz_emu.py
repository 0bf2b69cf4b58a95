"""Structure fuzzer for the kernels' LOGIC on the CPU emulator (tests/emu; test infrastructure).

Random small matrices whose row lengths are drawn to sit ON the kernels' internal boundaries --
the SpMV merge-path tile (1024 cost units, a row end costing 16: a tile is ~1000 non-zeros or 64
row ends), its tiny rows (<= 8 non-zeros, one lane each), the lane groups G = 4 / 8 / 16 / 32 and
their switch to the whole warp above 16 G non-zeros, the 31-row blocks; the SpMM column panels
(64 / 128 columns per pass); the SpGEMM bins (128 / 1024 C entries, 4096 A non-zeros, 16384-column
panels) -- are pushed through the C ABI of the emulated library and compared with the oracle:
SpMV (values within the parity gate, bit-exact where the design promises it), SpMM (bit-exact),
SpGEMM (bit-exact, values too: every bin adds in the reference's order), CSR<->CSC (bit-exact), triplets
(pattern bit-exact), CSR x sparse vector (bit-exact).

Every odd seed runs in INTEGER mode (tests/exact.py): A, B, x and y0 are small integers, every
sum is exact in f64 whatever its order, and the SpMV and dense-product checks become
bit-equality.  SpGEMM values are compared bit for bit in both modes.

    python tools/fuzz_emu.py --seconds 300 [--seed 1] [--schedule random:3]

Prints one line per failure with the seed that reproduces it; exit code 1 if any.
"""
import argparse
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import exact  # noqa: E402  (tests/exact.py: integer-valued inputs)


def setup(schedule, binop=False):
    os.environ["SPRS_B200_EMU"] = "1"
    if schedule:
        os.environ["CUEMU_SCHEDULE"] = schedule
    import torch
    import sprs_b200
    from conftest import emu_library
    from sprs_b200 import generate
    if binop:  # the emulated build with csrc/binop.cu (tests/emu_binop.py)
        from emu_binop import emu_binop_library
        sprs_b200._lib.LIB_PATH = emu_binop_library()
    else:
        sprs_b200._lib.LIB_PATH = emu_library()
    generate._device = lambda ctx: torch.device("cpu")
    generate._stream_ptr = lambda: None
    generate._sync = lambda: None
    from oracle import oracle as O
    return sprs_b200, O


BOUNDARY_LENS = [0, 0, 0, 1, 1, 2, 3, 5, 7, 8, 9, 10, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128,
                 129, 255, 256, 257, 511, 512, 513, 1007, 1008, 1009, 1023, 1024, 1025, 1129, 1130,
                 2047, 2048, 2049, 4095, 4096, 4097]


def row_lengths(rng, rows, cols):
    """Mix of regimes: boundary lengths, runs of equal short rows, runs of empties, hubs."""
    mode = rng.integers(0, 6)
    if mode == 0:
        lens = rng.choice(BOUNDARY_LENS, rows)
    elif mode == 1:   # constant short rows (register path / group sizes)
        lens = np.full(rows, rng.choice([1, 2, 3, 4, 6, 8, 12, 16, 24, 32, 42, 43, 48, 64, 96, 128]))
    elif mode == 2:   # long empty stretches around tile boundaries (64 row ends fill a tile)
        lens = rng.choice([0, 0, 0, 0, 1008, 1007, 1009, 496, 1, 2, 2032, 32, 64], rows)
    elif mode == 3:   # poisson
        lens = rng.poisson(rng.choice([1, 4, 20, 60]), rows)
    elif mode == 4:   # hubs + dust
        lens = rng.choice([0, 1, 2, 3], rows)
        for _ in range(rng.integers(1, 4)):
            lens[rng.integers(0, rows)] = rng.choice([384, 385, 700, 1152, 1500, 3000, 4100])
    else:             # rows of cost 512 / 1024 (length + 16): many rows end exactly on a cut
        lens = rng.choice([496, 1008, 2032, 0, 48, 112, 0], rows)
    return np.minimum(lens.astype(np.int64), cols)


def make_csr(rng, rows, cols, lens, integer=False):
    indptr = np.zeros(rows + 1, dtype=np.int64)
    np.cumsum(lens, out=indptr[1:])
    indices = np.empty(indptr[-1], dtype=np.int64)
    for r in range(rows):
        n = lens[r]
        if n:
            indices[indptr[r]:indptr[r + 1]] = np.sort(rng.choice(cols, size=n, replace=False))
    if integer:
        return indptr.astype(np.uint32), indices.astype(np.uint32), exact.int_csr_data(indptr, rng.integers(1 << 30))
    data = rng.standard_normal(indptr[-1])
    # a few special values: exact zeros, huge / tiny magnitudes
    if data.size:
        k = rng.integers(0, data.size, size=max(1, data.size // 50))
        data[k] = rng.choice([0.0, -0.0, 1e300, -1e300, 1e-300, 1.0], size=k.size)
    return indptr.astype(np.uint32), indices.astype(np.uint32), data


def gate(got, ref, bound, what, bits=False):
    """the parity gate; bits=True -> bit-equality instead (NaN by class): integer mode, where
    every sum is exact, and results summed in the reference's order"""
    if bits:
        g, r = np.ascontiguousarray(got, dtype=np.float64), np.ascontiguousarray(ref, dtype=np.float64)
        bad = (g.view(np.uint64) != r.view(np.uint64)) & ~(np.isnan(g) & np.isnan(r))
        if bad.any():
            i = int(np.flatnonzero(bad.ravel())[0])
            return "%s: element %d got %r want %r (must be bit-exact)" % (
                what, i, g.flat[i], r.flat[i])
        return None
    bad = ~(np.abs(got - ref) <= 1e-6 * bound + 1e-300)
    bad &= ~(np.isnan(got) & np.isnan(ref))
    bad &= ~((got == ref))     # equal infinities
    if bad.any():
        i = int(np.flatnonzero(bad)[0])
        return "%s: element %d got %r want %r" % (what, i, got.flat[i], ref.flat[i])
    return None


def push_case(sp, a, rows, cols, rng):
    import ctypes as C
    import torch
    ctx = sp.Context.default()
    mirror = a.device().h
    offset = int(rng.integers(0, 9))
    n_targets = int(rng.integers(2, 5))
    total = rows + offset + 3
    x = torch.from_numpy(rng.standard_normal(cols))
    ref = torch.full((rows,), -7.0, dtype=torch.float64)
    accumulate = int(rng.integers(0, 2))
    ctx.check(ctx.lib.sprs_b200_spmv_dev(ctx.h, mirror, C.c_void_p(x.data_ptr()),
                                         C.c_void_p(ref.data_ptr()), accumulate, None))
    for name in ("chunked", "fused"):
        bufs = [torch.full((total,), -7.0, dtype=torch.float64) for _ in range(n_targets)]
        ptrs = (C.c_void_p * n_targets)(*[b.data_ptr() for b in bufs])
        if name == "chunked":
            st = ctx.lib.sprs_b200_spmv_chunked_push_dev(
                ctx.h, mirror, C.c_void_p(x.data_ptr()), offset, n_targets, ptrs, accumulate,
                int(rng.integers(0, 9)), None)
        else:  # the SpMV kernel itself stores every row into all targets (MULTI flavour)
            if accumulate:
                continue  # targets 1.. receive target 0's sum: only defined for y = A x
            st = ctx.lib.sprs_b200_spmv_allgather_dev(
                ctx.h, mirror, C.c_void_p(x.data_ptr()), offset, n_targets, ptrs, accumulate, None)
        ctx.check(st)
        want = ref.numpy()
        for q, b in enumerate(bufs):
            got = b.numpy()
            if not np.array_equal(got[offset:offset + rows].view(np.uint64), want.view(np.uint64)):
                return "%s push: target %d differs from the plain SpMV" % (name, q)
            if not (np.all(got[:offset] == -7.0) and np.all(got[offset + rows:] == -7.0)):
                return "%s push: target %d written outside the row block" % (name, q)
    return None


def solver_case(sp, O, rng, n, ip, ind, d):
    """A + (row abs sum + 1) on the diagonal -> strictly dominant; device solve vs oracle."""
    import scipy.sparse as sparse
    A = sparse.csr_matrix((d, ind.astype(np.int64), ip.astype(np.int64)), shape=(n, n))
    A = (A + sparse.diags(np.asarray(abs(A).sum(axis=1)).ravel() + 1.0)).tocsr()
    A.sort_indices()
    csr = (A.indptr.astype(np.uint32), A.indices.astype(np.uint32), A.data.copy())
    b = rng.standard_normal(n)
    a = sp.CsMat((n, n), *csr)
    tol = 1e-10
    try:
        res = sp.linalg.BiCGSTAB.solve(a, np.zeros(n), b, tol, 300)
    except sp.linalg.NotConverged as ex:
        ok, ref = O.BiCGSTAB.solve(csr, np.zeros(n), b, tol, 300)
        return None if not ok else "bicgstab: device Err, oracle Ok after %d" % ref.iteration_count()
    ok, ref = O.BiCGSTAB.solve(csr, np.zeros(n), b, tol, 300)
    if not ok:
        return "bicgstab: device Ok, oracle Err"
    if not np.allclose(res.x(), ref.x(), rtol=1e-6, atol=1e-9):
        return "bicgstab: x differs from the oracle"
    if np.linalg.norm(b - A @ res.x()) >= tol * 1.001:
        return "bicgstab: accepted solution misses the tolerance"
    # (iteration counts are not compared: a near-breakdown step amplifies the last-bit
    # difference of the dot products' summation order into a different trajectory)
    return None


def one_case(sp, O, seed):
    rng = np.random.default_rng(seed)
    rows = int(rng.choice([1, 2, 7, 33, 100, 257, 600]))
    cols = int(rng.choice([1, 5, 64, 500, 1153, 4200]))
    if rng.integers(0, 4) == 0:
        cols = rows  # square: also feeds the solver
    lens = row_lengths(rng, rows, cols)
    integer = seed % 2 == 1  # small integers: every sum exact, the products' checks bit-equality
    ip, ind, d = make_csr(rng, rows, cols, lens, integer)
    idx = rng.choice([np.uint32, np.uint64])
    a = sp.CsMat.new((rows, cols), ip.astype(idx), ind.astype(idx), d)
    errs = []
    # ---- SpMV (accumulating free function and the operator)
    finite = np.where(np.abs(d) > 1e200, 1.0, d)  # keep the gate meaningful: no overflow sums
    af = sp.CsMat.new((rows, cols), ip, ind, finite)
    x = exact.x_values(np.arange(cols, dtype=np.int64), seed) if integer else rng.standard_normal(cols)
    y0 = exact.y0_values(rows, seed) if integer else rng.standard_normal(rows)
    got = y0.copy()
    sp.prod.mul_acc_mat_vec_csr(af, x, got)
    ref, bound = y0.copy(), np.abs(y0)
    O.mul_acc_mat_vec_csr(ip, ind, finite, x, ref)
    O.mul_acc_mat_vec_csr(ip, ind, np.abs(finite), np.abs(x), bound)
    e = gate(got, ref, bound, "spmv", integer)
    if e:
        errs.append(e)
    elif lens.max() <= 6 and int(ip[-1]) + 16 * rows < 1024:
        # `&A * &x` (y starts at 0), one partial tile of short rows: one lane sums each row in
        # storage order -> the reference's bits (cut rows and y0 != 0 only agree to rounding)
        ref0 = np.zeros(rows)
        O.mul_acc_mat_vec_csr(ip, ind, finite, x, ref0)
        if not np.array_equal(af * x, ref0):
            errs.append("spmv: short rows in one tile not bit-exact")
    # ---- pipelined all-gathers (chunked push / stream push) into local "peer" buffers:
    #      bit-identical to the plain device SpMV, nothing written outside the row block
    if rows >= 2 and os.environ.get("SPRS_B200_FUZZ_PUSH", "1") == "1":
        e = push_case(sp, af, rows, cols, rng)
        if e:
            errs.append(e)
    # ---- SpMM: bit-exact, k on both sides of the k >= 8 rule
    k = int(rng.choice([1, 3, 8, 9, 32, 33, 64, 70]))
    b = exact.mat_values(np.arange(cols * k, dtype=np.int64), seed).reshape(cols, k) if integer \
        else rng.standard_normal((cols, k))
    c = af * b
    cref = np.zeros((rows, k))
    O.csr_mulacc_dense_rowmaj(ip, ind, finite, b, cref)
    if k >= 8:
        if not np.array_equal(c, cref):
            errs.append("spmm k=%d: not bit-exact" % k)
    else:
        cb = np.zeros((rows, k))
        O.csr_mulacc_dense_rowmaj(ip, ind, np.abs(finite), np.abs(b), cb)
        e = gate(np.asarray(c), cref, cb, "spmm-colmaj k=%d" % k, integer)
        if e:
            errs.append(e)
    # ---- CSC operands (device CSC -> CSR, then the CSR kernels: same ascending-column sums)
    #      and arbitrary-stride dense views (prod.rs:632-651)
    acsc = af.to_other_storage()
    yc = np.zeros(rows)
    sp.prod.mul_acc_mat_vec_csc(acsc, x, yc) if af.is_csr() else None
    refc, bc = np.zeros(rows), np.zeros(rows)
    O.mul_acc_mat_vec_csr(ip, ind, finite, x, refc)
    O.mul_acc_mat_vec_csr(ip, ind, np.abs(finite), np.abs(x), bc)
    e = gate(yc, refc, bc, "csc spmv", integer)
    if e:
        errs.append(e)
    kk = int(rng.choice([8, 13, 40]))
    big = rng.standard_normal((2 * cols + 1, 2 * kk + 3))
    if integer:
        big = exact.mat_values(np.arange(big.size, dtype=np.int64), seed + 1).reshape(big.shape)
    view = big[::2][:cols, ::-2][:, :kk] if rng.integers(0, 2) else np.asfortranarray(big[:cols, :kk])
    outbig = np.zeros((rows * 2 + 1, kk + 2))
    out = outbig[1::2][:rows, 1:kk + 1]
    (sp.prod.csc_mulacc_dense_rowmaj if rng.integers(0, 2) else sp.prod.csc_mulacc_dense_colmaj)(
        acsc, view, out)
    want = np.zeros((rows, kk))
    O.csr_mulacc_dense_rowmaj(ip, ind, finite, np.ascontiguousarray(view), want)
    wb = np.zeros((rows, kk))
    O.csr_mulacc_dense_rowmaj(ip, ind, np.abs(finite), np.abs(np.ascontiguousarray(view)), wb)
    e = gate(np.ascontiguousarray(out), want, wb, "csc dense product on strided views", integer)
    if e:
        errs.append(e)
    if outbig[0::2].any() or outbig[:, 0].any() or outbig[:, kk + 1].any():
        errs.append("dense product wrote outside its output view")
    # ---- storage conversion: bit-exact, both directions
    t = a.to_other_storage()
    tip, tind, td = O.convert_mat_storage(rows, cols, ip, ind, d)
    if not (np.array_equal(t.indptr, tip) and np.array_equal(t.indices, tind) and
            np.array_equal(t.data.view(np.uint64), td.view(np.uint64))):
        errs.append("to_other_storage mismatch")
    back = t.to_other_storage()
    if not (np.array_equal(back.indptr, a.indptr) and np.array_equal(back.indices, a.indices) and
            np.array_equal(back.data.view(np.uint64), a.data.view(np.uint64))):
        errs.append("to_other_storage round trip mismatch")
    # ---- CSR x sparse vector: bit-exact
    vn = int(rng.integers(0, cols + 1))
    vi = np.sort(rng.choice(cols, vn, replace=False))
    vd = rng.standard_normal(vn)
    res = a * sp.CsVec(cols, vi, vd)
    oi, od = O.csr_mul_csvec(ip, ind, d, vi, vd)
    if not (np.array_equal(res.indices, oi.astype(np.int64)) and
            np.array_equal(res.data.view(np.uint64), od.view(np.uint64))):
        errs.append("csr_mul_csvec mismatch")
    if os.environ.get("SPRS_B200_FORCE_INDPTR64") == "1":
        return errs  # the SpGEMM refuses 64-bit-indptr operands (nnz >= 2^32): documented limit
    # ---- SpGEMM against a second matrix with its own structure
    # 9000 / 23000 columns: C rows beyond 4096 entries -> dense shared-memory panels (1 and 2)
    bcols = int(rng.choice([1, 9, 300, 2500, 2500, 9000, 23000]))
    blens = row_lengths(rng, cols, bcols)
    bip, bind, bd = make_csr(rng, cols, bcols, blens, integer)
    bd = np.where(np.abs(bd) > 1e200, 1.0, bd)
    bm = sp.CsMat.new((cols, bcols), bip.astype(idx), bind.astype(idx), bd)
    af2 = sp.CsMat.new((rows, cols), ip.astype(idx), ind.astype(idx), finite)
    cm = af2 * bm
    cip, cind, cd = O.mul_csr_csr((rows, cols), (ip, ind, finite), (cols, bcols), (bip, bind, bd),
                                  threads=1)
    if not (np.array_equal(cm.indptr, cip) and np.array_equal(cm.indices, cind)):
        errs.append("spgemm pattern mismatch")
    else:
        _, _, cb = O.mul_csr_csr((rows, cols), (ip, ind, np.abs(finite)), (cols, bcols),
                                 (bip, bind, np.abs(bd)), threads=1)
        e = gate(cm.data, cd, cb, "spgemm values", True)
        if e:
            errs.append(e)
        # storage dispatch (csmat.rs:1895-1949): CSC operands route through transposes; the
        # result is CSC only for CSC x CSR / CSC x CSC, and always the same matrix
        if (seed & 3) == 0 and rows * cols <= 200000:
            a_csc, b_csc = af2.to_other_storage(), bm.to_other_storage()
            for lhs, rhs, want_csc in ((af2, b_csc, False), (a_csc, bm, True), (a_csc, b_csc, True)):
                got = lhs * rhs
                if got.is_csc() != want_csc:
                    errs.append("spgemm dispatch: wrong result storage")
                    continue
                g = got.to_other_storage() if want_csc else got
                if not (np.array_equal(g.indptr, cip) and np.array_equal(g.indices, cind)):
                    errs.append("spgemm dispatch: pattern differs from CSR x CSR")
                elif gate(g.data, cd, cb, "spgemm dispatch values", True):
                    errs.append("spgemm dispatch: values differ from CSR x CSR")
    # ---- row slices: slice_outer + proper_indptr upload (slicing.rs:65-89), SpMV on the view
    if rows >= 3:
        lo = int(rng.integers(0, rows - 1))
        hi = int(rng.integers(lo + 1, rows + 1))
        sl = af.slice_outer(lo, hi)
        ys = sl * x
        e = gate(ys, refc[lo:hi], bc[lo:hi], "spmv on a row slice", integer)
        if e:
            errs.append(e)
    # ---- BiCGSTAB on a diagonally dominant system built from the same pattern
    if rows == cols and rows >= 2:
        e = solver_case(sp, O, rng, rows, ip, ind, finite)
        if e:
            errs.append(e)
    # ---- triplets: shuffled COO with duplicates
    if ip[-1]:
        r_of = np.repeat(np.arange(rows), lens)
        take = rng.integers(0, int(ip[-1]), size=int(ip[-1]) + int(ip[-1]) // 3)
        tr, tc, tv = r_of[take], ind[take].astype(np.int64), rng.standard_normal(take.size)
        m = sp.CsMat.from_triplets((rows, cols), tr, tc, tv)
        oip, oind, odat = O.triplets_to_csr((rows, cols), tr, tc, tv)
        # pattern exact; duplicate sums: the reference's sort is unstable, so the order of a
        # duplicate run's terms is unspecified there (SURVEY 8f-1) -- compare to rounding
        if not (np.array_equal(m.indptr, oip) and np.array_equal(m.indices, oind)):
            errs.append("from_triplets pattern mismatch")
        elif not np.allclose(m.data, odat, rtol=1e-12, atol=1e-12):
            errs.append("from_triplets values mismatch")
    return errs


BINOP_LENS = [0, 0, 1, 2, 15, 16, 17, 31, 32, 33, 63, 64, 65, 1007, 1008, 1023, 1024, 1025, 3000]


def binop_case(sp, O, seed):
    """--binop: `+`, `-`, mul_mat_same_storage and `* s` (csrc/binop.cu) against the binop oracle,
    bit for bit (NaN by class).  Row lengths sit on the tile (1024 cost units, a row end 16),
    lane (32 units) and snap boundaries; B overlaps A (forced equal pairs) or cancels it."""
    import binop_oracle as BO
    rng = np.random.default_rng(seed)
    rows, cols = int(rng.integers(0, 160)), int(rng.integers(1, 4000))
    la = np.minimum(rng.choice(BINOP_LENS, rows), cols)
    a = make_csr(rng, rows, cols, la, integer=bool(seed & 1))
    mode = rng.integers(0, 3)
    if mode == 0:    # independent patterns
        b = make_csr(rng, rows, cols, np.minimum(rng.choice(BINOP_LENS, rows), cols))
    else:            # A's pattern, thinned: equal pairs everywhere, exact cancellations (mode 2)
        keep = rng.random(a[1].size) < 0.7
        r_of = np.repeat(np.arange(rows), np.diff(a[0].astype(np.int64)))
        ip = np.zeros(rows + 1, np.int64)
        np.cumsum(np.bincount(r_of[keep], minlength=rows), out=ip[1:])
        d = a[2][keep] if mode == 2 else rng.standard_normal(int(keep.sum()))
        b = (ip.astype(np.uint32), a[1][keep], d)
    A, B = sp.CsMat.new((rows, cols), *a), sp.CsMat.new((rows, cols), *b)
    if rng.random() < 0.25:  # CSC + CSC
        A, B = A.to_other_storage(), B.to_other_storage()
    errs = []
    cast = lambda m: (m.indptr.astype(np.uint64), m.indices.astype(np.uint32), m.data)  # noqa: E731
    ops = [(BO.ADD, lambda: A + B), (BO.SUB, lambda: A - B),
           (BO.MUL, lambda: sp.binop.mul_mat_same_storage(A, B))]
    for op, f in [ops[i] for i in rng.permutation(3)]:
        got = f()
        e = BO.first_difference((got.indptr, got.indices, got.data), BO.binop(op, cast(A), cast(B)))
        if e:
            errs.append("binop %d: %s" % (op, e))
    s = float(rng.choice([2.0, -0.5, 0.0, np.inf]))
    got = A * s
    e = BO.first_difference((got.indptr, got.indices, got.data), BO.scale(cast(A), s))
    if e:
        errs.append("scale: " + e)
    return errs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=120)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--schedule", default="")
    ap.add_argument("--cases", type=int, default=0)
    ap.add_argument("--binop", action="store_true", help="fuzz the sparse binops instead")
    args = ap.parse_args()
    sp, O = setup(args.schedule, args.binop)
    t0 = time.time()
    n = fails = 0
    seed = args.seed
    while (args.cases and n < args.cases) or (not args.cases and time.time() - t0 < args.seconds):
        try:
            errs = (binop_case if args.binop else one_case)(sp, O, seed)
        except Exception as e:  # a panic / status code where none is expected is a finding too
            errs = ["exception %s: %s" % (type(e).__name__, e)]
        for e in errs:
            print("FAIL seed=%d: %s" % (seed, e), flush=True)
        fails += bool(errs)
        n += 1
        seed += 1
    print("%d cases, %d failing, %.0f s" % (n, fails, time.time() - t0))
    return 1 if fails else 0


if __name__ == "__main__":
    sys.exit(main())
