"""SpMV hot set (SPRS_B200_SPMV_HOT=auto|0|K, csrc/spmv.cu): x of the most-referenced columns is
staged in shared memory and the SpMV reads a tagged copy of the index stream.  Only the place an
x value is read from changes, so y must be BIT-identical to the SpMV without a hot set, on every
path that runs the kernel: plain and accumulating, the tile-range chunks of the host path, the
multi-target (fused all-gather) kernel and the 64-bit-indptr instantiations.

The switch is read once per process: each configuration runs this file as a child process that
writes its results to an .npz, and the parent compares the bits."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cases(out_path):
    """(child) every case's outputs, keyed by name"""
    sys.path.insert(0, ROOT)
    import torch
    import sprs_b200 as sp
    from sprs_b200 import generate as G
    ctx = sp.Context.default()
    res = {}

    def device_cases(tag, a, n_rows, n_cols):
        x = G.normal_vector(ctx, n_cols, 5)
        y = torch.empty(n_rows, device="cuda", dtype=torch.float64)
        G.spmv(ctx, a, x, y)
        res[tag + "/y"] = y.cpu().numpy()
        y0 = G.normal_vector(ctx, n_rows, 9)
        G.spmv(ctx, a, x, y0, accumulate=True)
        res[tag + "/y_acc"] = y0.cpu().numpy()
        # multi-target kernel: 2 targets (a store per row) and 3 (rows staged, TMA bulk stores)
        for nt in (2, 3):
            bufs = [torch.full((n_rows + 16,), -7.0, device="cuda", dtype=torch.float64)
                    for _ in range(nt)]
            ptrs = (C.c_void_p * nt)(*[b.data_ptr() + 8 * 2 for b in bufs])
            torch.cuda.synchronize()
            ctx.check(ctx.lib.sprs_b200_spmv_allgather_dev(ctx.h, a.mirror.h, C.c_void_p(x.data_ptr()),
                                                          0, nt, ptrs, 0, None))
            torch.cuda.synchronize()
            res[tag + "/multi%d" % nt] = torch.stack(bufs).cpu().numpy()
        # host path in chunks (SPRS_B200_E2E_MIN_TILES=1): spmv_launch_tile_range + carries
        hx = x.cpu().numpy()
        hy = np.full(n_rows, -777.0)
        ctx.check(ctx.lib.sprs_b200_mul_mat_vec(ctx.h, a.mirror.h, hx.ctypes.data_as(C.c_void_p), n_cols,
                                                hy.ctypes.data_as(C.c_void_p), n_rows))
        res[tag + "/host_chunked"] = hy

    # 1. a 1M R-MAT: skewed columns, ties at the K-th count split by column order
    n = 1_000_000
    device_cases("rmat", G.rmat_csr(ctx, n, 16, seed=23), n, n)
    # 2. rows made only of hot columns (512 referenced columns < every K used here), row lengths
    #    across the tiny / grouped / whole-warp sweeps of the kernel
    rng = np.random.default_rng(3)
    rows, cols = 20000, 300000
    lens = rng.choice([0, 1, 3, 8, 9, 20, 33, 64, 130, 512], rows)
    ip = np.zeros(rows + 1, dtype=np.int64)
    np.cumsum(lens, out=ip[1:])
    idx = np.concatenate([np.sort(rng.choice(512, size=int(k), replace=False)) * 577 for k in lens if k])
    dev = torch.device("cuda")
    ipt = torch.from_numpy(ip.astype(np.int32)).to(dev)
    idt = torch.from_numpy(idx.astype(np.int32)).to(dev)
    dat = torch.from_numpy(rng.standard_normal(int(ip[-1]))).to(dev)
    torch.cuda.synchronize()
    device_cases("hot_only", G.DeviceCsr(ctx, rows, cols, ipt, idt, dat), rows, cols)
    np.savez(out_path, **res)


def _child(tmp_path, name, **env):
    out = os.path.join(str(tmp_path), name + ".npz")
    e = dict(os.environ, SPRS_B200_E2E_MIN_TILES="1", SPRS_B200_E2E_CHUNKS="5", **env)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), out], capture_output=True,
                       text=True, timeout=900, env=e, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    return dict(np.load(out))


def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))


@pytest.mark.gpu
@pytest.mark.parametrize("indptr64", ["0", "1"])
def test_spmv_hot_set_bit_identical_child_process(tmp_path, indptr64):
    """Hot set off versus forced to K = 1023 and 1024 (the staging loop's stride: one slot per
    thread, and one short of it) and 24576 (the default: the largest stage, next to the
    multi-target kernel's own); with SPRS_B200_FORCE_INDPTR64 the uint64 instantiations."""
    ks = ["24576"] if indptr64 == "1" else ["1023", "1024", "24576"]
    ref = _child(tmp_path, "off", SPRS_B200_SPMV_HOT="0", SPRS_B200_FORCE_INDPTR64=indptr64)
    for key in ref:
        if "/multi" in key:  # every target holds the plain SpMV's y, nothing outside it
            y = ref[key.split("/")[0] + "/y"]
            assert all(_same_bits(t[2:-14], y) for t in ref[key]), key
            assert np.all(ref[key][:, :2] == -7.0) and np.all(ref[key][:, -14:] == -7.0), key
        if key.endswith("/host_chunked"):
            assert _same_bits(ref[key], ref[key.split("/")[0] + "/y"]), key
    for k in ks:
        got = _child(tmp_path, "k" + k, SPRS_B200_SPMV_HOT=k, SPRS_B200_FORCE_INDPTR64=indptr64)
        assert sorted(got) == sorted(ref)
        for key in ref:
            assert _same_bits(got[key], ref[key]), "K=%s: %s differs from the SpMV without a hot set" % (k, key)


if __name__ == "__main__":
    _cases(sys.argv[1])
