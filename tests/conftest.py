import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def emu_library():
    """tests/emu: the library's kernels compiled for the CPU against a CUDA-subset emulator.
    TEST INFRASTRUCTURE (kernel-logic pre-flight where no GPU is attached); never loaded by
    the package itself."""
    import subprocess
    d = os.path.join(ROOT, "tests", "emu")
    asan = os.environ.get("SPRS_B200_EMU_ASAN") == "1"  # needs LD_PRELOAD=libasan.so
    subprocess.check_call(["make", "-C", d, "-s"] + (["asan"] if asan else []),
                          stdout=subprocess.DEVNULL)
    return os.path.join(d, "build/asan/libsprs_b200_emu.so" if asan else "libsprs_b200_emu.so")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")
    if os.environ.get("SPRS_B200_EMU") == "1":
        # developer switch: run `-m gpu` tests against the emulator (those that only need the
        # C ABI and numpy work; the ones that allocate through torch.cuda do not)
        import sprs_b200
        import torch
        from sprs_b200 import generate
        sprs_b200._lib.LIB_PATH = emu_library()
        # "device" memory of the emulator is host memory: the bench/test plumbing that
        # allocates through torch uses CPU tensors there
        generate._device = lambda ctx: torch.device("cpu")
        generate._stream_ptr = lambda: None
        generate._sync = lambda: None


@pytest.fixture(scope="session")
def fixtures():
    """The reference's own known-answer data (tests/golden/make_fixtures.py)."""
    with open(os.path.join(ROOT, "tests", "golden", "sprs_fixtures.json")) as f:
        return json.load(f)


def mat_arrays(m, idx_dtype=np.uint32, ptr_dtype=None):
    ptr_dtype = ptr_dtype or idx_dtype
    return (np.array(m["indptr"], dtype=ptr_dtype), np.array(m["indices"], dtype=idx_dtype),
            np.array(m["data"], dtype=np.float64))


def rand_csr(rng, rows, cols, nnz_per_row, idx_dtype=np.uint32, skew=False, empty_frac=0.0):
    """Random CSR with strictly ascending unique columns per row (sprs invariant,
    sparse.rs:360-369).  skew=True draws power-law row lengths."""
    if skew:
        lens = np.minimum((rng.pareto(1.2, rows) * nnz_per_row * 0.3).astype(np.int64), cols)
    else:
        lens = rng.poisson(nnz_per_row, rows).astype(np.int64)
        lens = np.minimum(lens, cols)
    if empty_frac > 0:
        lens[rng.random(rows) < empty_frac] = 0
    indptr = np.zeros(rows + 1, dtype=np.int64)
    np.cumsum(lens, out=indptr[1:])
    indices = np.empty(indptr[-1], dtype=np.int64)
    for r in range(rows):
        n = lens[r]
        if n == 0:
            continue
        if n * 4 < cols:
            c = np.unique(rng.integers(0, cols, size=int(n * 1.3) + 8))
            while len(c) < n:
                c = np.unique(np.concatenate([c, rng.integers(0, cols, size=int(n) + 8)]))
            c = np.sort(rng.choice(c, size=n, replace=False))
        else:
            c = np.sort(rng.choice(cols, size=n, replace=False))
        indices[indptr[r]:indptr[r + 1]] = c
    data = rng.standard_normal(indptr[-1])
    return indptr.astype(idx_dtype), indices.astype(idx_dtype), data
