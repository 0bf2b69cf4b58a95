"""CPU pre-flight of tests/test_gpu_zzz_trisolve_ldl_bits.py on the emulated build with the
triangular solves and the LDL^T factorization (tests/emu_ldl.py).  The emulator reports 4 SMs, so
the first ticket wave is 256 warps and every wave seam of that file is real here; it runs the
CTAs of a launch one after another and the lanes of a warp in the order its schedule picks.

Its small cases run under the forward and a shuffled thread schedule; the full-size ones, the
64-bit indptr child and the two-stream test (CUDA streams) need the H100."""
import os
import subprocess
import sys

from conftest import ROOT
from emu_ldl import emu_ldl_library

SMALL = "not full_size and not child_process and not streams"


def test_emu_trisolve_ldl_bits(tmp_path):
    lib = emu_ldl_library()
    env = dict(os.environ, SPRS_B200_EMU="1", SPRS_B200_EMU_LDL_LIB=lib)
    procs = {}
    for sched in ("forward", "random:7"):
        procs["gpu file, " + sched] = subprocess.Popen(
            [sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-p", "no:cacheprovider",
             os.path.join(ROOT, "tests", "test_gpu_zzz_trisolve_ldl_bits.py"), "-k", SMALL],
            env=dict(env, CUEMU_SCHEDULE=sched), cwd=ROOT, stdout=subprocess.PIPE,
            stderr=subprocess.STDOUT, text=True)
    failures = []
    for name, p in procs.items():
        out, _ = p.communicate(timeout=3000)
        tail = "\n".join(out.splitlines()[-15:])
        ok = " passed" in tail and "failed" not in tail and "skipped" not in tail
        if p.returncode != 0 or not ok:
            failures.append("%s: exit %d\n%s" % (name, p.returncode, out[-2500:]))
    assert not failures, "\n\n".join(failures)
