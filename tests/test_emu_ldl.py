"""CPU pre-flight of the LDL^T factorization (csrc/ldl.cu, with the triangular solves of
csrc/trisolve.cu it uses) on the emulator, using the emulated build that has them
(tests/emu_ldl.py).  The emulator runs the CTAs of a launch one after another and the lanes of a
warp in the order its schedule picks, so these runs also check that the ticket order makes
progress without co-resident CTAs and that the lanes of a row are ordered where they share data:

  * the small tests of tests/test_gpu_ldl.py -- KATs, storages and permutations, Laplacians,
    forests, signed zeros and non-finite values, zero pivots, update, solve_dev, the panics --
    under the forward and a shuffled thread schedule;
  * tests/cpp/test_ldl_kats.cpp through the C++ host mirror."""
import os
import subprocess
import sys

from conftest import ROOT
from emu_ldl import emu_ldl_library

SMALL = "not large and not test_cpp and not child_process"


def test_emu_ldl_suite(tmp_path):
    lib = emu_ldl_library()
    env = dict(os.environ, SPRS_B200_EMU="1", SPRS_B200_EMU_LDL_LIB=lib)
    procs = {}
    for sched in ("forward", "random:7"):
        procs["gpu file, " + sched] = subprocess.Popen(
            [sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-p", "no:cacheprovider",
             os.path.join(ROOT, "tests", "test_gpu_ldl.py"), "-k", SMALL],
            env=dict(env, CUEMU_SCHEDULE=sched), cwd=ROOT, stdout=subprocess.PIPE,
            stderr=subprocess.STDOUT, text=True)
    exe = str(tmp_path / "ldl_kats_emu")
    lib_dir = os.path.dirname(lib)
    subprocess.check_call(["/usr/bin/g++", "-O1", "-std=c++17", "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "test_ldl_kats.cpp"),
                           "-L" + lib_dir, "-lsprs_b200_emu_ldl", "-Wl,-rpath," + lib_dir])
    for sched in ("forward", "reverse"):
        r = subprocess.run([exe], capture_output=True, text=True, timeout=600,
                           env=dict(os.environ, CUEMU_SCHEDULE=sched))
        assert r.returncode == 0 and r.stdout.startswith("OK "), r.stdout + r.stderr
    failures = []
    for name, p in procs.items():
        out, _ = p.communicate(timeout=1800)
        tail = "\n".join(out.splitlines()[-15:])
        ok = " passed" in tail and "failed" not in tail
        if p.returncode != 0 or not ok:
            failures.append("%s: exit %d\n%s" % (name, p.returncode, out[-2500:]))
    assert not failures, "\n\n".join(failures)
