"""CPU pre-flight of the triangular solves (csrc/trisolve.cu) on the emulator, using the emulated
build that has them (tests/emu_trisolve.py).  The emulator runs the CTAs of a launch one after
another, so these runs also check that the ticket order makes progress without co-resident CTAs:

  * the small tests of tests/test_gpu_trisolve.py -- KATs, values, NaN / Inf, singular
    matrices, shapes, the usolve_csc order, the plan, the panics -- under the forward and a
    shuffled thread schedule;
  * tests/cpp/test_trisolve_kats.cpp through the C++ host mirror."""
import os
import subprocess
import sys

from conftest import ROOT
from emu_trisolve import emu_trisolve_library

SMALL = "not full_size and not test_cpp and not child_process and not large"


def test_emu_trisolve_suite(tmp_path):
    lib = emu_trisolve_library()
    env = dict(os.environ, SPRS_B200_EMU="1", SPRS_B200_EMU_TRISOLVE_LIB=lib)
    procs = {}
    for sched in ("forward", "random:7"):
        procs["gpu file, " + sched] = subprocess.Popen(
            [sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-p", "no:cacheprovider",
             os.path.join(ROOT, "tests", "test_gpu_trisolve.py"), "-k", SMALL],
            env=dict(env, CUEMU_SCHEDULE=sched), cwd=ROOT, stdout=subprocess.PIPE,
            stderr=subprocess.STDOUT, text=True)
    exe = str(tmp_path / "trisolve_kats_emu")
    lib_dir = os.path.dirname(lib)
    subprocess.check_call(["/usr/bin/g++", "-O1", "-std=c++17", "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "test_trisolve_kats.cpp"),
                           "-L" + lib_dir, "-lsprs_b200_emu_trisolve", "-Wl,-rpath," + lib_dir])
    for sched in ("forward", "reverse"):
        r = subprocess.run([exe], capture_output=True, text=True, timeout=600,
                           env=dict(os.environ, CUEMU_SCHEDULE=sched))
        assert r.returncode == 0 and r.stdout.startswith("OK "), r.stdout + r.stderr
    failures = []
    for name, p in procs.items():
        out, _ = p.communicate(timeout=1800)
        tail = "\n".join(out.splitlines()[-15:])
        ok = " passed" in tail and "failed" not in tail and "skipped" not in tail
        if p.returncode != 0 or not ok:
            failures.append("%s: exit %d\n%s" % (name, p.returncode, out[-2500:]))
    assert not failures, "\n\n".join(failures)
