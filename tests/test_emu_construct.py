"""CPU pre-flight of the sparse matrix construction (csrc/construct.cu) on the emulator (see
tests/test_emu_preflight.py), using the emulated build that has it (tests/emu_construct.py):

  * the small tests of tests/test_gpu_construct.py -- KATs, panics, every storage combination,
    mixed indptr widths, the tile seams, edge shapes, value classes, composition -- under the
    forward and a shuffled thread schedule, and with 64-bit indptr forced;
  * tests/cpp/test_construct_kats.cpp through the C++ host mirror, forward and reverse
    schedules."""
import os
import subprocess
import sys

from conftest import ROOT
from emu_construct import emu_construct_library

SMALL = "not full_size and not test_cpp and not child_process"


def test_emu_construct_suite(tmp_path):
    lib = emu_construct_library()
    env = dict(os.environ, SPRS_B200_EMU="1", SPRS_B200_EMU_CONSTRUCT_LIB=lib)
    procs = {}
    for name, extra in (("forward", {"CUEMU_SCHEDULE": "forward"}),
                        ("random:7", {"CUEMU_SCHEDULE": "random:7"}),
                        ("indptr64", {"SPRS_B200_FORCE_INDPTR64": "1"})):
        procs[name] = subprocess.Popen(
            [sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-p", "no:cacheprovider",
             os.path.join(ROOT, "tests", "test_gpu_construct.py"), "-k", SMALL],
            env=dict(env, **extra), cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
            text=True)
    exe = str(tmp_path / "construct_kats_emu")
    lib_dir = os.path.dirname(lib)
    subprocess.check_call(["/usr/bin/g++", "-O1", "-std=c++17", "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "test_construct_kats.cpp"),
                           "-L" + lib_dir, "-lsprs_b200_emu_construct", "-Wl,-rpath," + lib_dir])
    for sched in ("forward", "reverse"):
        r = subprocess.run([exe], capture_output=True, text=True, timeout=600,
                           env=dict(os.environ, CUEMU_SCHEDULE=sched))
        assert r.returncode == 0 and r.stdout.startswith("OK "), r.stdout + r.stderr
    failures = []
    for name, p in procs.items():
        out, _ = p.communicate(timeout=1800)
        tail = "\n".join(out.splitlines()[-15:])
        if p.returncode != 0 or " passed" not in tail or "failed" in tail or "skipped" in tail:
            failures.append("%s: exit %d\n%s" % (name, p.returncode, out[-2500:]))
    assert not failures, "\n\n".join(failures)
