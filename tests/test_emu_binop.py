"""CPU pre-flight of the sparse binops (csrc/binop.cu) on the emulator (see
tests/test_emu_preflight.py), using the emulated build that has them (tests/emu_binop.py):

  * the small tests of tests/test_gpu_binop.py -- KATs, mixed storage, panics, the seam matrix,
    value classes, index widths, composition -- under the forward and a shuffled thread schedule;
  * tests/cpp/test_binop_kats.cpp through the C++ host mirror, forward and reverse schedules;
  * a fixed slice of `tools/fuzz_emu.py --binop`: row lengths on the tile, lane and snap
    boundaries, random ops, forced overlaps and cancellations, CSR and CSC, with 32- and 64-bit
    indptr -- against the binop oracle bit for bit."""
import os
import subprocess
import sys

from conftest import ROOT
from emu_binop import emu_binop_library

SMALL = "not full_size and not test_cpp and not indptr64 and not child_process"


def test_emu_binop_suite(tmp_path):
    lib = emu_binop_library()
    env = dict(os.environ, SPRS_B200_EMU="1", SPRS_B200_EMU_BINOP_LIB=lib)
    procs = {}
    for sched in ("forward", "random:7"):
        procs["gpu file, " + sched] = subprocess.Popen(
            [sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-p", "no:cacheprovider",
             os.path.join(ROOT, "tests", "test_gpu_binop.py"), "-k", SMALL],
            env=dict(env, CUEMU_SCHEDULE=sched), cwd=ROOT, stdout=subprocess.PIPE,
            stderr=subprocess.STDOUT, text=True)
    for name, extra, seed in (("fuzz", {}, "1"), ("fuzz, random:7", {"CUEMU_SCHEDULE": "random:7"}, "501"),
                              ("fuzz, indptr64", {"SPRS_B200_FORCE_INDPTR64": "1"}, "1001")):
        procs[name] = subprocess.Popen(
            [sys.executable, os.path.join(ROOT, "tools", "fuzz_emu.py"), "--binop", "--cases", "40",
             "--seed", seed], env=dict(os.environ, **extra), cwd=ROOT, stdout=subprocess.PIPE,
            stderr=subprocess.STDOUT, text=True)
    exe = str(tmp_path / "binop_kats_emu")
    lib_dir = os.path.dirname(lib)
    subprocess.check_call(["/usr/bin/g++", "-O1", "-std=c++17", "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "test_binop_kats.cpp"),
                           "-L" + lib_dir, "-lsprs_b200_emu_binop", "-Wl,-rpath," + lib_dir])
    for sched in ("forward", "reverse"):
        r = subprocess.run([exe], capture_output=True, text=True, timeout=600,
                           env=dict(os.environ, CUEMU_SCHEDULE=sched))
        assert r.returncode == 0 and r.stdout.startswith("OK "), r.stdout + r.stderr
    failures = []
    for name, p in procs.items():
        out, _ = p.communicate(timeout=900)
        tail = "\n".join(out.splitlines()[-15:])
        ok = " passed" in tail and "failed" not in tail and "skipped" not in tail \
            if name.startswith("gpu") else "0 failing" in out
        if p.returncode != 0 or not ok:
            failures.append("%s: exit %d\n%s" % (name, p.returncode, out[-2500:]))
    assert not failures, "\n\n".join(failures)
