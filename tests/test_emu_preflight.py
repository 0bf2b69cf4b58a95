"""CPU pre-flight of the CUDA kernels' LOGIC on tests/emu (a CUDA-subset emulator: one fiber
per thread, warp collectives, block barriers, mbarrier/TMA bookkeeping; see tests/emu/cuemu.h).

The library's own sources are compiled for the CPU, unmodified apart from a mechanical
rewrite of launches / shared-memory declarations / the PTX wrappers, into a SEPARATE library
that only this file and `SPRS_B200_EMU=1 pytest -m gpu` load.  This finds indexing, barrier
and host-sequencing bugs where no GPU is attached; it is NOT parity evidence (that is the
`-m gpu` suite on the H100) and says nothing about performance or the hardware memory model.
"""
import os
import subprocess
import sys

import pytest

from conftest import ROOT, emu_library

EMU = os.path.join(ROOT, "tests", "emu")
CXX = "/usr/bin/g++"


@pytest.fixture(scope="module")
def emu():
    return emu_library()


def _link_and_run(emu_lib, src, name):
    exe = os.path.join(EMU, "build", name)
    subprocess.check_call([CXX, "-O1", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "cpp", src),
                           "-L" + EMU, "-lsprs_b200_emu", "-Wl,-rpath," + EMU])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.rstrip().splitlines()[-1].startswith("OK "), r.stdout
    return r.stdout


def test_emu_cpp_reference_kats(emu, monkeypatch):
    """tests/cpp/test_reference_kats.cpp (the reference's product tests through the C++ host
    mirror) linked against the emulated library; forward and reverse thread schedules."""
    _link_and_run(emu, "test_reference_kats.cpp", "kats_emu")
    monkeypatch.setenv("CUEMU_SCHEDULE", "reverse")
    _link_and_run(emu, "test_reference_kats.cpp", "kats_emu")


def test_emu_cpp_bicgstab(emu):
    """bicgstab.rs:356-390 through the emulated solver kernels: the 4x4 system converges to an
    exactly zero residual like the oracle (iteration 45, three hard restarts)."""
    out = _link_and_run(emu, "test_bicgstab.cpp", "bicgstab_emu")
    assert "Iteration count 45" in out and "Hard restart count 3" in out


def _pytest_child(env_extra, args, timeout):
    env = dict(os.environ, SPRS_B200_EMU="1", **env_extra)
    return subprocess.Popen([sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider"] + args,
                            stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, env=env, cwd=ROOT), timeout


def test_emu_gpu_suite(emu):
    """Every `-m gpu` test that needs only the C ABI (all but the full-size ones, the
    multi-GPU ones and the natively linked C++ drivers) passes on the emulator -- under the
    default thread schedule and under a shuffled one (any order is a legal CUDA schedule, so a
    result that depends on it means a missing barrier) -- and so do the opt-in L2-blocked /
    chunked host path and the uint64-indptr kernel instantiations (each of those in child
    processes with its environment switch).  The three runs are independent processes and run
    side by side to keep the CPU suite short."""  # noqa
    suite = [os.path.join(ROOT, "tests"), "-k",
             "not full_size and not test_cpp and not indptr64 and not child_process and not test_comm"]
    runs = {
        "forward": _pytest_child({"CUEMU_SCHEDULE": "forward"}, suite, 1500),
        "random:7": _pytest_child({"CUEMU_SCHEDULE": "random:7"}, suite, 1500),
        "variants": _pytest_child({}, [os.path.join(ROOT, "tests", "test_gpu_zz_late.py"),
                                       os.path.join(ROOT, "tests", "test_gpu_zzz_e2e_chunked.py"), "-k",
                                       "indptr64 or child_process"], 900),
    }
    failures = []
    for name, (proc, timeout) in runs.items():
        try:
            out, err = proc.communicate(timeout=timeout)
        except subprocess.TimeoutExpired:
            proc.kill()
            out, err = proc.communicate()
            failures.append("%s: timed out\n%s" % (name, out[-1500:]))
            continue
        tail = "\n".join(out.splitlines()[-25:])
        if proc.returncode != 0 or " passed" not in tail or "failed" in tail:
            failures.append("%s: exit %d\n%s\n%s" % (name, proc.returncode, tail, err[-2000:]))
    assert not failures, "\n\n".join(failures)


def test_emu_structure_fuzz(emu):
    """tools/fuzz_emu.py: matrices whose row lengths sit on the kernels' internal boundaries
    (tile sizes, register-path row counts, lane groups, SpGEMM bins) through every product of
    the C ABI against the oracle; a fixed slice of the campaign that found nothing else in ~15000
    cases across the default and opt-in kernel variants."""
    runs = [({}, "1"), ({"SPRS_B200_SPMV_VARIANT": "512,8"}, "50001"),
            ({"SPRS_B200_FORCE_INDPTR64": "1", "SPRS_B200_E2E_CHUNKS": "3",
              "SPRS_B200_E2E_MIN_TILES": "1"}, "90001")]
    procs = [subprocess.Popen([sys.executable, os.path.join(ROOT, "tools", "fuzz_emu.py"), "--cases", "40",
                               "--seed", seed], env=dict(os.environ, **env), cwd=ROOT,
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
             for env, seed in runs]
    for p in procs:
        out, _ = p.communicate(timeout=900)
        assert p.returncode == 0 and "0 failing" in out, out[-3000:]
