"""CPU pre-flight of the SpMV hot set on tests/emu (see tests/test_emu_preflight.py): a slice of
tools/fuzz_emu.py with the hot set forced to K = 8 slots on every mirror, so that tagged
(shared-memory) and untagged (global) gathers mix inside one warp instruction, through every
SpMV entry point against the oracle -- plain, accumulating, CSC, row slices, the pipelined
pushes and the multi-target kernel, and the chunked host path."""
import os
import subprocess
import sys

from conftest import ROOT, emu_library


def test_emu_structure_fuzz_hot_set():
    emu_library()
    runs = [({"SPRS_B200_SPMV_HOT": "8"}, "120001"),
            ({"SPRS_B200_SPMV_HOT": "8", "SPRS_B200_FORCE_INDPTR64": "1", "SPRS_B200_E2E_CHUNKS": "3",
              "SPRS_B200_E2E_MIN_TILES": "1"}, "130001")]
    procs = [subprocess.Popen([sys.executable, os.path.join(ROOT, "tools", "fuzz_emu.py"), "--cases", "30",
                               "--seed", seed], env=dict(os.environ, **env), cwd=ROOT,
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
             for env, seed in runs]
    for p in procs:
        out, _ = p.communicate(timeout=900)
        assert p.returncode == 0 and "0 failing" in out, out[-3000:]
