"""TEST INFRASTRUCTURE ONLY: the CPU-emulated library (tests/emu) with csrc/trisolve.cu in it.

tests/emu builds libsprs_b200_emu.so from a fixed list of the library's sources; the triangular
solves are added here the same way as the binops (tests/emu_binop.py) -- trisolve.cu rewritten
by tests/emu/transform.py, compiled with the emulator's flags against tests/emu/cuemu.h, linked
with the emulator's own objects into tests/emu/build/trisolve/libsprs_b200_emu_trisolve.so.
The few device functions the solve uses beyond the emulator's subset are stated below: a
single OS thread runs every CUDA thread there, so acquire / release are plain accesses.  Loaded
only by tests/test_emu_trisolve.py and the `SPRS_B200_EMU_TRISOLVE_LIB` hook of
tests/test_gpu_trisolve.py.
"""
import glob
import hashlib
import os
import re
import subprocess
import sys

from conftest import ROOT, emu_library
from emu_binop import CXXFLAGS, EMU, GEN

STAND_INS = r"""#include "cuemu.h"
static inline uint32_t ld_acquire_u32(const uint32_t* p) { return *(const volatile uint32_t*)p; }
static inline void st_release_u32(uint32_t* p, uint32_t v) {
    *(volatile uint32_t*)p = v;
    cuemu::note_progress();
}
static inline double __ddiv_rn(double a, double b) { return a / b; }
"""


def emu_trisolve_library():
    """Path of the emulated library with the triangular solves; rebuilt when a source changed."""
    emu_library()  # the emulator's objects and the rewritten headers under GEN
    sys.path.insert(0, EMU)
    import transform
    src = STAND_INS + transform.transform(
        "trisolve.cu", open(os.path.join(ROOT, "sprs_b200", "csrc", "trisolve.cu")).read())
    srcs = re.search(r"^SRCS = (.*)$", open(os.path.join(EMU, "Makefile")).read(), re.M).group(1)
    base = [os.path.join(EMU, "build", n + ".o") for n in srcs.split() + ["cuemu"]]
    key = hashlib.sha1(src.encode() + b"".join(open(o, "rb").read() for o in base) +
                       b"".join(open(h, "rb").read() for h in sorted(glob.glob(os.path.join(GEN, "*.cuh"))))
                       ).hexdigest()[:12]
    out = os.path.join(EMU, "build", "trisolve")
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, "libsprs_b200_emu_trisolve.so")
    stamp = os.path.join(out, "key")
    if os.path.exists(so) and os.path.exists(stamp) and open(stamp).read() == key:
        return so
    tag = ".%d" % os.getpid()
    cpp, obj = os.path.join(out, "trisolve%s.cpp" % tag), os.path.join(out, "trisolve%s.o" % tag)
    with open(cpp, "w") as f:
        f.write(src)
    subprocess.check_call(["/usr/bin/g++"] + CXXFLAGS + ["-I" + EMU, "-I" + GEN, "-c", cpp, "-o", obj])
    subprocess.check_call(["/usr/bin/g++", "-shared", "-o", so + tag] + base + [obj])
    os.replace(so + tag, so)
    with open(stamp + tag, "w") as f:
        f.write(key)
    os.replace(stamp + tag, stamp)
    os.remove(cpp)
    os.remove(obj)
    return so
