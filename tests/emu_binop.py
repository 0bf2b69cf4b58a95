"""TEST INFRASTRUCTURE ONLY: the CPU-emulated library (tests/emu) with csrc/binop.cu in it.

tests/emu builds libsprs_b200_emu.so from a fixed list of the library's sources; the binop
kernels are added here the same way -- binop.cu rewritten by tests/emu/transform.py, compiled
with the emulator's flags against tests/emu/cuemu.h -- and linked with the emulator's own objects
into tests/emu/build/binop/libsprs_b200_emu_binop.so.  Loaded only by tests/test_emu_binop.py,
the `SPRS_B200_EMU_BINOP_LIB` hook of tests/test_gpu_binop.py and `tools/fuzz_emu.py --binop`.
"""
import glob
import hashlib
import os
import re
import subprocess
import sys

from conftest import ROOT, emu_library

EMU = os.path.join(ROOT, "tests", "emu")
GEN = os.path.join(EMU, "build", "gen", "a", "b")  # transform.py's output (tests/emu/Makefile)
CXXFLAGS = ["-O1", "-g", "-std=c++17", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas",
            "-Wno-unused-function", "-Wno-unused-variable", "-Wno-unused-but-set-variable",
            "-Wno-sign-compare"]


def emu_binop_library():
    """Path of the emulated library with the binops; rebuilt when a source changed."""
    emu_library()  # the emulator's objects and the rewritten headers under GEN
    sys.path.insert(0, EMU)
    import transform
    src = transform.transform("binop.cu",
                              open(os.path.join(ROOT, "sprs_b200", "csrc", "binop.cu")).read())
    # the emulator's own objects: SRCS of tests/emu/Makefile + cuemu.o
    srcs = re.search(r"^SRCS = (.*)$", open(os.path.join(EMU, "Makefile")).read(), re.M).group(1)
    base = [os.path.join(EMU, "build", n + ".o") for n in srcs.split() + ["cuemu"]]
    key = hashlib.sha1(src.encode() + b"".join(open(o, "rb").read() for o in base) +
                       b"".join(open(h, "rb").read() for h in sorted(glob.glob(os.path.join(GEN, "*.cuh"))))
                       ).hexdigest()[:12]
    out = os.path.join(EMU, "build", "binop")
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, "libsprs_b200_emu_binop.so")
    stamp = os.path.join(out, "key")
    if os.path.exists(so) and os.path.exists(stamp) and open(stamp).read() == key:
        return so
    tag = ".%d" % os.getpid()
    cpp, obj = os.path.join(out, "binop%s.cpp" % tag), os.path.join(out, "binop%s.o" % tag)
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
