"""TEST INFRASTRUCTURE ONLY: the CPU-emulated library (tests/emu) with csrc/trisolve.cu and
csrc/ldl.cu in it.

Built the same way as the triangular solves' emulated library (tests/emu_trisolve.py): each
source rewritten by tests/emu/transform.py, prefixed with the same stand-ins for the device
functions beyond the emulator's subset (acquire / release as plain accesses: one OS thread
runs every CUDA thread), compiled with the emulator's flags and linked with the emulator's own
objects into tests/emu/build/ldl/libsprs_b200_emu_ldl.so.  The factorization's solves run on
the triangular-solve kernel, so both sources are in it.  Loaded only by tests/test_emu_ldl.py
through the `SPRS_B200_EMU_LDL_LIB` hook of tests/test_gpu_ldl.py.
"""
import glob
import hashlib
import os
import re
import subprocess
import sys

from conftest import ROOT, emu_library
from emu_binop import CXXFLAGS, EMU, GEN
from emu_trisolve import STAND_INS

SOURCES = ("trisolve.cu", "ldl.cu")


def emu_ldl_library():
    """Path of the emulated library with the factorization; rebuilt when a source changed."""
    emu_library()  # the emulator's objects and the rewritten headers under GEN
    sys.path.insert(0, EMU)
    import transform
    srcs = {name: STAND_INS + transform.transform(
        name, open(os.path.join(ROOT, "sprs_b200", "csrc", name)).read()) for name in SOURCES}
    names = re.search(r"^SRCS = (.*)$", open(os.path.join(EMU, "Makefile")).read(), re.M).group(1)
    base = [os.path.join(EMU, "build", n + ".o") for n in names.split() + ["cuemu"]]
    key = hashlib.sha1(b"".join(srcs[n].encode() for n in SOURCES) +
                       b"".join(open(o, "rb").read() for o in base) +
                       b"".join(open(h, "rb").read() for h in sorted(glob.glob(os.path.join(GEN, "*.cuh"))))
                       ).hexdigest()[:12]
    out = os.path.join(EMU, "build", "ldl")
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, "libsprs_b200_emu_ldl.so")
    stamp = os.path.join(out, "key")
    if os.path.exists(so) and os.path.exists(stamp) and open(stamp).read() == key:
        return so
    tag = ".%d" % os.getpid()
    objs = []
    for name in SOURCES:
        stem = name[:-3]
        cpp, obj = os.path.join(out, stem + tag + ".cpp"), os.path.join(out, stem + tag + ".o")
        with open(cpp, "w") as f:
            f.write(srcs[name])
        subprocess.check_call(["/usr/bin/g++"] + CXXFLAGS + ["-I" + EMU, "-I" + GEN, "-c", cpp,
                                                             "-o", obj])
        os.remove(cpp)
        objs.append(obj)
    subprocess.check_call(["/usr/bin/g++", "-shared", "-o", so + tag] + base + objs)
    os.replace(so + tag, so)
    with open(stamp + tag, "w") as f:
        f.write(key)
    os.replace(stamp + tag, stamp)
    for obj in objs:
        os.remove(obj)
    return so
