"""TEST INFRASTRUCTURE ONLY: the CPU-emulated library (tests/emu) with csrc/construct.cu in it.

Built the same way as tests/emu_binop.py: construct.cu -- and binop.cu, whose result helpers
(new_result / alloc_result / finish_result) it uses -- rewritten by tests/emu/transform.py,
compiled with the emulator's flags against tests/emu/cuemu.h and linked with the emulator's own
objects into tests/emu/build/construct/libsprs_b200_emu_construct.so.  Loaded only by
tests/test_emu_construct.py and the `SPRS_B200_EMU_CONSTRUCT_LIB` hook of
tests/test_gpu_construct.py.
"""
import glob
import hashlib
import os
import re
import subprocess
import sys

from conftest import ROOT, emu_library
from emu_binop import CXXFLAGS

EMU = os.path.join(ROOT, "tests", "emu")
GEN = os.path.join(EMU, "build", "gen", "a", "b")  # transform.py's output (tests/emu/Makefile)
SOURCES = ("binop.cu", "construct.cu")


def emu_construct_library():
    """Path of the emulated library with the construction kernels; rebuilt when a source
    changed."""
    emu_library()  # the emulator's objects and the rewritten headers under GEN
    sys.path.insert(0, EMU)
    import transform
    srcs = [transform.transform(n, open(os.path.join(ROOT, "sprs_b200", "csrc", n)).read())
            for n in SOURCES]
    names = re.search(r"^SRCS = (.*)$", open(os.path.join(EMU, "Makefile")).read(), re.M).group(1)
    base = [os.path.join(EMU, "build", n + ".o") for n in names.split() + ["cuemu"]]
    key = hashlib.sha1("".join(srcs).encode() + b"".join(open(o, "rb").read() for o in base) +
                       b"".join(open(h, "rb").read() for h in sorted(glob.glob(os.path.join(GEN, "*.cuh"))))
                       ).hexdigest()[:12]
    out = os.path.join(EMU, "build", "construct")
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, "libsprs_b200_emu_construct.so")
    stamp = os.path.join(out, "key")
    if os.path.exists(so) and os.path.exists(stamp) and open(stamp).read() == key:
        return so
    tag = ".%d" % os.getpid()
    objs = []
    for name, src in zip(SOURCES, srcs):
        stem = name[:-3]
        cpp, obj = os.path.join(out, stem + tag + ".cpp"), os.path.join(out, stem + tag + ".o")
        with open(cpp, "w") as f:
            f.write(src)
        subprocess.check_call(["/usr/bin/g++"] + CXXFLAGS + ["-I" + EMU, "-I" + GEN, "-c", cpp,
                                                            "-o", obj])
        os.remove(cpp)
        objs.append(obj)
    subprocess.check_call(["/usr/bin/g++", "-shared", "-o", so + tag] + base + objs)
    os.replace(so + tag, so)
    with open(stamp + tag, "w") as f:
        f.write(key)
    os.replace(stamp + tag, stamp)
    for o in objs:
        os.remove(o)
    return so
