"""Compile the unmodified DBoW3 sources of the reference (DBoW3Py/DBoW3/src) with the OpenCV stand-in header under
include/ and driver.cpp into oracle/_ref/libdbow3_ref.so: the reference bag-of-words implementation that
tools/make_golden_loop.py and tools/loop_stream.py call through ctypes.

    python -m oracle.dbow3_ref.build [reference root]

Explicit flags, no -march=native; -ffp-contract=off keeps every multiply and add separately rounded.  Nothing is built
(and None is returned) when the reference sources are absent."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT_DIR = os.path.join(os.path.dirname(HERE), "_ref")
LIB = os.path.join(OUT_DIR, "libdbow3_ref.so")
REFERENCE_ROOT = os.environ.get("VISTA_SLAM_REFERENCE", "/root/reference")
CXX_SOURCES = ["Vocabulary.cpp", "DescManip.cpp", "ScoringObject.cpp", "BowVector.cpp", "FeatureVector.cpp"]
FLAGS = ["-O2", "-fPIC", "-ffp-contract=off"]


def src_dir(root=REFERENCE_ROOT):
    return os.path.join(root, "DBoW3Py", "DBoW3", "src")


def build(root=REFERENCE_ROOT, force=False):
    src = src_dir(root)
    if not os.path.isdir(src):
        return None
    inputs = [os.path.join(src, f) for f in CXX_SOURCES + ["quicklz.c"]] + [os.path.join(HERE, "driver.cpp"),
                                                                            os.path.join(HERE, "include", "opencv2",
                                                                                         "core", "core.hpp")]
    if not force and os.path.exists(LIB) and all(os.path.getmtime(LIB) >= os.path.getmtime(f) for f in inputs):
        return LIB
    os.makedirs(OUT_DIR, exist_ok=True)
    objs = []
    inc = ["-I", os.path.join(HERE, "include"), "-I", src]
    for f in CXX_SOURCES + ["driver.cpp"]:
        path = os.path.join(HERE if f == "driver.cpp" else src, f)
        obj = os.path.join(OUT_DIR, f.replace(".cpp", ".o"))
        subprocess.run(["g++", "-std=c++14"] + FLAGS + inc + ["-c", path, "-o", obj], check=True)
        objs.append(obj)
    obj = os.path.join(OUT_DIR, "quicklz.o")
    subprocess.run(["gcc"] + FLAGS + ["-c", os.path.join(src, "quicklz.c"), "-o", obj], check=True)
    objs.append(obj)
    subprocess.run(["g++", "-shared", "-o", LIB] + objs, check=True)
    return LIB


def load():
    """ctypes handle of the compiled reference, or None when it has not been built."""
    import ctypes
    if not os.path.exists(LIB):
        return None
    L = ctypes.CDLL(LIB)
    vp, i, u8p, ip, dp = (ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p)
    L.dbow_create.restype = vp
    L.dbow_create.argtypes = [u8p, ip, i, i, i, i, i, ctypes.c_uint]
    L.dbow_load.restype = vp
    L.dbow_load.argtypes = [ctypes.c_char_p, ctypes.c_char_p, i]
    L.dbow_save.argtypes = [vp, ctypes.c_char_p, i]
    L.dbow_free.argtypes = [vp]
    L.dbow_free.restype = None
    L.dbow_nodes.argtypes = [vp]
    L.dbow_dump.argtypes = [vp, ip, ip, dp, u8p, ip, ip]
    L.dbow_transform.argtypes = [vp, u8p, i, ip, dp, i]
    L.dbow_score.restype = ctypes.c_double
    L.dbow_score.argtypes = [vp, ip, dp, i, ip, dp, i]
    return L


if __name__ == "__main__":
    print(build(*(sys.argv[1:2] or [REFERENCE_ROOT]), force=True))
