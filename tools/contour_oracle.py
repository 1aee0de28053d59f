"""Loader of the contour oracle (tools/contour_oracle.c): compiles it with the C compiler into a temporary directory,
loads it and removes the directory, so nothing is written into the tree.  TEST AND MEASUREMENT INFRASTRUCTURE only.

    lib = contour_oracle.load()
    steps = lib.gso_trace_contours(img, visited, w, h, records, count, ends)
"""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCE = os.path.join(ROOT, "tools", "contour_oracle.c")
FLAGS = ["-std=c99", "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-pedantic", "-ffp-contract=off"]

_lib = None


def load():
    global _lib
    if _lib is None:
        cc = os.environ.get("CC") or shutil.which("gcc") or shutil.which("cc")
        if cc is None:
            raise RuntimeError("no C compiler found for tools/contour_oracle.c")
        d = tempfile.mkdtemp(prefix="gs_contour_oracle_")
        try:
            so = os.path.join(d, "libcontour_oracle.so")
            r = subprocess.run([cc] + FLAGS + ["-I", os.path.join(ROOT, "include"), "-o", so, SOURCE],
                               capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError("building the contour oracle failed:\n" + r.stdout + r.stderr)
            lib = C.CDLL(so)
        finally:
            shutil.rmtree(d, ignore_errors=True)
        lib.gso_trace_contour.restype = C.c_uint
        lib.gso_trace_contour.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_void_p]
        lib.gso_trace_contours.restype = C.c_ulonglong
        lib.gso_trace_contours.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_void_p, C.c_uint,
                                           C.c_void_p]
        _lib = lib
    return _lib
