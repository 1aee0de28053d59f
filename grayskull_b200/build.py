"""Build libgrayskull_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m grayskull_b200.build            # incremental
    python -m grayskull_b200.build --force

The .so is git-ignored and rebuilt by __graft_entry__.build().  cudart is linked statically and the
driver API (cuTensorMapEncodeTiled) is resolved at run time, so the library loads on machines
without a GPU driver (the CPU-side tests check its exported symbols there).
"""
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libgrayskull_b200.so")
SOURCES = ["runtime.cu", "stencil3.cu", "box.cu", "resample.cu", "integral.cu", "fast_orb.cu", "match.cu", "histogram.cu", "filter.cu", "lbp.cu", "blobs.cu",
           "morph.cu", "api.cu", "roi.cu", "pyramid.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-fmad=false", "-Xcompiler", "-fPIC", "-Xptxas", "-v",
              "-I", os.path.join(os.path.dirname(HERE), "include")]


def nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _deps_mtime():
    files = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    files += [os.path.join(os.path.dirname(HERE), "include", f)
              for f in ("grayskull.h", "grayskull_b200.h", "grayskull_b200_roi.h", "grayskull_b200_pyramid.h")]
    files.append(os.path.join(HERE, "cli", "gsb_magick.c"))
    return max(os.path.getmtime(f) for f in files)


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    newest = _deps_mtime()
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= newest:
        if not os.path.exists(os.path.join(HERE, "gsb_magick")):
            build_cli()
        return LIB
    cc = nvcc()

    def compile_one(src):
        obj = os.path.join(OBJ, src.replace(".cu", ".o"))
        cmd = [cc] + NVCC_FLAGS + ["-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        with open(obj + ".log", "w") as f:
            f.write(r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s" % (src, r.stdout + r.stderr))
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    # export only the C ABI (gs_*); C++ symbols stay local
    vs = os.path.join(OBJ, "exports.map")
    with open(vs, "w") as f:
        f.write("{ global: gs_*; local: *; };\n")
    cmd = [cc, "-shared", "-o", LIB] + objs + ["-Xlinker", "--version-script=" + vs]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    build_cli()
    return LIB


def build_cli():
    """gsb_magick: the C99 batch-pipeline CLI on the device-resident ABI (cli/gsb_magick.c)"""
    exe = os.path.join(HERE, "gsb_magick")
    cmd = ["gcc", "-std=c99", "-O2", "-Wall", "-Wextra", "-Werror", "-pedantic", "-D_POSIX_C_SOURCE=200809L",
           "-I", os.path.join(os.path.dirname(HERE), "include"), "-o", exe, os.path.join(HERE, "cli", "gsb_magick.c"),
           "-L" + HERE, "-l:" + os.path.basename(LIB), "-Wl,-rpath,$ORIGIN"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("gsb_magick build failed:\n" + r.stdout + r.stderr)
    return exe


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
