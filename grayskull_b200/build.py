"""Build libgrayskull_b200.so and its companions libgrayskull_b200_roi.so and libgrayskull_b200_pyramid.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

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
# the companion library of region-of-interest calls (include/grayskull_b200_roi.h), linked against LIB
ROI_DIR = os.path.join(HERE, "roi")
ROI_LIB = os.path.join(HERE, "libgrayskull_b200_roi.so")
ROI_SOURCES = ["roi.cu"]
# the companion library of pyramid ORB (include/grayskull_b200_pyramid.h), linked against LIB
PYR_DIR = os.path.join(HERE, "pyramid")
PYR_LIB = os.path.join(HERE, "libgrayskull_b200_pyramid.so")
PYR_SOURCES = ["pyramid.cu"]
SOURCES = ["runtime.cu", "stencil3.cu", "box.cu", "resample.cu", "integral.cu", "fast_orb.cu", "match.cu", "histogram.cu", "filter.cu", "lbp.cu", "blobs.cu",
           "morph.cu", "api.cu"]
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
    files += [os.path.join(ROI_DIR, f) for f in os.listdir(ROI_DIR)]
    files += [os.path.join(PYR_DIR, f) for f in os.listdir(PYR_DIR)]
    files += [os.path.join(os.path.dirname(HERE), "include", f)
              for f in ("grayskull.h", "grayskull_b200.h", "grayskull_b200_roi.h", "grayskull_b200_pyramid.h")]
    files.append(os.path.join(HERE, "cli", "gsb_magick.c"))
    return max(os.path.getmtime(f) for f in files)


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    newest = _deps_mtime()
    if not force and all(os.path.exists(p) and os.path.getmtime(p) >= newest for p in (LIB, ROI_LIB, PYR_LIB)):
        if not os.path.exists(os.path.join(HERE, "gsb_magick")):
            build_cli()
        return LIB
    cc = nvcc()

    def compile_one(src):
        obj = os.path.join(OBJ, os.path.basename(src).replace(".cu", ".o"))
        cmd = [cc] + NVCC_FLAGS + ["-c", src if os.path.isabs(src) else os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        with open(obj + ".log", "w") as f:
            f.write(r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s" % (src, r.stdout + r.stderr))
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    roi_srcs = [os.path.join(ROI_DIR, f) for f in ROI_SOURCES]
    pyr_srcs = [os.path.join(PYR_DIR, f) for f in PYR_SOURCES]
    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES) + len(roi_srcs) + len(pyr_srcs))) as ex:
        all_objs = list(ex.map(compile_one, SOURCES + roi_srcs + pyr_srcs))
    objs, roi_objs = all_objs[:len(SOURCES)], all_objs[len(SOURCES):len(SOURCES) + len(roi_srcs)]
    pyr_objs = all_objs[len(SOURCES) + len(roi_srcs):]
    # export only the C ABI (gs_* and the internal gsb_* hooks); C++ symbols stay local
    vs = os.path.join(OBJ, "exports.map")
    with open(vs, "w") as f:
        f.write("{ global: gs_*; gsb_*; local: *; };\n")
    cmd = [cc, "-shared", "-o", LIB] + objs + ["-Xlinker", "--version-script=" + vs]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    # the companions: each its own static cudart, the main library's hooks resolved through DT_NEEDED + $ORIGIN
    for lib, lib_objs in ((ROI_LIB, roi_objs), (PYR_LIB, pyr_objs)):
        cmd = [cc, "-shared", "-o", lib] + lib_objs + ["-Xlinker", "--version-script=" + vs, "-L" + HERE,
                                                       "-l:" + os.path.basename(LIB), "-Xlinker", "-rpath,$ORIGIN"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link of %s failed:\n%s" % (os.path.basename(lib), r.stdout + r.stderr))
    build_cli()
    return LIB


def build_cli():
    """gsb_magick: the C99 batch-pipeline CLI on the device-resident ABI (cli/gsb_magick.c)"""
    exe = os.path.join(HERE, "gsb_magick")
    cmd = ["gcc", "-std=c99", "-O2", "-Wall", "-Wextra", "-Werror", "-pedantic", "-D_POSIX_C_SOURCE=200809L",
           "-I", os.path.join(os.path.dirname(HERE), "include"), "-o", exe, os.path.join(HERE, "cli", "gsb_magick.c"),
           "-L" + HERE, "-l:" + os.path.basename(ROI_LIB), "-l:" + os.path.basename(PYR_LIB), "-l:" + os.path.basename(LIB), "-Wl,-rpath,$ORIGIN"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("gsb_magick build failed:\n" + r.stdout + r.stderr)
    return exe


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
