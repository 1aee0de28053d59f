"""Build libgrayskull_b200.so and its companions libgrayskull_draw.so, libgrayskull_contour.so, libgrayskull_color.so,
libgrayskull_corners.so, libgrayskull_group.so and libgrayskull_homography.so in-tree with nvcc for sm_90a (H100;
cross-compiles without a GPU), and the gsb_magick CLI on all seven.

    python -m grayskull_b200.build            # incremental
    python -m grayskull_b200.build --force

The .so files are git-ignored and rebuilt by __graft_entry__.build().  cudart is linked statically and the
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
# the companion library of the annotated pictures (include/grayskull_draw.h): its own sources, launch helper and error
# text, not linked against LIB
DRAW_DIR = os.path.join(HERE, "draw")
DRAW_LIB = os.path.join(HERE, "libgrayskull_draw.so")
DRAW_SOURCES = ["draw.cu"]
# the companion library of contour tracing (include/grayskull_contour.h), built the same way
CONTOUR_DIR = os.path.join(HERE, "contour")
CONTOUR_LIB = os.path.join(HERE, "libgrayskull_contour.so")
CONTOUR_SOURCES = ["contour.cu"]
# the companion library of the colour conversions (include/grayskull_color.h), built the same way
COLOR_DIR = os.path.join(HERE, "color")
COLOR_LIB = os.path.join(HERE, "libgrayskull_color.so")
COLOR_SOURCES = ["color.cu"]
# the companion library of the largest-blob pick and batched blob corners (include/grayskull_corners.h), built the same way
CORNERS_DIR = os.path.join(HERE, "corners")
CORNERS_LIB = os.path.join(HERE, "libgrayskull_corners.so")
CORNERS_SOURCES = ["corners.cu"]
# the companion library of detection grouping (include/grayskull_group.h), built the same way
GROUP_DIR = os.path.join(HERE, "group")
GROUP_LIB = os.path.join(HERE, "libgrayskull_group.so")
GROUP_SOURCES = ["group.cu"]
# the companion library of template homographies (include/grayskull_homography.h), built the same way
HOMOGRAPHY_DIR = os.path.join(HERE, "homography")
HOMOGRAPHY_LIB = os.path.join(HERE, "libgrayskull_homography.so")
HOMOGRAPHY_SOURCES = ["homography.cu"]
CASCADE_NPZ = os.path.join(HERE, "data", "frontalface.npz")
CASCADE_H = os.path.join(OBJ, "frontalface_cascade.h")
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
    files += [os.path.join(DRAW_DIR, f) for f in os.listdir(DRAW_DIR)]
    files += [os.path.join(CONTOUR_DIR, f) for f in os.listdir(CONTOUR_DIR)]
    files += [os.path.join(COLOR_DIR, f) for f in os.listdir(COLOR_DIR)]
    files += [os.path.join(CORNERS_DIR, f) for f in os.listdir(CORNERS_DIR)]
    files += [os.path.join(GROUP_DIR, f) for f in os.listdir(GROUP_DIR)]
    files += [os.path.join(HOMOGRAPHY_DIR, f) for f in os.listdir(HOMOGRAPHY_DIR)]
    files += [os.path.join(os.path.dirname(HERE), "include", f)
              for f in ("grayskull.h", "grayskull_b200.h", "grayskull_b200_roi.h", "grayskull_b200_pyramid.h",
                        "grayskull_draw.h", "grayskull_contour.h", "grayskull_color.h", "grayskull_corners.h",
                        "grayskull_group.h", "grayskull_homography.h")]
    files += [os.path.join(HERE, "cli", "gsb_magick.c"), CASCADE_NPZ]
    return max(os.path.getmtime(f) for f in files)


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    newest = _deps_mtime()
    if not force and all(os.path.exists(p) and os.path.getmtime(p) >= newest
                         for p in (LIB, DRAW_LIB, CONTOUR_LIB, COLOR_LIB, CORNERS_LIB, GROUP_LIB, HOMOGRAPHY_LIB)):
        if not os.path.exists(os.path.join(HERE, "gsb_magick")):
            build_cli()
        return LIB
    cc = nvcc()

    def compile_one(src):
        obj = os.path.join(OBJ, os.path.basename(src).replace(".cu", ".o"))
        cmd = [cc] + NVCC_FLAGS + ["-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        with open(obj + ".log", "w") as f:
            f.write(r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s" % (src, r.stdout + r.stderr))
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    draw_srcs = [os.path.join(DRAW_DIR, f) for f in DRAW_SOURCES]   # absolute: os.path.join keeps them as they are
    contour_srcs = [os.path.join(CONTOUR_DIR, f) for f in CONTOUR_SOURCES]
    color_srcs = [os.path.join(COLOR_DIR, f) for f in COLOR_SOURCES]
    corners_srcs = [os.path.join(CORNERS_DIR, f) for f in CORNERS_SOURCES]
    group_srcs = [os.path.join(GROUP_DIR, f) for f in GROUP_SOURCES]
    homography_srcs = [os.path.join(HOMOGRAPHY_DIR, f) for f in HOMOGRAPHY_SOURCES]
    companion_srcs = draw_srcs + contour_srcs + color_srcs + corners_srcs + group_srcs + homography_srcs
    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES) + len(companion_srcs))) as ex:
        all_objs = list(ex.map(compile_one, SOURCES + companion_srcs))
    objs = all_objs[:len(SOURCES)]
    draw_objs = all_objs[len(SOURCES):len(SOURCES) + len(draw_srcs)]
    contour_objs = all_objs[len(SOURCES) + len(draw_srcs):len(SOURCES) + len(draw_srcs) + len(contour_srcs)]
    color_objs = all_objs[len(SOURCES) + len(draw_srcs) + len(contour_srcs):
                          len(SOURCES) + len(draw_srcs) + len(contour_srcs) + len(color_srcs)]
    corners_objs = all_objs[len(SOURCES) + len(draw_srcs) + len(contour_srcs) + len(color_srcs):
                            len(all_objs) - len(group_srcs) - len(homography_srcs)]
    group_objs = all_objs[len(all_objs) - len(group_srcs) - len(homography_srcs):len(all_objs) - len(homography_srcs)]
    homography_objs = all_objs[len(all_objs) - len(homography_srcs):]
    # export only the C ABI (gs_*); C++ symbols stay local
    vs = os.path.join(OBJ, "exports.map")
    with open(vs, "w") as f:
        f.write("{ global: gs_*; local: *; };\n")
    cmd = [cc, "-shared", "-o", LIB] + objs + ["-Xlinker", "--version-script=" + vs]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    # the companions: each its own static cudart, the same export rule
    for lib, lib_objs in ((DRAW_LIB, draw_objs), (CONTOUR_LIB, contour_objs), (COLOR_LIB, color_objs),
                         (CORNERS_LIB, corners_objs), (GROUP_LIB, group_objs), (HOMOGRAPHY_LIB, homography_objs)):
        r = subprocess.run([cc, "-shared", "-o", lib] + lib_objs + ["-Xlinker", "--version-script=" + vs],
                           capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link of %s failed:\n%s" % (os.path.basename(lib), r.stdout + r.stderr))
    build_cli()
    return LIB


def write_cascade_header():
    """build/frontalface_cascade.h: the frontalface cascade of data/frontalface.npz as a C99 `static const struct
    gs_lbp_cascade frontalface`, for the CLI's faces stage.  Floats are written as hex literals, so they are exact."""
    import numpy as np
    z = np.load(CASCADE_NPZ)
    ctype = {np.dtype(np.int8): "int8_t", np.dtype(np.uint16): "uint16_t", np.dtype(np.int32): "int32_t",
             np.dtype(np.float32): "float"}
    lines = ["/* generated by grayskull_b200/build.py from grayskull_b200/data/frontalface.npz -- do not edit */"]
    for k in ("features", "weak_feature_idx", "weak_left_val", "weak_right_val", "weak_subset_offset",
              "weak_num_subsets", "subsets", "stage_weak_start", "stage_nweaks", "stage_threshold"):
        a = z[k]
        vals = [float(v).hex() + "f" for v in a] if a.dtype == np.float32 else [str(int(v)) for v in a]
        lines.append("static const %s frontalface_%s[%d] = {%s};" % (ctype[a.dtype], k, len(a), ", ".join(vals)))
    win = z["window"]
    lines.append("static const struct gs_lbp_cascade frontalface = {%d, %d, %d, %d, %d, frontalface_features, "
                 "frontalface_weak_feature_idx, frontalface_weak_left_val, frontalface_weak_right_val, "
                 "frontalface_weak_subset_offset, frontalface_weak_num_subsets, frontalface_subsets, "
                 "frontalface_stage_weak_start, frontalface_stage_nweaks, frontalface_stage_threshold};"
                 % (int(win[0]), int(win[1]), len(z["features"]) // 4, len(z["weak_feature_idx"]),
                    len(z["stage_threshold"])))
    os.makedirs(OBJ, exist_ok=True)
    with open(CASCADE_H, "w") as f:
        f.write("\n".join(lines) + "\n")


def build_cli():
    """gsb_magick: the C99 batch-pipeline CLI on the device-resident ABI (cli/gsb_magick.c), on all seven libraries"""
    exe = os.path.join(HERE, "gsb_magick")
    write_cascade_header()
    cmd = ["gcc", "-std=c99", "-O2", "-Wall", "-Wextra", "-Werror", "-pedantic", "-D_POSIX_C_SOURCE=200809L",
           "-I", os.path.join(os.path.dirname(HERE), "include"), "-I", OBJ, "-o", exe,
           os.path.join(HERE, "cli", "gsb_magick.c"),
           "-L" + HERE, "-l:" + os.path.basename(DRAW_LIB), "-l:" + os.path.basename(CONTOUR_LIB),
           "-l:" + os.path.basename(COLOR_LIB), "-l:" + os.path.basename(CORNERS_LIB),
           "-l:" + os.path.basename(GROUP_LIB), "-l:" + os.path.basename(HOMOGRAPHY_LIB),
           "-l:" + os.path.basename(LIB), "-Wl,-rpath,$ORIGIN"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("gsb_magick build failed:\n" + r.stdout + r.stderr)
    return exe


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
