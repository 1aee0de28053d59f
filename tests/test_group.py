"""Neighbour-counted grouping of LBP detections on the device (include/grayskull_group.h, libgrayskull_group.so).

The rule is the header's, restated here as a numpy model (model_frame).  On the CPU the model is pinned against
hand-built lists whose groups are written out, and the companion is checked as a library.  On the GPU the call is
checked against the model, with poisoned outputs, on the detector's own lists for the lena frame and for c4-shaped
frames, on synthetic clustered lists with chains and exact-boundary pairs, at 65536 records per frame, past 65535
frames and with chunked workspaces; then on the caller's stream, two streams and a CUDA graph; and through gsb_magick's
faces-grouped stage against the same chain built from the library calls.
"""
import ctypes as C
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

import _libs as L
from _gpu import Region, lib, traced, witness, witnessed  # noqa: F401

ROOT = L.ROOT
M32 = 0xFFFFFFFF
FAR = 1 << 40
RECT = L.RECT_DTYPE

# every kernel of libgrayskull_group.so, and which path launches it
KERNELS = {
    "gsb::k_group_init": "group",
    "gsb::k_group_pairs": "group",
    "gsb::k_group_roots": "group",
    "gsb::k_group_filter": "group",
    "gsb::k_group_emit": "group",
    "gsb::k_group_copy": "copy",
}
GROUP_KERNELS = [k for k, v in KERNELS.items() if v == "group"]


# ---- the rule, restated -------------------------------------------------------------------------------------------
def _similar_pairs(r, eps):
    """rule 1 over records r (c, 4) int64 -> (i, j) index arrays of the similar pairs, i != j.  Records are compared
    in x order, offset by offset, until every pair at the offset is farther apart in x than any pair's delta."""
    c = len(r)
    if c < 2:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    order = np.argsort(r[:, 0], kind="stable")
    s = r[order]
    bound = (eps * float(int(r[:, 2].max()) + int(r[:, 3].max()))) * 0.5
    ii, jj = [], []
    for k in range(1, c):
        a, b = s[:-k], s[k:]
        if float((b[:, 0] - a[:, 0]).min()) > bound:
            break
        delta = (eps * (np.minimum(a[:, 2], b[:, 2]) + np.minimum(a[:, 3], b[:, 3])).astype(np.float64)) * 0.5
        ok = np.ones(len(a), bool)
        for d in (a[:, 0] - b[:, 0], a[:, 1] - b[:, 1], (a[:, 0] + a[:, 2]) - (b[:, 0] + b[:, 2]),
                  (a[:, 1] + a[:, 3]) - (b[:, 1] + b[:, 3])):
            ok &= np.abs(d).astype(np.float64) <= delta
        ii.append(order[:-k][ok])
        jj.append(order[k:][ok])
    return (np.concatenate(ii), np.concatenate(jj)) if ii else (np.zeros(0, np.int64), np.zeros(0, np.int64))


def model_frame(recs, k, eps, out_stride):
    """the header's rule for one frame's used records recs (c,) RECT_DTYPE -> (rects (q, 4) uint32, weights (q,))"""
    c = len(recs)
    r = np.stack([recs[f].astype(np.int64) for f in ("x", "y", "w", "h")], -1).reshape(c, 4)
    if k == 0:                                                   # rule 6
        q = min(c, out_stride)
        return r[:q].astype(np.uint32), np.ones(q, np.uint32)
    if c == 0:
        return np.zeros((0, 4), np.uint32), np.zeros(0, np.uint32)
    with np.errstate(over="ignore"):                             # a huge eps: delta and the slack are inf
        return _group_frame(r, k, eps, out_stride)


def _group_frame(r, k, eps, out_stride):
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    c = len(r)
    i, j = _similar_pairs(r, eps)
    _, lab = connected_components(coo_matrix((np.ones(len(i)), (i, j)), shape=(c, c)), directed=False)
    first = np.full(lab.max() + 1, c, np.int64)
    np.minimum.at(first, lab, np.arange(c))
    rank = np.empty_like(first)
    rank[np.argsort(first)] = np.arange(len(first))               # groups in order of their smallest record
    g = rank[lab]
    G = len(first)
    m = np.bincount(g, minlength=G).astype(np.int64)
    box = np.zeros((G, 4), np.int64)
    s = np.float32(1) / m.astype(np.float32)
    for q in range(4):
        S = np.zeros(G, np.int64)
        np.add.at(S, g, r[:, q])
        v = np.rint(S.astype(np.float32) * s).astype(np.float64)    # fp32 product, half to even
        box[:, q] = np.where(v >= 2.0 ** 32, M32, v).astype(np.int64)
    strong = np.flatnonzero(m > k)
    keep = np.zeros(G, bool)
    if len(strong):
        b, mm = box[strong], m[strong]
        dx = np.minimum(np.rint(b[:, 2].astype(np.float64) * eps), float(FAR)).astype(np.int64)   # per j
        dy = np.minimum(np.rint(b[:, 3].astype(np.float64) * eps), float(FAR)).astype(np.int64)
        bi, bj = b[:, None, :], b[None, :, :]
        mi, mj = mm[:, None], mm[None, :]
        inside = ((bi[..., 0] >= bj[..., 0] - dx[None, :]) & (bi[..., 1] >= bj[..., 1] - dy[None, :]) &
                  (bi[..., 0] + bi[..., 2] <= bj[..., 0] + bj[..., 2] + dx[None, :]) &
                  (bi[..., 1] + bi[..., 3] <= bj[..., 1] + bj[..., 3] + dy[None, :]) &
                  ((mj > np.maximum(3, mi)) | (mi < 3)))
        np.fill_diagonal(inside, False)
        keep[strong] = ~inside.any(axis=1)
    out = np.flatnonzero(keep)[:out_stride]
    return box[out].astype(np.uint32), m[out].astype(np.uint32)


def used(rects, counts, f):
    stride = rects.shape[1]
    return stride if counts is None else min(int(counts[f]), stride)


def model_batch(rects, counts, k, eps, out_stride, frames=None):
    """rects (n, stride) RECT_DTYPE, counts (n,) or None -> [(rects, weights)] of each frame in `frames`"""
    fs = range(rects.shape[0]) if frames is None else frames
    return {f: model_frame(rects[f, :used(rects, counts, f)], k, eps, out_stride) for f in fs}


def R(*rows):
    a = np.zeros(len(rows), RECT)
    for i, row in enumerate(rows):
        a[i] = tuple(v & M32 for v in row)
    return a


def grouped(rows, k, eps, out_stride=100):
    got, wt = model_frame(R(*rows), k, eps, out_stride)
    return [tuple(int(v) for v in x) for x in got], [int(v) for v in wt]


# ---- CPU: the model against hand-built lists -------------------------------------------------------------------------
def test_transitive_chain_is_one_group():
    # delta = 0.2 * 200 * 0.5 = 20: A~B and B~C at 15, A and C 30 apart
    rows = [(0, 0, 100, 100), (15, 0, 100, 100), (30, 0, 100, 100)]
    assert grouped(rows, 2, 0.2) == ([(15, 0, 100, 100)], [3])
    assert grouped(rows, 3, 0.2) == ([], [])
    assert grouped([rows[0], rows[2]], 0, 0.2) == ([rows[0], rows[2]], [1, 1])
    # the chain's order does not matter: C, A, B still meet through B
    assert grouped([rows[2], rows[0], rows[1]], 2, 0.2) == ([(15, 0, 100, 100)], [3])


def test_double_delta_boundary():
    # eps 0.7, min w + min h = 180: delta is 62.999999999999996, so 63 apart is not similar and 62 is
    assert (0.7 * 180.0) * 0.5 == 62.999999999999996
    # (groups of 4, so that neither contains the other)
    a, b = (0, 0, 90, 90), (63, 0, 90, 90)
    assert grouped([a] * 4 + [b] * 4, 1, 0.7) == ([(0, 0, 90, 90), (63, 0, 90, 90)], [4, 4])
    b = (62, 0, 90, 90)
    assert grouped([a] * 4 + [b] * 4, 1, 0.7) == ([(31, 0, 90, 90)], [8])
    # the same in y and at the far edges
    assert grouped([a] * 4 + [(0, 63, 90, 90)] * 4, 1, 0.7)[1] == [4, 4]
    assert grouped([a] * 4 + [(0, 62, 90, 90)] * 4, 1, 0.7)[1] == [8]
    assert grouped([a] * 4 + [(0, 0, 153, 90)] * 4, 1, 0.7)[1] == [4, 4]   # x + w differs by 63
    # groups of 2 at 63 apart contain each other (dx = rint(63.0) = 63, m_i < 3), and both go
    assert grouped([a] * 2 + [(63, 0, 90, 90)] * 2, 1, 0.7) == ([], [])


def test_half_even_containment_slack():
    # eps 0.5: w_j = 5 gives dx = rint(2.5) = 2, w_j = 7 gives rint(3.5) = 4.  The small groups are not similar to
    # the big one (delta 1), only contained by it or not.
    big5, big7 = [(10, 10, 5, 5)] * 5, [(10, 10, 7, 7)] * 5
    assert grouped(big5 + [(8, 10, 2, 2)] * 2, 1, 0.5) == ([(10, 10, 5, 5)], [5])
    assert grouped(big5 + [(7, 10, 2, 2)] * 2, 1, 0.5) == ([(10, 10, 5, 5), (7, 10, 2, 2)], [5, 2])
    assert grouped(big7 + [(6, 10, 2, 2)] * 2, 1, 0.5) == ([(10, 10, 7, 7)], [5])
    assert grouped(big7 + [(5, 10, 2, 2)] * 2, 1, 0.5) == ([(10, 10, 7, 7), (5, 10, 2, 2)], [5, 2])


def test_fp32_averages_on_halves():
    # m = 2: sums 1 and 21 give 0.5 -> 0 and 10.5 -> 10; 203 gives 101.5 -> 102 (half to even)
    rows = [(0, 0, 10, 10), (1, 1, 11, 11), (101, 101, 10, 10), (102, 102, 11, 11)]
    assert grouped(rows, 1, 0.2) == ([(0, 0, 10, 10), (102, 102, 10, 10)], [2, 2])
    # m = 4, sum 10: 10 * 0.25 = 2.5 -> 2; m = 3, sum 3: 3 * fp32(1/3) rounds to 1.0 in fp32
    assert grouped([(2, 0, 40, 40), (3, 0, 40, 40), (2, 0, 40, 40), (3, 0, 40, 40)], 1, 0.2)[0] == [(2, 0, 40, 40)]
    assert grouped([(1, 1, 40, 40)] * 3, 1, 0.2)[0] == [(1, 1, 40, 40)]
    # m = 3 and sum 2^24 + 3: (float)S is 16777220, times fp32(1/3) is 5592407.0 (exact: 5592406.33)
    big = (1 << 24) + 3
    rows = [(big // 3, 0, 4000, 4000), (big // 3, 0, 4000, 4000), (big - 2 * (big // 3), 0, 4000, 4000)]
    got = grouped(rows, 1, 0.2)[0][0][0]
    assert got == int(np.rint(np.float32(big) * (np.float32(1) / np.float32(3)))) == 5592407


def test_containment_weight_rule():
    big, small = (0, 0, 100, 100), (10, 10, 20, 20)        # 10 apart, delta 4: never similar
    def case(mj, mi, k=1):
        return grouped([big] * mj + [small] * mi, k, 0.2)
    assert case(5, 4) == ([big], [5])                      # m_j = 5 > max(3, 4)
    assert case(4, 4) == ([big, small], [4, 4])            # m_j = 4 is not above max(3, 4)
    assert case(4, 3) == ([big], [4])                      # 4 > max(3, 3)
    assert case(3, 3) == ([big, small], [3, 3])            # at max(3, m_i), and m_i is not below 3
    assert case(2, 2) == ([big], [2])                      # m_i < 3: any containing group removes it
    assert case(3, 2, k=2) == ([big], [3])                 # m_i = 2 is not above K: it never survives
    # two equal groups of 2 contain each other and both go; of 4 neither beats the other
    a = [(0, 0, 50, 50)] * 2 + [(200, 0, 50, 50)] * 2
    assert grouped(a, 1, 0.2) == ([(0, 0, 50, 50), (200, 0, 50, 50)], [2, 2])
    assert grouped([(0, 0, 50, 50)] * 2 + [(0, 0, 50, 50)], 1, 0.0)[1] == [3]
    # eps 0.5 on 50 x 10: delta 15 and dx 25, so 20 apart is not similar and each contains the other
    twins = [(0, 0, 50, 10)] * 2 + [(20, 0, 50, 10)] * 2
    assert grouped(twins, 1, 0.5) == ([], [])
    twins4 = [(0, 0, 50, 10)] * 4 + [(20, 0, 50, 10)] * 4
    assert grouped(twins4, 1, 0.5) == ([(0, 0, 50, 10), (20, 0, 50, 10)], [4, 4])


def test_k0_copies_and_list_bounds():
    rows = [(5, 5, 10, 10), (5, 5, 10, 10), (300, 0, 20, 20)]
    assert grouped(rows, 0, 0.2) == (rows, [1, 1, 1])
    assert grouped(rows, 0, 0.2, out_stride=2) == (rows[:2], [1, 1])
    rects = np.zeros((3, 4), RECT)
    rects[:] = R(*(rows + [(9, 9, 9, 9)]))
    out = model_batch(rects, np.array([7, 2, 0]), 1, 0.2, 10)
    assert [len(out[f][0]) for f in range(3)] == [1, 1, 0]   # counts above the stride mean the stride
    assert len(model_batch(rects, None, 1, 0.2, 10)[1][0]) == 1
    assert model_batch(np.zeros((2, 0), RECT), None, 1, 0.2, 4)[1][0].shape == (0, 4)   # stride 0
    # out_stride below the survivors: the first ones in group order
    three = [(0, 0, 10, 10)] * 2 + [(100, 0, 10, 10)] * 2 + [(200, 0, 10, 10)] * 2
    assert grouped(three, 1, 0.2, out_stride=2) == ([(0, 0, 10, 10), (100, 0, 10, 10)], [2, 2])


def test_coordinates_near_2_32():
    top = M32
    # 0 and 2^32 - 1 are 2^32 - 1 apart, not 1 as a 32-bit difference would say
    assert grouped([(0, 0, 10, 10), (top, 0, 10, 10)], 0, 0.2)[0] == [(0, 0, 10, 10), (top, 0, 10, 10)]
    assert grouped([(0, 0, 10, 10), (0, 0, 10, 10), (top, 0, 10, 10), (top, 0, 10, 10)], 1, 0.2)[1] == [2, 2]
    # x + w past 2^32 compared exactly; the average 2^32 - 6.5 rounds to 2^32 in fp32 and is clamped
    got, wt = grouped([(top - 5, 0, 10, 10), (top - 6, 0, 10, 10)], 1, 0.2)
    assert got == [(top, 0, 10, 10)] and wt == [2]
    # widths near 2^32: delta is huge, every difference fits it, and the huge eps saturates the slack
    w = top - 10
    assert grouped([(0, 0, w, w), (1 << 30, 1 << 30, w, w)], 1, 0.5)[1] == [2]
    assert grouped([(0, 0, w, w), (0, 0, w, w), (3, 3, 2, 2), (3, 3, 2, 2)], 1, 1e300)[1] == [4]   # delta is inf


# ---- CPU: the library ------------------------------------------------------------------------------------------------
HEADER = os.path.join(ROOT, "include", "grayskull_group.h")


def _declarations():
    txt = open(HEADER).read()
    txt = txt[txt.rindex('extern "C" {'):]
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return {m.group(2): (m.group(1).strip().split("\n")[-1].strip(), [a.strip() for a in m.group(3).split(",") if a.strip() != "void"])
            for m in re.finditer(r"([\w\s\*]+?)\b(gs_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", txt)}


def test_companion_exports_exactly_its_header():
    from grayskull_b200 import build, group
    build.build()
    declared = sorted(_declarations())
    assert len(declared) == 3 and sorted(group.SIGNATURES) == declared
    nm = subprocess.run(["nm", "-D", "--defined-only", group.LIB_PATH], capture_output=True, text=True,
                        check=True).stdout
    assert sorted(ln.split()[-1] for ln in nm.splitlines() if " T " in ln) == declared
    needed = subprocess.run(["readelf", "-d", group.LIB_PATH], capture_output=True, text=True, check=True).stdout
    assert "libgrayskull_b200" not in needed
    assert group.lib().gs_b200_group_last_error() == b"no error"


def test_main_library_exports_nothing_of_it():
    from grayskull_b200 import _lib
    main = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True,
                          check=True).stdout
    assert "group" not in main
    assert not any("k_group" in k for k in L.sass_functions())


def test_ctypes_table_matches_the_header():
    from grayskull_b200 import group
    want_of = {"double": C.c_double, "size_t": C.c_size_t}
    for name, (ret, args) in _declarations().items():
        res, argtypes = group.SIGNATURES[name]
        assert res is {"int": C.c_int, "size_t": C.c_size_t}.get(ret, C.c_char_p), name
        assert len(argtypes) == len(args), name
        for a, t in zip(args, argtypes):
            kind = a.split()[0] if a.split()[0] != "const" else a.split()[1]
            want = C.c_void_p if "*" in a or kind == "gs_b200_stream" else want_of.get(kind, C.c_uint)
            assert t is want, (name, a)


def test_header_compiles_as_c99(tmp_path):
    for first in ("", '#include "grayskull_b200.h"\n', '#include "grayskull_draw.h"\n'):
        src = tmp_path / "t.c"
        src.write_text(first + '#include "grayskull_group.h"\n'
                       'int main(void) { struct gs_rect r = {0, 0, 1, 1};\n'
                       '  return gs_b200_group_last_error() == 0 && r.w == 2 && gs_b200_group_rects_work_bytes(1, 1); }\n')
        r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-fsyntax-only",
                            "-I", os.path.join(ROOT, "include"), str(src)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    assert not re.match(r"grayskull_b200.*\.h$", "grayskull_group.h")


def test_every_companion_kernel_is_sm90a_and_has_a_row():
    from grayskull_b200 import group
    tool = L.cuda_tool("cuobjdump")
    if tool is None:
        pytest.skip("cuobjdump not found")
    listing = subprocess.run([tool, "-sass", group.LIB_PATH], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for cubin in re.split(r"^\s*(?=code for sm_\w+\s*$)", listing, flags=re.M)[1:]:
        arch, *parts = re.split(r"^\s*Function : (\S+)\s*$", cubin, flags=re.M)
        for name in L.demangle(parts[0::2]):
            funcs[L.kernel_id(name)] = arch.strip().splitlines()[0]
    assert set(funcs) == set(KERNELS)
    assert all(arch == "code for sm_90a" for arch in funcs.values())


def test_launches_go_through_the_companions_helper():
    d = os.path.join(ROOT, "grayskull_b200", "group")
    text = {f: open(os.path.join(d, f)).read() for f in sorted(os.listdir(d))}
    sites = [(f, m.start()) for f, t in text.items() for m in re.finditer(r"<<<", t)]
    assert len(sites) == 1
    f, at = sites[0]
    assert text[f].rindex("static int launch(", 0, at) < at < text[f].index("cudaGetLastError")
    assert text[f].count("cudaGetLastError") == 1
    from grayskull_b200 import build
    assert not set(build.GROUP_SOURCES) & set(build.SOURCES)


def test_companion_object_makes_no_blocking_runtime_call():
    from grayskull_b200 import build
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm not found")
    blocking = re.compile(r"^(cudaMemcpy|cudaMemcpyToSymbol|cudaMemset|cudaMemcpy2D|cudaDeviceSynchronize|"
                          r"cudaStreamSynchronize|cudaEventSynchronize|cudaMalloc\w*|cudaFree\w*|cudaStreamCreate\w*|"
                          r"cudaStreamDestroy|cudaMemcpyAsync|cudaMemsetAsync)$")
    for s in build.GROUP_SOURCES:
        o = os.path.join(build.OBJ, s.replace(".cu", ".o"))
        syms = [ln.split()[-1] for ln in subprocess.run([nm, "-u", o], capture_output=True, text=True,
                                                         check=True).stdout.splitlines()]
        assert "cudaGetLastError" in syms
        assert not [x for x in syms if blocking.match(x)], syms


def test_work_bytes():
    from grayskull_b200 import group
    one = group.work_bytes(4096, 1)
    assert one == 64 * 4096 + 4 + 16 and group.work_bytes(4096, 3) == 3 * (64 * 4096 + 4) + 16
    assert group.work_bytes(0, 5) == 5 * 4 + 16
    assert group.work_bytes(M32, M32) == 2 ** 64 - 1          # about 2^70 does not fit: size_t saturates
    assert group.work_bytes(65536, 64) == 64 * (64 * 65536 + 4) + 16


def _run_py(expr):
    code = ("import ctypes as C, sys; sys.path.insert(0, %r); from grayskull_b200 import group; "
            "L = group.lib(); P = C.c_void_p(4096); rc = %s; print('rc', rc); print(L.gs_b200_group_last_error())")
    return subprocess.run([sys.executable, "-c", code % (ROOT, expr)], capture_output=True, text=True, timeout=120)


def test_empty_batch_missing_pointer_and_bad_arguments_without_a_gpu():
    call = "L.gs_b200_group_rects_batch(P, P, 4, %d, 3, %s, %s, P, %s, 4, %s, %s, None)"
    ok = _run_py(call % (0, "0.2", "None", "None", "None", "0"))
    assert ok.returncode == 0 and "rc 0" in ok.stdout, (ok.stdout, ok.stderr)
    for missing in ((2, "0.2", "None", "P", "P", "1 << 20"), (2, "0.2", "P", "None", "P", "1 << 20"),
                    (2, "0.2", "P", "P", "None", "1 << 20")):
        bad = _run_py(call % missing)
        assert bad.returncode != 0 and "Assertion failed: " in bad.stderr, (missing, bad.stderr)
    # refused before anything is enqueued
    for eps in ("-0.5", "float('nan')", "float('inf')", "-float('inf')"):
        r = _run_py(call % (2, eps, "P", "P", "P", "1 << 20"))
        assert r.returncode == 0 and "rc 1" in r.stdout and "eps" in r.stdout, (eps, r.stdout, r.stderr)
    need = 64 * 4 + 4    # one frame of stride 4; P is 16-byte aligned
    for wb, k in ((need - 1, 3), (0, 3), (need - 1, 0)):
        r = _run_py((call % (2, "0.2", "P", "P", "P", str(wb))).replace(", 3, 0.2", ", %d, 0.2" % k))
        assert r.returncode == 0 and "rc 1" in r.stdout and "work_bytes" in r.stdout, (wb, r.stdout, r.stderr)
    # an unaligned work pointer loses its first bytes to the 16-byte boundary
    r = _run_py(call % (2, "0.2", "P", "P", "C.c_void_p(4100)", str(need)))
    assert "rc 1" in r.stdout and "work_bytes" in r.stdout, r.stdout


# ---- GPU -------------------------------------------------------------------------------------------------------------
def glib():
    from grayskull_b200 import group
    return group.lib()


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()


def _s():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class Case:
    """one call: rects (n, stride) RECT_DTYPE and counts (None: all), into poisoned out / weights / out_counts"""

    def __init__(self, rects, counts, k, eps, out_stride=None):
        self.rects, self.counts, self.k, self.eps = rects, counts, k, eps
        self.n, self.stride = rects.shape
        self.out_stride = self.stride if out_stride is None else out_stride

    def buffers(self, off=0, work_frames=None, weights=True):
        import torch
        n, os_ = self.n, self.out_stride
        self.rec = Region(self.rects.nbytes, 4 * off, self.rects, seed=1)
        self.out = Region(16 * n * os_, 4 * off, seed=2)
        self.wt = Region(4 * n * os_, 4 * off, seed=3) if weights else None
        self.oc = Region(4 * n, 4 * off, seed=4)
        self.count_t = None if self.counts is None else _dev(np.asarray(self.counts, np.uint32))
        frames = n if work_frames is None else work_frames
        self.wb = glib().gs_b200_group_rects_work_bytes(self.stride, frames)
        self.work = torch.empty(self.wb + 64, dtype=torch.uint8, device="cuda")
        self.work_ptr = self.work.data_ptr() + off
        return self

    def call(self, s=None, wb=None):
        cp = None if self.count_t is None else self.count_t.data_ptr()
        return glib().gs_b200_group_rects_batch(self.rec.ptr, cp, self.stride, self.n, self.k, self.eps, self.out.ptr,
                                                self.wt.ptr if self.wt else None, self.oc.ptr, self.out_stride,
                                                self.work_ptr, self.wb if wb is None else wb,
                                                _s() if s is None else s)

    def check(self, what, frames=None):
        self.rec.read(what)
        got = self.out.read(what).view(np.uint32).reshape(self.n, self.out_stride, 4)
        before = self.out.before().view(np.uint32).reshape(self.n, self.out_stride, 4)
        gw = self.wt.read(what).view(np.uint32).reshape(self.n, self.out_stride) if self.wt else None
        wbefore = self.wt.before().view(np.uint32).reshape(self.n, self.out_stride) if self.wt else None
        gc = self.oc.read(what).view(np.uint32)
        want = model_batch(self.rects, self.counts, self.k, self.eps, self.out_stride, frames)
        for f, (wr, ww) in want.items():
            q = len(wr)
            assert gc[f] == q, "%s: frame %d: %d groups, want %d" % (what, f, gc[f], q)
            assert np.array_equal(got[f, :q], wr), "%s: frame %d: %s, want %s" % (what, f, got[f, :q][:5], wr[:5])
            assert np.array_equal(got[f, q:], before[f, q:]), "%s: frame %d wrote past its count" % (what, f)
            if gw is not None:
                assert np.array_equal(gw[f, :q], ww) and np.array_equal(gw[f, q:], wbefore[f, q:]), (what, f)
        return want


def clustered(n, stride, seed, span=4000, chains=True, shuffle=True):
    """records around cluster centres (faces of 24..200 px, jittered as the detector's windows are), chains that only
    transitivity joins, exact-boundary pairs at eps 0.7 and duplicates; per frame a random count"""
    rng = np.random.default_rng(seed)
    out = np.zeros((n, stride), RECT)
    for f in range(n):
        rows = []
        while len(rows) < stride:
            kind = rng.integers(0, 6)
            x, y, s = int(rng.integers(0, span)), int(rng.integers(0, span)), int(rng.integers(24, 200))
            if kind == 0 and chains:     # a chain of growing offsets
                for q in range(int(rng.integers(3, 8))):
                    rows.append((x + q * max(1, s // 10), y, s, s))
            elif kind == 1:              # 63 vs 62 apart at min w + min h = 180
                rows += [(x, y, 90, 90), (x + int(rng.integers(62, 64)), y, 90, 90)]
            elif kind == 2:              # a big group and a small one inside it
                rows += [(x, y, 100, 100)] * int(rng.integers(1, 7)) + [(x + 10, y + 10, 20, 20)] * int(rng.integers(1, 6))
            else:                        # a face: jittered windows of nearby sizes
                for _ in range(int(rng.integers(1, 30))):
                    d = int(rng.integers(-s // 12 - 1, s // 12 + 2))
                    rows.append((x + int(rng.integers(-s // 10 - 1, s // 10 + 2)),
                                 y + int(rng.integers(-s // 10 - 1, s // 10 + 2)), s + d, s + d))
        rows = rows[:stride]
        if shuffle:
            rng.shuffle(rows)
        out[f] = R(*rows)
    return out


def detector_lists(frames, max_rects, sf, mn, mx, step):
    import torch
    from grayskull_b200 import api
    import grayskull_b200 as g
    cas = g.load_cascade()
    src = torch.from_numpy(np.ascontiguousarray(frames)).cuda() if isinstance(frames, np.ndarray) else frames
    ii = api.integral_batch(src)
    rects, counts = api.lbp_detect_batch(cas, ii, max_rects, sf, mn, mx, step)
    r = rects.cpu().numpy().view(np.uint32).reshape(len(counts), max_rects, 4)
    return np.ascontiguousarray(r).view(RECT).reshape(len(counts), max_rects), counts.cpu().numpy().view(np.uint32)


def _lena():
    return np.ascontiguousarray(np.load(os.path.join(ROOT, "tests", "golden", "lena_golden.npz"))["lena"])


@pytest.fixture(scope="module")
def c4_lists(lib):
    """the detector's lists at the c4 parameters for two 3840x2160 frames of blurred noise, and for lena at the
    faces verb's parameters with step 1"""
    import torch
    from grayskull_b200 import api
    gen = torch.Generator(device="cuda").manual_seed(4)
    noise = torch.randint(0, 256, (2, 2160, 3840), dtype=torch.uint8, device="cuda", generator=gen)
    c4 = detector_lists(api.blur_batch(noise, 3), 65536, 1.1, 1.0, 4.0, 2)
    lena = detector_lists(_lena()[None], 4096, 1.2, 1.0, 4.0, 1)
    return c4, lena


@pytest.mark.gpu
@pytest.mark.parametrize("eps", [0.2, 0.5, 0.7])
def test_detector_lists_match_the_model(lib, witness, c4_lists, eps):
    (c4, c4n), (lena, lenan) = c4_lists
    assert c4n.max() > 200 and lenan[0] > 10, (c4n, lenan)
    cut = int(c4n.max())                                       # the used part of the 65536-record lists
    for k in (0, 1, 3, 5):
        for name, rects, counts in (("c4", c4[:, :cut + 3], c4n), ("lena", lena, lenan)):
            c = Case(rects, counts, k, eps)
            what = "%s K=%d eps=%g" % (name, k, eps)

            def run():
                c.buffers()
                rc, seen = traced(lambda: c.call())
                assert rc == 0, glib().gs_b200_group_last_error()
                want = c.check(what)
                if k:
                    assert any(len(v[0]) for v in want.values()) or name == "c4"
                return seen

            witnessed(witness, run, GROUP_KERNELS if k else ["gsb::k_group_copy"], what)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["aligned", "offset", "counts-null", "no-weights", "short-out"])
def test_clustered_lists_match_the_model(lib, layout):
    rects = clustered(5, 700, seed=11)
    counts = None if layout == "counts-null" else np.array([700, 0, 350, 9999, 1], np.uint32)
    for k, eps in ((1, 0.2), (3, 0.7), (2, 0.5), (5, 0.0), (1, 3.0)):
        c = Case(rects, counts, k, eps, out_stride=7 if layout == "short-out" else None)
        c.buffers(off=3 if layout == "offset" else 0, weights=layout != "no-weights")
        assert c.call() == 0, glib().gs_b200_group_last_error()
        c.check("%s K=%d eps=%g" % (layout, k, eps))


@pytest.mark.gpu
def test_hand_built_lists_on_the_device(lib):
    """the CPU cases' lists, one frame each, through the device"""
    lists = [
        [(0, 0, 100, 100), (15, 0, 100, 100), (30, 0, 100, 100)],
        [(0, 0, 90, 90)] * 2 + [(63, 0, 90, 90)] * 2 + [(300, 0, 90, 90)] * 2 + [(362, 0, 90, 90)] * 2,
        [(10, 10, 5, 5)] * 5 + [(8, 10, 2, 2)] * 2 + [(40, 10, 7, 7)] * 5 + [(35, 10, 2, 2)] * 2,
        [(0, 0, 10, 10), (1, 1, 11, 11), (101, 101, 10, 10), (102, 102, 11, 11)],
        [(0, 0, 100, 100)] * 4 + [(10, 10, 20, 20)] * 3 + [(500, 0, 100, 100)] * 3 + [(510, 10, 20, 20)] * 3,
        [(0, 0, 10, 10), (M32, 0, 10, 10), (M32 - 5, 0, 10, 10), (M32 - 6, 0, 10, 10), (0, 0, 10, 10)],
    ]
    stride = max(len(x) for x in lists)
    rects = np.zeros((len(lists), stride), RECT)
    counts = np.array([len(x) for x in lists], np.uint32)
    for f, x in enumerate(lists):
        rects[f, :len(x)] = R(*x)
    for k, eps in ((1, 0.2), (2, 0.2), (1, 0.7), (1, 0.5), (0, 0.2), (2, 0.0)):
        c = Case(rects, counts, k, eps).buffers()
        assert c.call() == 0
        c.check("hand-built K=%d eps=%g" % (k, eps))


@pytest.mark.gpu
def test_65536_records_per_frame(lib, witness):
    rects = clustered(2, 65536, seed=12, span=60000)
    c = Case(rects, None, 3, 0.2)

    def run():
        c.buffers()
        rc, seen = traced(lambda: c.call())
        assert rc == 0
        c.check("65536 records")
        return seen

    witnessed(witness, run, GROUP_KERNELS, "65536 records")
    # one frame's state in `work`: two chunks, the same bytes
    c.buffers(work_frames=1)
    assert c.call() == 0
    c.check("65536 records, chunked")


@pytest.mark.gpu
def test_work_sizes(lib):
    rects = clustered(7, 300, seed=13)
    counts = np.random.default_rng(13).integers(0, 400, 7).astype(np.uint32)
    for frames in (7, 1, 3, 2):
        c = Case(rects, counts, 2, 0.2).buffers(off=1, work_frames=frames)
        assert c.call() == 0
        c.check("work for %d frames" % frames)
    c = Case(rects, counts, 2, 0.2).buffers(work_frames=1)      # work is 16-byte aligned: no bytes lost to padding
    one = c.wb - 16
    assert c.call(wb=one - 1) == 1                              # cudaErrorInvalidValue, nothing written
    assert "work_bytes" in glib().gs_b200_group_last_error().decode()
    assert np.array_equal(c.out.read("refused"), c.out.before())
    assert np.array_equal(c.oc.read("refused"), c.oc.before())
    assert c.call(wb=one) == 0
    c.check("work for exactly one frame")


@pytest.mark.gpu
def test_batches_above_the_grid_limit(lib):
    n, stride = 65536 + 3, 6
    rng = np.random.default_rng(14)
    base = rng.integers(0, 300, (n, 1, 2))
    jit = rng.integers(0, 4, (n, stride, 2))
    rects = np.zeros((n, stride), RECT)
    rects["x"], rects["y"] = base[..., 0] + jit[..., 0], base[..., 1] + jit[..., 1]
    rects["w"] = rects["h"] = 30 + rng.integers(0, 3, (n, stride))
    rects["x"][:, 4:] += 200                                # a second group in most frames
    counts = rng.integers(0, 8, n).astype(np.uint32)
    frames = list(range(100)) + list(range(n - 100, n))
    for k in (0, 1):
        c = Case(rects, counts, k, 0.2).buffers()
        assert c.call() == 0
        c.check("65539 frames K=%d" % k, frames=frames)
    c = Case(rects, counts, 1, 0.2).buffers(work_frames=40000)
    assert c.call() == 0
    c.check("65539 frames in chunks", frames=frames)


@pytest.mark.gpu
def test_empty_lists_write_only_counts(lib):
    rects = clustered(3, 20, seed=15)
    for stride_zero in (True, False):
        c = Case(np.zeros((3, 0), RECT) if stride_zero else rects, None, 2, 0.2, out_stride=0 if not stride_zero else 5)
        c.buffers()
        assert c.call() == 0
        assert (c.oc.read("empty").view(np.uint32) == 0).all()
        assert np.array_equal(c.out.read("empty"), c.out.before()) and np.array_equal(c.wt.read("empty"), c.wt.before())


# ---- GPU: streams ----------------------------------------------------------------------------------------------------
def _sleep(s, cycles):
    import torch
    with torch.cuda.stream(s):
        torch.cuda._sleep(int(cycles))


@pytest.mark.gpu
def test_ordered_behind_a_sleeping_stream_without_a_host_wait(lib):
    import torch
    rects = clustered(3, 500, seed=21)
    c = Case(rects, np.array([500, 300, 77], np.uint32), 2, 0.2).buffers()
    s, u = torch.cuda.Stream(), torch.cuda.Stream()
    real = _dev(rects)
    out0 = torch.from_numpy(c.out.before()).cuda()          # host copies wait for their stream: all made up front
    with torch.cuda.stream(s):
        c.rec.t[c.rec.off:c.rec.off + c.rec.nbytes].zero_()
    assert c.call(C.c_void_p(s.cuda_stream)) == 0           # warm, on zeros
    torch.cuda.synchronize()
    _sleep(u, 400_000_000)
    _sleep(s, 200_000_000)
    with torch.cuda.stream(s):
        c.rec.t[c.rec.off:c.rec.off + c.rec.nbytes].copy_(real)
        c.out.t[c.out.off:c.out.off + c.out.nbytes].copy_(out0)
    assert c.call(C.c_void_p(s.cuda_stream)) == 0
    s_done, u_done = s.query(), u.query()
    torch.cuda.synchronize()
    assert not s_done and not u_done, "the call waited for its stream or for the device"
    c.check("behind a sleep")


@pytest.mark.gpu
def test_two_streams_at_once(lib):
    import torch
    s0, s1 = torch.cuda.Stream(), torch.cuda.Stream()
    cases = [(Case(clustered(3, 400, seed=seed), None, 1 + seed % 3, 0.2).buffers(), st)
             for seed, st in ((22, s0), (23, s1), (24, s0), (25, s1))]
    _sleep(s1, 50_000_000)
    for c, st in cases:
        assert c.call(C.c_void_p(st.cuda_stream)) == 0
    torch.cuda.synchronize()
    for c, _ in cases:
        c.check("two streams")


@pytest.mark.gpu
def test_graph_capture_and_replay_on_new_inputs(lib):
    import torch
    n, stride = 3, 600
    c = Case(clustered(n, stride, seed=26), np.array([600, 20, 300], np.uint32), 3, 0.2).buffers(work_frames=2)
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        assert c.call(C.c_void_p(s.cuda_stream)) == 0
    for seed in (31, 32):
        fresh = clustered(n, stride, seed=seed)
        counts = np.random.default_rng(seed).integers(0, stride + 5, n).astype(np.uint32)
        with torch.cuda.stream(s):
            c.rec.t[c.rec.off:c.rec.off + c.rec.nbytes].copy_(_dev(fresh))
            c.count_t.copy_(_dev(counts))
            c.out.t.copy_(torch.from_numpy(c.out.host).cuda())   # poisoned again: slots past the count stay so
            c.wt.t.copy_(torch.from_numpy(c.wt.host).cuda())
            g.replay()
        s.synchronize()
        c.rects, c.counts = fresh, counts
        c.rec.host[c.rec.off:c.rec.off + c.rec.nbytes] = np.frombuffer(fresh.tobytes(), np.uint8)
        c.check("replay %d" % seed)


# ---- GPU: the chain and the CLI --------------------------------------------------------------------------------------
def _pgm(path, a):
    h, w = a.shape
    path.write_bytes(b"P5\n%d %d\n255\n" % (w, h) + a.tobytes())
    return str(path)


def _read_pgm(path):
    data = open(path, "rb").read()
    m = re.match(rb"P5\s+(\d+)\s+(\d+)\s+255\s", data)
    w, h = int(m.group(1)), int(m.group(2))
    return np.frombuffer(data[m.end():], np.uint8).reshape(h, w)


@pytest.mark.gpu
@pytest.mark.parametrize("step,k", [(1, 3), (2, 1), (1, 0)])
def test_gsb_magick_faces_grouped_matches_the_library_chain(lib, tmp_path, step, k):
    """faces-grouped:S:K writes, byte for byte, the picture of detect -> group -> draw_rects, and prints the counts"""
    import torch
    import grayskull_b200 as g
    from grayskull_b200 import api, build, draw, group
    exe = os.path.join(os.path.dirname(build.LIB), "gsb_magick")
    lena = _lena()
    frames = [lena, np.ascontiguousarray(lena[:, ::-1]), L.natural_like(lena.shape[1], lena.shape[0], 5)]
    ins = [_pgm(tmp_path / ("in%d.pgm" % f), a) for f, a in enumerate(frames)]
    r = subprocess.run([exe, "faces-grouped:%d:%d" % (step, k), str(tmp_path / "o_")] + ins, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    src = torch.from_numpy(np.stack(frames)).cuda()
    ii = api.integral_batch(src)
    rects, counts = api.lbp_detect_batch(g.load_cascade(), ii, 4096, 1.2, 1.0, 4.0, step)
    groups, weights, gcounts = group.group_rects_batch(rects, counts, k, 0.2)
    pic = draw.draw_rects_batch(src, groups, gcounts).cpu().numpy()
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("frame ")]
    cn, gn = counts.cpu().numpy(), gcounts.cpu().numpy()
    assert gn[0] > 0 and cn[0] > gn[0] or k == 0
    for f in range(len(frames)):
        assert lines[f] == "frame %d: %d windows, %d faces" % (f, cn[f], gn[f]), lines
        assert np.array_equal(_read_pgm(tmp_path / ("o_%04d.pgm" % f)), pic[f]), f
    # and the library chain's groups are the model's
    rn = np.ascontiguousarray(rects.cpu().numpy().view(np.uint32)).view(RECT).reshape(len(frames), 4096)
    for f, (wr, ww) in model_batch(rn, cn.view(np.uint32), k, 0.2, 4096).items():
        q = len(wr)
        assert gn[f] == q and np.array_equal(groups[f, :q].cpu().numpy().view(np.uint32), wr)
        assert np.array_equal(weights[f, :q].cpu().numpy().view(np.uint32), ww)
