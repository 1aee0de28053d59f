"""Every batch entry point runs on the caller's stream and only there: ordered behind work already queued on it, with
no hidden wait on the host, correct on two streams at once, on cudaStreamPerThread from two host threads, and inside a
captured CUDA graph.

CASES is the coverage record: one row per entry point of include/grayskull_b200*.h that takes a gs_b200_stream, with
a tiled and a generic geometry where the host code has both.  A compute row takes its buffers, its call, its expected
outputs and its inputs for a seed from tests/_calls.py; the transfer rows describe themselves here.  Seed 1 is the
real input; seed 2 is the "poison", the same op's valid inputs for another seed, so a read that is not ordered behind
the copy of the real inputs computes wrong values but never addresses out of bounds.

  * CPU: CASES names every such entry point the header declares; the census of blocking or legacy-stream runtime
    calls each object of the library imports, each with its reason.
  * GPU A: on a non-blocking stream behind a sleep, the real inputs are copied over the poison, the outputs are
    overwritten, the call is made and its outputs cloned.  Right after the call returns neither that stream nor a
    second sleeping stream may have finished, and the clones must be bit-exact.
  * GPU B: every row on two streams at once, at two geometries.
  * GPU C: cudaStreamPerThread from two host threads, ops whose scratch holds values.
  * GPU D: every row captured into a CUDA graph and replayed with new inputs and changed host parameters; a capture
    that would grow the workspace is refused.
"""
import ctypes as C
import glob
import os
import re
import shutil
import subprocess
import threading
import time

import numpy as np
import pytest

import _calls as calls
import _libs as L
from _gpu import O, frames, lib  # noqa: F401

ROOT = L.ROOT
POISON = calls.POISON                # what the outputs hold before a call
SLEEP_MIN_CYCLES = 40_000_000        # ~20 ms at 1.98 GHz
SLEEP_MAX_CYCLES = 400_000_000       # ~200 ms: the bound on any one sleep
CAPTURE_UNSUPPORTED = 900            # cudaErrorStreamCaptureUnsupported


def _second(p):
    """the second geometry of a row (part B): the row's own, else one more frame and two more rows"""
    if "second" in p:
        return p["second"]
    q = dict(p)
    if "n" in q:
        q["n"] += 1
    if "h" in q:
        q["h"] += 2
    return q


def case(cid, fn, **p):
    """a row: id, the entry point it calls, its parameters"""
    return cid, fn, p


K7X5 = (np.random.default_rng(75).integers(-8, 9, (5, 7)).astype(np.int8).view(np.uint8), 9)
CASES = [
    case("blur-tma", "gs_b200_blur_batch", w=272, h=70, n=3, r=3),
    case("blur-ragged", "gs_b200_blur_batch", w=100, h=70, n=3, r=9),
    case("adaptive-tma", "gs_b200_adaptive_threshold_batch", w=272, h=70, n=3, r=3, c=2),
    case("adaptive-ragged", "gs_b200_adaptive_threshold_batch", w=100, h=70, n=3, r=5, c=-1),
    case("sobel-tma", "gs_b200_sobel_batch", w=272, h=41, n=3),
    case("sobel-ragged", "gs_b200_sobel_batch", w=100, h=37, n=3),
    case("blur_sobel-tma", "gs_b200_blur_sobel_batch", w=272, h=70, n=3, r=3),
    case("blur_sobel-staged", "gs_b200_blur_sobel_batch", w=1080, h=40, n=2, r=5),     # WS_STAGE_FUSED
    case("erode-tma", "gs_b200_erode_batch", w=272, h=41, n=3),
    case("erode-ragged", "gs_b200_erode_batch", w=100, h=37, n=3),
    case("dilate-tma", "gs_b200_dilate_batch", w=272, h=41, n=3),
    case("dilate-ragged", "gs_b200_dilate_batch", w=100, h=37, n=3),
    case("erode_n-9", "gs_b200_erode_n_batch", w=272, h=70, n=2, iters=9),
    case("erode_n-17", "gs_b200_erode_n_batch", w=272, h=70, n=2, iters=17),               # two composed launches
    case("erode_n-ragged", "gs_b200_erode_n_batch", w=100, h=37, n=3, iters=3),            # row / column path
    case("dilate_n-9", "gs_b200_dilate_n_batch", w=272, h=70, n=2, iters=9),
    case("dilate_n-ragged", "gs_b200_dilate_n_batch", w=100, h=37, n=3, iters=4),
    case("resize-tiled", "gs_b200_resize_batch", w=272, h=60, n=3, dw=200, dh=50),
    case("resize-ragged", "gs_b200_resize_batch", w=100, h=37, n=3, dw=37, dh=50),
    case("downsample-vec", "gs_b200_downsample_batch", w=272, h=41, n=3),
    case("downsample-ragged", "gs_b200_downsample_batch", w=100, h=37, n=3),
    case("integral-bands", "gs_b200_integral_batch", w=40, h=17, n=3, env="bands"),
    case("integral-strips", "gs_b200_integral_batch", w=1000, h=37, n=3, env="strips"),
    case("integral-ragged", "gs_b200_integral_batch", w=100, h=37, n=3),
    case("histogram-vec", "gs_b200_histogram_batch", w=272, h=41, n=3),
    case("histogram-ragged", "gs_b200_histogram_batch", w=100, h=37, n=3),
    case("otsu-vec", "gs_b200_otsu_threshold_batch", w=272, h=41, n=3, with_hist=0),
    case("otsu-ragged", "gs_b200_otsu_threshold_batch", w=101, h=37, n=3, with_hist=0),
    case("threshold-vec", "gs_b200_threshold_batch", w=272, h=41, n=3, t=100),
    case("threshold-ragged", "gs_b200_threshold_batch", w=100, h=37, n=3, t=100),
    case("threshold_each-vec", "gs_b200_threshold_each_batch", w=272, h=41, n=3, offset=10),
    case("threshold_each-ragged", "gs_b200_threshold_each_batch", w=100, h=37, n=3, offset=-20),
    case("filter-3x3", "gs_b200_filter_batch", w=272, h=41, n=3, k="sharpen"),
    case("filter-7x5", "gs_b200_filter_batch", w=272, h=41, n=3, k=K7X5),
    case("match_template-packed", "gs_b200_match_template_batch", w=256, h=60, n=3, tw=30, th=24),
    case("match_template-ragged", "gs_b200_match_template_batch", w=101, h=37, n=3, tw=9, th=4),
    case("find_best_match", "gs_b200_find_best_match_batch", w=101, h=37, n=3),
    case("blobs-overflow", "gs_b200_blobs_batch", w=100, h=37, n=3, nb=12),
    case("blob_corners", "gs_b200_blob_corners", w=100, h=37),
    case("perspective-host", "gs_b200_perspective_correct_batch", w=200, h=150, n=3, dw=90, dh=71, per_frame=0),
    case("perspective-per_frame", "gs_b200_perspective_correct_batch", w=200, h=150, n=3, dw=90, dh=71, per_frame=1),
    case("fast-tiled", "gs_b200_fast_batch", w=272, h=60, n=3, t=20, nkps=400),
    case("fast-ragged", "gs_b200_fast_batch", w=101, h=37, n=3, t=10, nkps=400),
    case("orb-tiled", "gs_b200_orb_extract_batch", w=272, h=60, n=3, t=20, nkps=400),
    case("orb-ragged", "gs_b200_orb_extract_batch", w=202, h=60, n=3, t=20, nkps=400),
    case("match_orb", "gs_b200_match_orb_batch", n=3, s1=130, s2=90, mm=150),
    case("lbp-chunked", "gs_b200_lbp_detect_batch", w=136, h=130, n=3, mr=1000, chunk="1"),
    case("lbp-ragged", "gs_b200_lbp_detect_batch", w=130, h=130, n=2, mr=1000),
    # the copy kernel (nearest, an unscaled region) or the gather kernel, then the same on a ragged second geometry
    case("crop_resize-nearest", "gs_b200_crop_resize_batch", w=272, h=70, n=3, dw=64, dh=48, roi=(9, 4, 64, 48), mode=0,
         second=dict(w=101, h=37, n=2, dw=33, dh=20, roi=(9, 4, 33, 20), mode=0)),
    case("crop_resize-bilinear", "gs_b200_crop_resize_batch", w=272, h=70, n=3, dw=64, dh=48, roi=(9, 4, 80, 33), mode=1,
         second=dict(w=101, h=37, n=2, dw=33, dh=20, roi=(9, 4, 80, 33), mode=1)),
    case("rois_resize-nearest", "gs_b200_rois_resize_batch", w=272, h=70, n=3, dw=64, dh=48, mr=5, mode=0,
         second=dict(w=101, h=37, n=2, dw=33, dh=20, mr=5, mode=0)),
    case("rois_resize-bilinear", "gs_b200_rois_resize_batch", w=272, h=70, n=3, dw=64, dh=48, mr=5, mode=1,
         second=dict(w=101, h=37, n=2, dw=33, dh=20, mr=5, mode=1)),
    case("orb_pyramid", "gs_b200_orb_pyramid_batch", w=320, h=240, n=3, nkps=600, levels=3, t=20,
         second=dict(w=264, h=131, n=2, nkps=301, levels=4, t=20)),
    case("memcpy_h2d", "gs_b200_memcpy_h2d", bytes=100003),
    case("memcpy_d2h", "gs_b200_memcpy_d2h", bytes=100003),
    case("memset", "gs_b200_memset", bytes=100003),
    case("stream_sync", "gs_b200_stream_sync"),
]

# rows whose call waits by design, with the reason; every other call must return before its stream has run it
WAITS = {"stream_sync": "gs_b200_stream_sync waits for its own stream, and only for it"}

# rows that refuse graph capture by design, with the reason; the rest must capture and replay
NO_CAPTURE = {"filter-7x5": "the generic filter copies its host weights from pageable memory, which a graph would "
                            "capture by pointer; it returns cudaErrorStreamCaptureUnsupported"}

# part C: ops whose workspace holds values only (no tickets, flags or indices a race could turn into a hang)
PER_THREAD = ("otsu-ragged", "filter-7x5", "match_template-packed", "find_best_match", "erode_n-17", "dilate_n-ragged",
              "blur_sobel-staged")


# ---- CPU -----------------------------------------------------------------------------------------------------------
def test_cases_cover_every_stream_entry_point():
    declared = set()
    for path in glob.glob(os.path.join(ROOT, "include", "grayskull_b200*.h")):
        with open(path) as f:
            text = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
        for m in re.finditer(r"\b(gs_b200_\w+)\s*\(([^)]*)\)\s*;", text):
            if "gs_b200_stream" in m.group(2):
                declared.add(m.group(1))
    assert len(declared) >= 32, sorted(declared)
    named = {fn for _, fn, _ in CASES}
    assert declared == named, "header entry points without a row: %s; rows naming no entry point: %s" % (
        sorted(declared - named), sorted(named - declared))
    ids = [cid for cid, _, _ in CASES]
    assert len(ids) == len(set(ids))
    assert set(WAITS) | set(NO_CAPTURE) | set(PER_THREAD) <= set(ids)


# (object, runtime call) pairs that may block the host or use the legacy stream, each with its reason
BLOCKING = {
    ("api.o", "cudaMemcpy"): "single-image calls are synchronous (gs_filter / gs_perspective_correct read device "
                             "parameters back)",
    ("api.o", "cudaStreamCreate"): "single-image calls are synchronous: each host thread's own stream",
    ("api.o", "cudaStreamDestroy"): "single-image calls are synchronous: the thread's stream goes with the thread",
    ("api.o", "cudaStreamSynchronize"): "single-image calls are synchronous",
    ("fast_orb.o", "cudaMalloc"): "the once-per-process trig check on its private stream",
    ("fast_orb.o", "cudaFree"): "the once-per-process trig check on its private stream",
    ("fast_orb.o", "cudaStreamCreateWithFlags"): "the once-per-process trig check on its private stream",
    ("fast_orb.o", "cudaStreamDestroy"): "the once-per-process trig check on its private stream",
    ("fast_orb.o", "cudaStreamSynchronize"): "the once-per-process trig check on its private stream",
    ("lbp.o", "cudaMalloc"): "plan upload: a cache miss allocates the plan's tables",
    ("lbp.o", "cudaFree"): "plan upload: an evicted plan is freed once nobody holds it",
    ("lbp.o", "cudaStreamSynchronize"): "single-image gs_lbp_window stages its tables and waits",
    ("runtime.o", "cudaMalloc"): "workspace growth, and gs_b200_malloc",
    ("runtime.o", "cudaFree"): "workspace growth, and gs_b200_free / gs_b200_image_free",
    ("runtime.o", "cudaStreamSynchronize"): "workspace growth waits for the stream's use of the old arena; "
                                            "plan upload on its private stream; gs_b200_stream_sync",
    ("runtime.o", "cudaStreamCreateWithFlags"): "plan upload: the private non-blocking stream of upload()",
    ("runtime.o", "cudaStreamDestroy"): "plan upload: the private non-blocking stream of upload()",
    ("runtime.o", "cudaMallocHost"): "gs_b200_malloc_host",
    ("runtime.o", "cudaFreeHost"): "gs_b200_free_host",
    ("runtime.o", "cudaMallocManaged"): "gs_b200_alloc",
}
_BLOCKING_RE = re.compile(r"^(cudaMemcpy|cudaMemcpyToSymbol|cudaMemset|cudaMemcpy2D|cudaDeviceSynchronize|"
                          r"cudaStreamSynchronize|cudaEventSynchronize|cudaMalloc\w*|cudaFree\w*|cudaStreamCreate\w*|"
                          r"cudaStreamDestroy)$")


def test_blocking_runtime_calls_census():
    """cudart is linked statically, so each object's undefined symbols show the runtime calls the .so hides"""
    from grayskull_b200 import build
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm not found")
    objs = [os.path.join(build.OBJ, s.replace(".cu", ".o")) for s in build.SOURCES]
    missing = [o for o in objs if not os.path.exists(o)]
    assert not missing, "objects missing (rebuild with `python -m grayskull_b200.build --force`): %s" % missing
    found = set()
    for o in objs:
        out = subprocess.run([nm, "-u", o], capture_output=True, text=True, check=True).stdout
        for line in out.splitlines():
            sym = line.split()[-1]
            if _BLOCKING_RE.match(sym):
                found.add((os.path.basename(o), sym))
    unexplained = sorted(found - set(BLOCKING))
    assert not unexplained, "blocking or legacy-stream runtime calls without a reason: %s" % unexplained
    stale = sorted(set(BLOCKING) - found)
    assert not stale, "reasons for calls the objects no longer make: %s" % stale


# ---- GPU: the rows -------------------------------------------------------------------------------------------------
def _transfer(fn, p):
    """the rows that move or set bytes -> (spec, inputs for a seed); `host` names the buffer in pinned host memory"""
    import grayskull_b200 as g
    lib, nb = g.lib(), p.get("bytes", 0)
    if fn == "gs_b200_stream_sync":
        return calls.Spec({}, {}, lambda P, n, s: lib.gs_b200_stream_sync(s), lambda ins, bf: {}), lambda seed: {}
    if fn == "gs_b200_memset":
        return calls.Spec({}, {"dst": nb}, lambda P, n, s: lib.gs_b200_memset(P["dst"], 0x3C, nb, s),
                          lambda ins, bf: {"dst": np.full(nb, 0x3C, np.uint8)}), lambda seed: {}
    sp = calls.Spec({"src": nb}, {"dst": nb}, lambda P, n, s: getattr(lib, fn)(P["dst"], P["src"], nb, s),
                    lambda ins, bf: {"dst": ins["src"]})
    sp.host = {"src"} if fn.endswith("h2d") else {"dst"}
    return sp, lambda seed: {"src": np.random.default_rng(seed).integers(0, 256, (1, nb)).astype(np.uint8)}


class Run:
    """one row's buffers: every input on the device (or pinned, for a host input) starts as the poison; the real and
    poison inputs wait on the device, so staging either is a device copy on the stream"""

    def __init__(self, fn, p):
        import torch
        self.fn, self.n = fn, p.get("n", 1)
        if fn.endswith(("_batch", "blob_corners")):
            self.spec, gen = calls.spec(fn, p), lambda seed: calls.inputs(fn, p, self.n, seed)
        else:
            self.spec, gen = _transfer(fn, p)
        host = getattr(self.spec, "host", ())
        self.data = {seed: gen(seed) for seed in (1, 2)}
        self.src = {seed: {b: torch.from_numpy(calls.flat(x, 1 if b in self.spec.shared else self.n)).cuda()
                           for b, x in d.items()} for seed, d in self.data.items()}
        self.ins = {b: torch.empty(a.numel(), dtype=torch.uint8, pin_memory=True) if b in host else torch.empty_like(a)
                    for b, a in self.src[2].items()}
        for b, t in self.ins.items():
            t.copy_(self.src[2][b])
        self.before = calls.filled(self.spec, self.n)
        self.outs = {b: torch.empty(calls.flat(x, self.n).size, dtype=torch.uint8, pin_memory=b in host,
                                    device="cpu" if b in host else "cuda") for b, x in self.before.items()}
        torch.cuda.synchronize()

    def call(self, s):
        """the library call on torch stream s (None: cudaStreamPerThread) -> rc"""
        handle = C.c_void_p(2) if s is None else C.c_void_p(s.cuda_stream)
        return self.spec.call({b: t.data_ptr() for b, t in dict(self.ins, **self.outs).items()}, self.n, handle)

    def stage(self, s, seed):
        """enqueue on s: the inputs of `seed` over the device inputs, the poison over the device outputs (host outputs
        are filled now, on the host)"""
        import torch
        with torch.cuda.stream(s):
            for b, t in self.ins.items():
                t.copy_(self.src[seed][b], non_blocking=True)
            for t in self.outs.values():
                t.fill_(POISON)

    def results(self):
        return {b: self.outs[b] if b in self.outs else self.ins[b] for b in self.spec.outs}

    def grab(self, s):
        """enqueue on s: clones of the device results (host results are read after the sync)"""
        import torch
        with torch.cuda.stream(s):
            return {b: t.clone() if t.is_cuda else t for b, t in self.results().items()}

    def verify(self, got, seed, what=""):
        want = self.spec.expect(self.data[seed], self.before)
        for b, t in got.items():
            g, w = t.cpu().numpy(), calls.flat(want[b], self.n)
            assert np.array_equal(g, w), "%s%s (inputs of seed %d): %s: byte %d of %d differs" % (
                self.fn, what, seed, b, int(np.argmax(g != w)), g.size)

    def run_sync(self, s, seed=2):
        """one plain call on s, checked: the warm-up (sizes the workspace, builds the LBP plan, the ORB tables)"""
        self.stage(s, seed)
        rc = self.call(s)
        _ok(rc, self.fn)
        s.synchronize()
        self.verify(self.results(), seed, " warm-up")


def _ok(rc, what):
    from grayskull_b200 import _lib
    _lib.check(rc, what)


def _cudart():
    for line in open("/proc/self/maps"):
        path = line.split()[-1]
        if "libcudart.so" in os.path.basename(path):
            rt = C.CDLL(path)
            rt.cudaStreamGetFlags.argtypes = [C.c_void_p, C.POINTER(C.c_uint)]
            return rt
    pytest.fail("libcudart is not loaded in this process")


def _sleep(s, cycles):
    import torch
    with torch.cuda.stream(s):
        torch.cuda._sleep(int(cycles))


def _ids(rows):
    return [pytest.param(fn, p, id=cid) for cid, fn, p in rows]


# ---- GPU A: ordered behind pending work, no hidden waits -----------------------------------------------------------
@pytest.mark.gpu
def test_side_streams_are_non_blocking(lib):
    import torch
    flags = C.c_uint(7)
    s = torch.cuda.Stream()
    assert _cudart().cudaStreamGetFlags(C.c_void_p(s.cuda_stream), C.byref(flags)) == 0
    assert flags.value == 1, "torch.cuda.Stream() is not cudaStreamNonBlocking: the legacy stream would order it"


@pytest.mark.gpu
@pytest.mark.parametrize("fn,p", _ids(CASES))
def test_ordered_and_asynchronous(lib, fn, p, request):
    import torch
    cid = request.node.callspec.id
    run, s, u = Run(fn, p), torch.cuda.Stream(), torch.cuda.Stream()
    run.run_sync(s)
    t0 = time.perf_counter()                     # the host time of a warm call
    _ok(run.call(s), fn)
    host = time.perf_counter() - t0
    s.synchronize()
    cycles = min(max(SLEEP_MIN_CYCLES, 10 * host * 1.98e9), SLEEP_MAX_CYCLES)
    _sleep(u, min(2 * cycles, SLEEP_MAX_CYCLES))   # outlasts s's sleep, so a call that waits for s alone is told apart
    _sleep(s, cycles)
    run.stage(s, 1)
    rc = run.call(s)
    s_done, u_done = s.query(), u.query()
    got = run.grab(s)
    torch.cuda.synchronize()
    _ok(rc, fn)
    if cid in WAITS:
        assert s_done and not u_done, "%s: expected to wait for its stream and only for it" % fn
    else:
        assert not s_done, "%s returned after its stream had drained: it waited for it" % fn
        assert not u_done, "%s returned after another stream had drained: it synchronised the device" % fn
    run.verify(got, 1)


@pytest.mark.gpu
def test_single_image_calls_follow_the_legacy_stream(lib):
    """INTEGRATION.md §5: work queued on the legacy stream is ordered before a single-image call on device memory"""
    import torch
    from grayskull_b200._lib import Image
    Od = L.oracle()
    w, h = 272, 70
    a = frames(w, h, 1, 1)[0]
    src = torch.zeros((h, w), dtype=torch.uint8, device="cuda")
    dst = torch.zeros_like(src)
    real = torch.from_numpy(a).cuda()
    torch.cuda.synchronize()
    for op in ("blur", "sobel"):
        dst.fill_(POISON)
        src.zero_()
        torch.cuda.synchronize()
        stream = torch.cuda.default_stream()
        _sleep(stream, SLEEP_MIN_CYCLES)
        src.copy_(real)                           # the legacy stream: behind the sleep
        di, si = Image(w, h, dst.data_ptr()), Image(w, h, src.data_ptr())
        if op == "blur":
            lib.gs_blur(di, si, 3)
            want = L.o_blur(Od, a, 3)
        else:
            lib.gs_sobel(di, si)
            want = L.o_sobel(Od, a, POISON)
        assert np.array_equal(dst.cpu().numpy(), want), op


# ---- GPU B: two streams at once ------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("head_sleep", [False, True], ids=["interleaved", "nested"])
def test_two_streams_at_once(lib, head_sleep):
    import torch
    s0, s1 = torch.cuda.Stream(), torch.cuda.Stream()
    pairs = [(Run(fn, p), Run(fn, _second(p))) for cid, fn, p in CASES if cid not in WAITS]
    for r0, r1 in pairs:                         # each stream's workspace sized for its own geometry
        r0.run_sync(s0)
        r1.run_sync(s1)
    if head_sleep:                               # s0's whole sequence runs while s1 is held
        _sleep(s1, SLEEP_MIN_CYCLES)
    got = []
    for r0, r1 in pairs:
        for r, s in ((r0, s0), (r1, s1)):
            r.stage(s, 1)
            _ok(r.call(s), r.fn)
            got.append((r, r.grab(s)))
    torch.cuda.synchronize()
    for k, (r, g) in enumerate(got):
        r.verify(g, 1, " on stream %d" % (k % 2))


# ---- GPU C: cudaStreamPerThread from two host threads ----------------------------------------------------------------
def _long_filter():
    """thread A's long call: a generic 9x9 filter over 64 identical 2048 x 2048 frames (256 MiB)"""
    import torch
    import grayskull_b200 as g
    w = h = 2048
    n = 64
    a = L.natural_like(w, h, 5)
    k = np.random.default_rng(9).integers(-3, 4, (9, 9)).astype(np.int8).view(np.uint8)
    k = np.ascontiguousarray(k)
    src = torch.from_numpy(a).cuda().expand(n, h, w).contiguous()
    dst = torch.empty_like(src)
    want = np.zeros_like(a)
    L.oracle().gso_filter(L.ptr(want), L.ptr(a), w, h, L.ptr(k), 9, 9, 7)
    call = lambda: g.lib().gs_b200_filter_batch(dst.data_ptr(), src.data_ptr(), w, h, n, k.ctypes.data, 9, 9, 7,  # noqa
                                                C.c_void_p(2))
    return call, dst, torch.from_numpy(want).cuda()


@pytest.mark.gpu
def test_stream_per_thread_has_per_thread_scratch(lib):
    import torch
    rows = {cid: (fn, p) for cid, fn, p in CASES}
    runs = {who: [Run(*rows[cid]) for cid in PER_THREAD] for who in "AB"}
    long_call, long_dst, long_want = _long_filter()
    staged = [{b: t.cpu().numpy() for b, t in r.src[1].items()} for r in runs["B"]]
    torch.cuda.synchronize()
    a_returned, errors, got = threading.Event(), [], {}

    def sync():
        _ok(lib.gs_b200_stream_sync(C.c_void_p(2)), "gs_b200_stream_sync")

    def warm(who):
        for r in runs[who]:
            _ok(r.call(None), r.fn)
        if who == "A":
            _ok(long_call(), "long filter")
        sync()

    def thread_a():
        try:
            _ok(long_call(), "long filter")
            a_returned.set()
            sync()
        except BaseException as e:   # noqa: B036
            errors.append(e)
            a_returned.set()

    def thread_b():
        try:
            a_returned.wait(60)
            # nothing on the legacy stream from here on: it would wait for thread A's stream
            for r, host in zip(runs["B"], staged):
                for b, t in r.ins.items():            # the real inputs, on this thread's stream only
                    _ok(lib.gs_b200_memcpy_h2d(t.data_ptr(), host[b].ctypes.data, host[b].nbytes, C.c_void_p(2)), "h2d")
                for t in r.outs.values():
                    _ok(lib.gs_b200_memset(t.data_ptr(), POISON, t.numel(), C.c_void_p(2)), "memset")
                _ok(r.call(None), r.fn)
            sync()
            got["B"] = [{b: t.cpu() for b, t in r.results().items()} for r in runs["B"]]
        except BaseException as e:   # noqa: B036
            errors.append(e)

    # warm-ups run one thread after the other, so that no arena grows while the other thread's work runs
    ta = threading.Thread(target=warm, args=("A",))
    ta.start()
    ta.join()
    tb = threading.Thread(target=warm, args=("B",))
    tb.start()
    tb.join()
    long_dst.zero_()
    torch.cuda.synchronize()
    ta, tb = threading.Thread(target=thread_a), threading.Thread(target=thread_b)
    tb.start()
    ta.start()
    ta.join(120)
    tb.join(120)
    assert not ta.is_alive() and not tb.is_alive()
    if errors:
        raise errors[0]
    torch.cuda.synchronize()
    for r, g in zip(runs["B"], got["B"]):
        r.verify(g, 1, " (thread B)")
    bad = [f for f in range(long_dst.shape[0]) if not torch.equal(long_dst[f], long_want)]
    assert not bad, "thread A's filter differs from the oracle in frames %s: its scratch was not its own" % bad


# ---- GPU D: CUDA graph capture -------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("fn,p", _ids([c for c in CASES if c[0] not in WAITS]))
def test_graph_capture_and_replay(lib, fn, p, request):
    import torch
    cid = request.node.callspec.id
    run, s = Run(fn, p), torch.cuda.Stream()
    run.run_sync(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        rc = run.call(s)
    if cid in NO_CAPTURE:
        assert rc == CAPTURE_UNSUPPORTED, (rc, lib.gs_b200_last_error())
        run.run_sync(s, 1)                       # still correct uncaptured
        return
    _ok(rc, fn)
    if run.spec.mutate:
        run.spec.mutate()                        # the graph keeps the values it captured
    for seed in (1, 2):
        run.stage(s, seed)
        with torch.cuda.stream(s):
            g.replay()
        got = run.grab(s)
        s.synchronize()
        run.verify(got, seed, " replay")


GROW = [pytest.param("gs_b200_otsu_threshold_batch", dict(w=101, h=37, n=2, with_hist=0),
                     dict(w=101, h=37, n=64, with_hist=0), False, id="otsu"),
        # torch may report the invalidated capture itself; the call's status is what counts
        pytest.param("gs_b200_orb_pyramid_batch", dict(w=128, h=96, n=1, nkps=50, levels=3, t=20),
                     dict(w=512, h=384, n=3, nkps=2000, levels=3, t=20), True, id="orb_pyramid")]


@pytest.mark.gpu
@pytest.mark.parametrize("fn,small,big,torch_may_refuse", GROW)
def test_workspace_cannot_grow_inside_a_capture(lib, fn, small, big, torch_may_refuse):
    """a capture that would need a larger arena fails with a clear error and leaves the arena as it was"""
    import torch
    small, big = Run(fn, small), Run(fn, big)
    s = torch.cuda.Stream()
    small.run_sync(s)
    g, rc = torch.cuda.CUDAGraph(), None
    try:
        with torch.cuda.graph(g, stream=s):
            rc = big.call(s)
    except RuntimeError:
        if not torch_may_refuse:
            raise
    assert rc == CAPTURE_UNSUPPORTED, (rc, lib.gs_b200_last_error())
    assert b"capturing" in lib.gs_b200_last_error()
    small.run_sync(s, 1)                         # the old arena still serves the small geometry
    big.run_sync(s, 1)                           # and the next uncaptured call grows it
