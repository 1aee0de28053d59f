"""ORB over an image pyramid on the device (include/grayskull_b200_pyramid.h), bit-exact with the reference CLI's
multi-scale ORB: extract_pyramid_orb_nm of its `orb` verb.

pyramid_orb() (tests/_libs.py) restates that helper from its behaviour on the oracle's gso_downsample / gso_orb_extract, with its
one buffer (pyramid levels 1..L-1, then score maps 0..L-1) as a numpy array; orb_verb_line() restates the verb's
printed line, the 1 MiB buffer it shares between the template and the scene included.  test_dispatch_paths.py has the
rows that pick each kernel of the call, the pyramid's own (gsb::k_pyr_*) included, and checks that its launches go
through gsb::launch; test_host_logic.py checks the exports, the binding table and that every kernel is sm_90a,
test_streams.py the runtime calls of pyramid.o.

  * CPU: the level rule; the restatement equals the compiled reference CLI (when oracle/_ref is built) on lena and on
    template / scene pairs of different sizes, one of which the stale buffer changes.
  * GPU: every frame bit-exact against the restatement -- keypoints up to the count, untouched slots after it, every
    pyramid byte and every score-map byte with the caller's bytes as the maps' start -- at tiled and generic widths,
    L = 1..4 and a request for 5, skipped early levels, corner-rich frames whose last level's per-frame cap truncates,
    trig mode 1, n = 0 and nkps = 0; the CLI's orb stage against the compiled reference CLI.  test_streams.py
    runs the call on the caller's stream, on two streams at once, in a graph, and refuses its workspace growth under
    capture.
"""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import _libs as L
from _calls import POISON
from _libs import layout, level_rule, pyramid_orb
from _gpu import O, frames, lib, traced, witness, witnessed  # noqa: F401

ROOT = L.ROOT
QUOTA, MERGE = "gsb::k_pyr_quota", "gsb::k_pyr_merge"
FAST_T, FAST_G = "gsb::k_fast_tiled2<true>", "gsb::k_fast_tiled2<false>"   # TMA tile loads, or plain loads
SELECT, BRIEF_W, BRIEF_B = "gsb::k_orb_select", "gsb::k_orb_brief<true>", "gsb::k_orb_brief<false>"
DOWN = "gsb::k_downsample_vec"
BUF = 1024 * 1024        # nanomagick.c:299


# ---- the reference CLI's orb verb, restated ------------------------------------------------------------------------------
def orb_verb_line(Od, tpl, scene, stale=True):
    """the line the orb verb prints (nanomagick.c:299-311).  stale: one zeroed 1 MiB buffer shared by both calls, as
    there; otherwise each call gets a zeroed buffer of its own."""
    buf = np.zeros(BUF, np.uint8)
    kt = pyramid_orb(Od, tpl, 2500, 20, buf, 3)
    if not stale:
        buf[:] = 0
    ks = pyramid_orb(Od, scene, 2500, 20, buf, 3)
    m = L.o_match(Od, kt, ks, 300, 60.0)
    return "Template: %u keypoints, Scene: %u keypoints, Matches: %u" % (len(kt), len(ks), len(m))


def pyramid_lib():
    from grayskull_b200 import pyramid
    return pyramid.lib()


# ---- CPU: the library --------------------------------------------------------------------------------------------------
def test_levels_follow_the_helper_rule():
    lp = pyramid_lib()
    sides = [1, 7, 31, 32, 63, 64, 65, 127, 128, 129, 255, 256, 257, 300, 640, 1080, 1920, 4096]
    for w in sides:
        for h in sides:
            for lv in (0, 1, 2, 3, 4, 5, 9):
                assert lp.gs_b200_orb_pyramid_levels(w, h, lv) == level_rule(w, h, lv), (w, h, lv)
    # 63 / 64 / 65: 63 / 2 = 31 stops at level 1, 64 / 2 = 32 runs and 32 / 2 = 16 stops, 65 likewise
    assert [level_rule(s, 500, 4) for s in (63, 64, 65, 128, 129)] == [1, 2, 2, 3, 3]
    assert level_rule(1000, 1000, 5) == 4 and level_rule(1000, 1000, 0) == 0 and level_rule(5, 5, 1) == 1


def test_zero_quota_and_empty_batch_run_without_a_gpu():
    """n == 0 returns before anything is enqueued; a missing pointer aborts with the assert's text"""
    code = ("import ctypes as C, sys; sys.path.insert(0, %r); from grayskull_b200 import pyramid; "
            "L = pyramid.lib(); P = C.c_void_p(4096); rc = %s; print('rc', rc)")
    ok = subprocess.run([sys.executable, "-c", code % (ROOT, "L.gs_b200_orb_pyramid_batch(P, 64, 64, 0, 3, P, P, P, "
                                                                 "P, 100, 20, None)")],
                        capture_output=True, text=True, timeout=120)
    assert ok.returncode == 0 and "rc 0" in ok.stdout, (ok.stdout, ok.stderr)
    bad = subprocess.run([sys.executable, "-c", code % (ROOT, "L.gs_b200_orb_pyramid_batch(P, 64, 64, 2, 3, P, P, P, "
                                                                  "None, 100, 20, None)")],
                         capture_output=True, text=True, timeout=120)
    assert bad.returncode != 0 and "Assertion failed: counts" in bad.stderr, bad.stderr


# ---- CPU: the restatement against the compiled reference CLI ------------------------------------------------------------
def _nanomagick():
    path = os.path.join(ROOT, "oracle", "_ref", "nanomagick_cpu")
    return path if os.path.exists(path) else None


def _pgm(path, a):
    with open(path, "wb") as f:
        f.write(b"P5\n%d %d\n255\n" % (a.shape[1], a.shape[0]) + a.tobytes())
    return str(path)


def _verb_line(exe, tpl_path, scene_path, out):
    r = subprocess.run([exe, "orb", tpl_path, scene_path, str(out)], capture_output=True, text=True, timeout=300)
    m = re.search(r"Template: \d+ keypoints, Scene: \d+ keypoints, Matches: \d+", r.stdout)
    assert m, (r.stdout, r.stderr)
    return m.group(0)


def _lena():
    return np.ascontiguousarray(np.load(os.path.join(ROOT, "tests", "golden", "lena_golden.npz"))["lena"])


def stale_pair():
    """a template / scene pair whose scene line the stale buffer changes: the 38-px-wide noise scene has a single level
    whose score map starts as the template's pyramid pixels, so its ring suppresses FAST survivors in columns 3 and 34;
    those survivors fill FAST's 5000 cap ahead of the margin-passing ones, so the cap window and the count move"""
    rng = np.random.default_rng(71)
    tpl = L.natural_like(640, 480, 70)
    scene = rng.integers(0, 256, (2600, 38), dtype=np.uint8)
    return tpl, scene


def verb_pairs():
    rng = np.random.default_rng(5)
    lena = _lena()
    return {
        "lena": (lena, lena),
        "lena-crop": (np.ascontiguousarray(lena[40:200, 30:230]), lena),
        "small-big": (L.natural_like(96, 80, 3), L.natural_like(400, 300, 4)),
        "big-small": (L.natural_like(500, 400, 6), rng.integers(0, 256, (130, 190), dtype=np.uint8)),
        "stale": stale_pair(),
    }


@pytest.mark.skipif(_nanomagick() is None, reason="oracle/_ref/nanomagick_cpu not built (no reference checkout)")
def test_restatement_matches_reference_cli(tmp_path):
    exe, Od = _nanomagick(), L.oracle()
    for name, (tpl, scene) in verb_pairs().items():
        want = _verb_line(exe, _pgm(tmp_path / ("%s_t.pgm" % name), tpl), _pgm(tmp_path / ("%s_s.pgm" % name), scene),
                          tmp_path / ("%s_o.pgm" % name))
        assert orb_verb_line(Od, tpl, scene) == want, name
        if name == "lena":
            assert want == "Template: 340 keypoints, Scene: 340 keypoints, Matches: 300"
    tpl, scene = stale_pair()
    assert orb_verb_line(Od, tpl, scene, stale=False) != orb_verb_line(Od, tpl, scene), "the stale ring changed nothing"


# ---- GPU: parity ---------------------------------------------------------------------------------------------------------
def corner_rich(w, h, seed):
    """uniform noise: FAST survivors everywhere, so early levels fill their quota and caps truncate"""
    return np.random.default_rng(seed).integers(0, 256, (h, w), dtype=np.uint8)


def _case(cid, w, h, n, nkps, levels, t=20, maps="random", kind="mixed", kernels=(), trig=0):
    return pytest.param(dict(w=w, h=h, n=n, nkps=nkps, levels=levels, t=t, maps=maps, kind=kind, kernels=kernels,
                             trig=trig), id=cid)


CASES = [
    # w % 16 == 0: tiled FAST and word BRIEF on every level
    _case("tiled-L3", 512, 384, 3, 600, 3, kernels=(FAST_T, BRIEF_W, DOWN)),
    _case("tiled-L4", 1024, 256, 2, 900, 4, kernels=(FAST_T, BRIEF_W)),
    _case("tiled-ask5", 640, 512, 2, 1003, 5, kernels=(FAST_T,)),                    # 4 levels run; 1003 % 4 != 0
    # odd and 8 mod 16 widths: their levels take the generic FAST and byte BRIEF
    _case("odd-L3", 333, 201, 3, 400, 3, kernels=(FAST_G, BRIEF_B)),
    _case("w8mod16-L3", 264, 200, 2, 500, 3, kernels=(FAST_G, BRIEF_W, BRIEF_B)),     # 264, 132, 66
    _case("w8mod16-L2", 200, 130, 3, 301, 2, kernels=(FAST_G, BRIEF_W)),            # 200, 100
    # level counts 1 and 2 from the 32-px rule
    _case("L1-narrow", 63, 400, 3, 300, 3, kernels=(FAST_G,)),
    _case("L2-rule", 128, 64, 2, 200, 4),
    _case("L1-asked", 256, 128, 2, 150, 1, kernels=(FAST_T,)),
    # nkps < L: the early levels are skipped, the last level takes everything
    _case("skip-early", 256, 256, 3, 2, 3),
    _case("skip-early4", 512, 512, 2, 3, 4),
    # corner-rich frames: early levels fill their quota and the last level's cap 4 * q_f < 5000 truncates
    _case("rich", 1280, 960, 2, 2500, 3, kind="rich"),
    _case("rich-odd", 331, 417, 2, 60, 3, kind="rich"),
    # zeroed maps, a high threshold, trig mode 1
    _case("zero-maps", 320, 240, 3, 500, 3, maps="zero"),
    _case("t-high", 320, 240, 3, 500, 3, t=200),
    _case("trig1", 400, 300, 2, 700, 3, trig=1),
]


def _frames(c):
    if c["kind"] == "rich":
        return np.stack([corner_rich(c["w"], c["h"], 100 + f) for f in range(c["n"])])
    return frames(c["w"], c["h"], c["n"], 7 + c["w"])


def _run(lp, src_np, nkps, t, levels, maps_np):
    """one device call with the given start of the score maps; poison in pyr and kps -> (counts, kps, pyr, maps, seen)"""
    import torch
    n, h, w = src_np.shape
    sizes, _, _, _ = layout(w, h, levels)
    below = sum(a * b for a, b in sizes[1:]) * n
    src = torch.from_numpy(src_np).cuda()
    sm = torch.from_numpy(maps_np.copy()).cuda() if maps_np.size else torch.zeros(1, dtype=torch.uint8, device="cuda")
    pyr = torch.full((max(below, 1),), POISON, dtype=torch.uint8, device="cuda")
    kps = torch.full((n, max(nkps, 1), 48), POISON, dtype=torch.uint8, device="cuda")
    counts = torch.full((max(n, 1),), 0x7777, dtype=torch.int32, device="cuda")
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc, seen = traced(lambda: lp.gs_b200_orb_pyramid_batch(src.data_ptr(), w, h, n, levels, pyr.data_ptr() if below else None,
                                                           sm.data_ptr(), kps.data_ptr(), counts.data_ptr(), nkps, t, s))
    return rc, counts.cpu().numpy(), kps.cpu().numpy(), pyr.cpu().numpy()[:below], sm.cpu().numpy()[:maps_np.size], seen


def _check(c, counts, kps, pyr, maps, want):
    kl, wpyr, wmaps = want
    nkps = c["nkps"]
    for f, k in enumerate(kl):
        assert counts[f] == len(k), "frame %d: count %d, want %d" % (f, counts[f], len(k))
        got = kps[f].reshape(-1)[:len(k) * 48].view(L.KP_DTYPE)
        if c["trig"]:
            for fld in ("x", "y", "response"):
                assert np.array_equal(got[fld], k[fld]), (f, fld)
            assert np.abs(got["angle"] - k["angle"]).max(initial=0) <= 1e-5, f
            same = got["angle"].view(np.uint32) == k["angle"].view(np.uint32)
            assert np.array_equal(got["descriptor"][same], k["descriptor"][same]), f
        else:
            assert got.tobytes() == k.tobytes(), "frame %d: keypoints differ" % f
        assert (kps[f].reshape(-1)[len(k) * 48:nkps * 48] == POISON).all(), "frame %d: a slot past the count was written" % f
    assert np.array_equal(pyr, wpyr), "pyramid bytes differ"
    assert np.array_equal(maps, wmaps), "score-map bytes differ"


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES)
def test_pyramid_vs_restatement(lib, O, witness, c):
    lp = pyramid_lib()
    src = _frames(c)
    n, h, w = src.shape
    sizes, _, _, _ = layout(w, h, c["levels"])
    nmaps = sum(a * b for a, b in sizes) * n
    maps = (np.random.default_rng(w + h).integers(0, 256, nmaps, dtype=np.uint8) if c["maps"] == "random"
            else np.zeros(nmaps, np.uint8))
    want = L.pyramid_expected(O, src, c["nkps"], c["t"], c["levels"], maps)

    def run():
        lib.gs_b200_set_trig_mode(c["trig"])
        try:
            rc, counts, kps, pyr, got_maps, seen = _run(lp, src, c["nkps"], c["t"], c["levels"], maps)
        finally:
            lib.gs_b200_set_trig_mode(0)
        assert rc == 0, lib.gs_b200_last_error()
        _check(c, counts, kps, pyr, got_maps, want)
        return seen
    kernels = [QUOTA, MERGE, SELECT, "gsb::k_orb_moments", "gsb::k_orb_trig"] + list(c["kernels"])
    witnessed(witness, run, kernels, "orb_pyramid %s" % c)
    if c["kind"] == "rich":
        # the last level's per-frame cap truncates: with cap 5000 its list would differ
        capped = L.pyramid_expected(O, src, c["nkps"], c["t"], c["levels"], maps, last_cap_5000=True)[0]
        for f in range(n):
            assert capped[f].tobytes() != want[0][f].tobytes(), "frame %d: the last level's cap did not truncate" % f


@pytest.mark.gpu
def test_empty_batch_and_zero_quota(lib, O):
    import torch
    lp = pyramid_lib()
    src = torch.from_numpy(frames(128, 96, 2, 3)).cuda()
    kps = torch.full((2, 4, 48), POISON, dtype=torch.uint8, device="cuda")
    sm = torch.full((2 * (128 * 96 + 64 * 48),), 0x3C, dtype=torch.uint8, device="cuda")
    pyr = torch.full((2 * 64 * 48,), POISON, dtype=torch.uint8, device="cuda")
    counts = torch.full((2,), 0x7777, dtype=torch.int32, device="cuda")
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for n, nkps, levels in ((0, 4, 2), (2, 0, 2), (2, 4, 0)):
        counts.fill_(0x7777)
        assert lp.gs_b200_orb_pyramid_batch(src.data_ptr(), 128, 96, n, levels, pyr.data_ptr(), sm.data_ptr(),
                                            kps.data_ptr(), counts.data_ptr(), nkps, 20, s) == 0
        torch.cuda.synchronize()
        assert counts.tolist() == ([0x7777] * 2 if n == 0 else [0, 0]), (n, nkps, levels)
        assert bool((kps == POISON).all()) and bool((pyr == POISON).all()) and bool((sm == 0x3C).all())
    buf = np.zeros(layout(128, 96, 2)[3], np.uint8)
    assert len(pyramid_orb(O, src[0].cpu().numpy(), 0, 20, buf, 2)) == 0


@pytest.mark.gpu
def test_python_wrapper(lib, O):
    from grayskull_b200 import api, pyramid
    a = frames(300, 200, 2, 12)
    import torch
    kps, counts, sm, pyr = pyramid.orb_pyramid_batch(torch.from_numpy(a).cuda(), 500, 20, levels=3)
    torch.cuda.synchronize()
    got = api.kps_to_numpy(kps, counts)
    kl, wpyr, wmaps = L.pyramid_expected(O, a, 500, 20, 3, np.zeros(sm.numel(), np.uint8))
    for f in range(2):
        assert got[f].tobytes() == kl[f].tobytes(), f
    assert np.array_equal(pyr.cpu().numpy(), wpyr) and np.array_equal(sm.cpu().numpy(), wmaps)


# ---- GPU: the CLI's orb stage ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("pair", ["same-size", "other-size"])
def test_gsb_magick_orb_stage(lib, O, tmp_path, pair):
    from grayskull_b200 import build
    exe = os.path.join(os.path.dirname(build.LIB), "gsb_magick")
    lena = _lena()
    if pair == "same-size":
        tpl, scenes = lena, [lena, np.ascontiguousarray(lena[:, ::-1]), L.natural_like(lena.shape[1], lena.shape[0], 2)]
    else:
        tpl = np.ascontiguousarray(lena[60:220, 50:250])
        scenes = [lena, L.natural_like(lena.shape[1], lena.shape[0], 8), corner_rich(lena.shape[1], lena.shape[0], 9)]
    tp = _pgm(tmp_path / "tpl.pgm", tpl)
    ins = [_pgm(tmp_path / ("in%d.pgm" % f), s) for f, s in enumerate(scenes)]
    r = subprocess.run([exe, "orb:" + tp, str(tmp_path / "out")] + ins, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("frame ")]
    ref = _nanomagick()
    for f, s in enumerate(scenes):
        want = orb_verb_line(O, tpl, s)
        if ref is not None:
            assert _verb_line(ref, tp, ins[f], tmp_path / ("ref%d.pgm" % f)) == want
        assert lines[f] == "frame %d: %s" % (f, want), (lines, want)
        data = (tmp_path / ("out%04d.pgm" % f)).read_bytes()
        assert data[-s.size:] == s.tobytes(), "frame %d changed" % f
