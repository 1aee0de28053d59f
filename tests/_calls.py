"""One description of each public batch call of include/grayskull_b200*.h, keyed by its C symbol, for the table-driven
GPU tests (test_dispatch_paths.py, test_streams.py, test_batch_limits.py).  TEST INFRASTRUCTURE only.

spec(sym, g) describes the call at the geometry and scalars g:
  * ins / outs: buffer name -> bytes per frame (a list: level-major segments, each holding every frame); a name in both
    is read and written in place; a name in `shared` is one buffer for the whole batch (its total bytes);
  * call(P, n, s): the C call on the device pointers P[name] over n frames on stream s -> status, under spec.env;
  * expect(ins, before) -> {out: its expected bytes per frame}.  ins hold k distinct frames (leading axis); before holds
    each output's bytes per frame before the call, which sobel's 1-px frame and the list slots past a count keep;
  * mutate(): changes the host parameters a captured graph holds by value (filter weights, the perspective host quad,
    match_orb's max_distance, the LBP cascade).
inputs(sym, g, k, seed) is the default input generator: seed 1 gives the real inputs, another seed valid inputs of the
same call that differ from them (the poison of test_streams.py).  Buffers a caller fills before a call hold POISON."""
import os

import numpy as np

import _libs as L

POISON = 0xA5
LBP = (1.1, 1.0, 4.0, 2)                  # scale_factor, min_scale, max_scale, step


class Spec:
    def __init__(self, ins, outs, call, expect, shared=(), mutate=None, env=None):
        self.ins, self.outs, self.expect, self.shared = ins, outs, expect, set(shared)
        self._call, self.mutate, self.env = call, mutate, env or {}

    def call(self, P, n, s):
        old = {k: os.environ.get(k) for k in self.env}
        os.environ.update(self.env)
        try:
            return self._call(P, n, s)
        finally:
            for k, v in old.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v


def segments(x, k):
    """k frames of a buffer (an array with the frames on its leading axis, or a list of level-major segments of such)
    -> [(k, bytes per frame) uint8] per segment"""
    return [np.frombuffer(np.ascontiguousarray(a).tobytes(), np.uint8).reshape(k, -1) for a in
            (x if isinstance(x, list) else [x])]


def flat(x, k):
    """k frames of a buffer -> its bytes as they lie on the device (none for a list of no segments: a 1-level pyramid)"""
    return np.concatenate([np.zeros(0, np.uint8)] + [s.reshape(-1) for s in segments(x, k)])


def unflat(b, per, k):
    """a buffer's bytes on the device -> (k, bytes per frame), or a list of those per segment when `per` is a list"""
    if not isinstance(per, list):
        return b[:k * per].reshape(k, per)
    out, off = [], 0
    for p in per:
        out.append(b[off:off + k * p].reshape(k, p))
        off += k * p
    return out


def filled(sp, k, byte=POISON):
    """expect()'s `before` for k frames of every output of sp that is not also an input, all `byte`"""
    return {o: unflat(np.full(k * sum(per if isinstance(per, list) else [per]), byte, np.uint8), per, k)
            for o, per in sp.outs.items() if o not in sp.ins}


def records(lists, before):
    """per frame: its records, then the bytes the slots after them held before"""
    out = np.array(before, np.uint8).reshape(len(lists), -1)
    for i, r in enumerate(lists):
        b = np.frombuffer(np.ascontiguousarray(r).tobytes(), np.uint8)
        out[i, :b.size] = b
    return out


def counts(lists):
    return np.array([len(r) for r in lists], np.uint32)


def o_blobs(O, a, nb):
    h, w = a.shape
    labels, blobs = np.zeros((h, w), np.uint16), np.zeros(nb, L.BLOB_DTYPE)
    m = O.gso_blobs(L.ptr(a), w, h, L.ptr(labels), L.ptr(blobs), nb)
    return labels, blobs[:m]


def filter_weights(k):
    """a filter_kernel name, or (uint8 weights, norm)"""
    return L.filter_kernel(k) if isinstance(k, str) else k


def host_quad():
    """the host corners of perspective_correct with per_frame = 0"""
    return np.random.default_rng(5).integers(0, 140, (4, 2)).astype(np.uint32)


def _each(fn, xs):
    return np.stack([fn(a) for a in xs])


def spec(sym, g):
    import grayskull_b200 as gb
    lib, O = gb.lib(), L.oracle()
    w, h = g.get("w"), g.get("h")
    px = (w or 0) * (h or 0)
    one = {"src": px}

    if sym in ("gs_b200_blur_batch", "gs_b200_adaptive_threshold_batch", "gs_b200_blur_sobel_batch"):
        r = g["r"]
        if sym == "gs_b200_blur_batch":
            return Spec(one, {"dst": px}, lambda P, n, s: lib.gs_b200_blur_batch(P["dst"], P["src"], w, h, n, r, s),
                        lambda ins, bf: {"dst": _each(lambda a: L.o_blur(O, a, r), ins["src"])})
        if sym == "gs_b200_adaptive_threshold_batch":
            c = g["c"]
            return Spec(one, {"dst": px},
                        lambda P, n, s: lib.gs_b200_adaptive_threshold_batch(P["dst"], P["src"], w, h, n, r, c, s),
                        lambda ins, bf: {"dst": _each(lambda a: L.o_adaptive(O, a, r, c), ins["src"])})
        return Spec(one, {"dst": px}, lambda P, n, s: lib.gs_b200_blur_sobel_batch(P["dst"], P["src"], w, h, n, r, s),
                    lambda ins, bf: {"dst": np.stack([L.o_sobel(O, L.o_blur(O, a, r), b.reshape(h, w))
                                                      for a, b in zip(ins["src"], bf["dst"])])})
    if sym in ("gs_b200_sobel_batch", "gs_b200_erode_batch", "gs_b200_dilate_batch"):
        f = getattr(lib, sym)
        if sym == "gs_b200_sobel_batch":
            want = lambda ins, bf: {"dst": np.stack([L.o_sobel(O, a, b.reshape(h, w))           # noqa: E731
                                                     for a, b in zip(ins["src"], bf["dst"])])}
        else:
            want = lambda ins, bf: {"dst": _each(lambda a: L.o_morph(O, a, "dilate" in sym), ins["src"])}  # noqa: E731
        return Spec(one, {"dst": px}, lambda P, n, s: f(P["dst"], P["src"], w, h, n, s), want)
    if sym in ("gs_b200_erode_n_batch", "gs_b200_dilate_n_batch"):
        f, it = getattr(lib, sym), g["iters"]

        def morph_n(a):
            for _ in range(min(it, max(w, h))):     # past max(w, h) - 1 passes the square covers the frame
                a = L.o_morph(O, a, "dilate" in sym)
            return a
        return Spec(one, {"dst": px}, lambda P, n, s: f(P["dst"], P["src"], w, h, n, it, s),
                    lambda ins, bf: {"dst": _each(morph_n, ins["src"])})
    if sym == "gs_b200_resize_batch":
        dw, dh = g["dw"], g["dh"]
        return Spec(one, {"dst": dw * dh}, lambda P, n, s: lib.gs_b200_resize_batch(P["dst"], dw, dh, P["src"], w, h, n, s),
                    lambda ins, bf: {"dst": _each(lambda a: L.o_resize(O, a, dw, dh), ins["src"])})
    if sym == "gs_b200_downsample_batch":
        return Spec(one, {"dst": (w // 2) * (h // 2)},
                    lambda P, n, s: lib.gs_b200_downsample_batch(P["dst"], P["src"], w, h, n, s),
                    lambda ins, bf: {"dst": _each(lambda a: L.o_down(O, a), ins["src"])})
    if sym == "gs_b200_integral_batch":
        return Spec(one, {"ii": 4 * px}, lambda P, n, s: lib.gs_b200_integral_batch(P["ii"], P["src"], w, h, n, s),
                    lambda ins, bf: {"ii": _each(lambda a: L.o_integral(O, a), ins["src"])},
                    env={"GS_B200_INTEGRAL": g["env"]} if "env" in g else None)
    hist = lambda a: np.bincount(a.ravel(), minlength=256).astype(np.uint32)     # noqa: E731
    if sym == "gs_b200_histogram_batch":
        return Spec(one, {"hist": 1024}, lambda P, n, s: lib.gs_b200_histogram_batch(P["hist"], P["src"], w, h, n, s),
                    lambda ins, bf: {"hist": _each(hist, ins["src"])})
    if sym == "gs_b200_otsu_threshold_batch":
        # with_hist = 0: no histogram output (a null pointer)
        with_hist = g.get("with_hist", 1)

        def want(ins, bf):
            out = {"thresh": np.array([O.gso_otsu_threshold(L.ptr(a), w, h) for a in ins["src"]], np.uint8)}
            if with_hist:
                out["hist"] = _each(hist, ins["src"])
            return out
        return Spec(one, dict({"thresh": 1}, **({"hist": 1024} if with_hist else {})),
                    lambda P, n, s: lib.gs_b200_otsu_threshold_batch(P["thresh"], P.get("hist"), P["src"], w, h, n, s),
                    want)
    if sym in ("gs_b200_threshold_batch", "gs_b200_threshold_each_batch"):
        each = sym == "gs_b200_threshold_each_batch"

        def want(ins, bf):
            out, thr = [], np.asarray(ins.get("thresh", ())).reshape(-1)
            for i, a in enumerate(ins["src"]):
                b = np.array(a, np.uint8).reshape(h, w)
                O.gso_threshold(L.ptr(b), w, h, (int(thr[i]) + g["offset"]) & 255 if each else g["t"])
                out.append(b)
            return {"src": np.stack(out)}
        if each:
            return Spec(dict(one, thresh=1), one, lambda P, n, s: lib.gs_b200_threshold_each_batch(
                P["src"], w, h, n, P["thresh"], g["offset"], s), want)
        return Spec(one, one, lambda P, n, s: lib.gs_b200_threshold_batch(P["src"], w, h, n, g["t"], s), want)
    if sym == "gs_b200_filter_batch":
        k, norm = filter_weights(g["k"])
        ks = np.ascontiguousarray(k).copy()            # the host weights a call reads
        k0 = ks.copy()

        def want(ins, bf):
            out = []
            for a in ins["src"]:
                d = np.zeros((h, w), np.uint8)
                O.gso_filter(L.ptr(d), L.ptr(a), w, h, L.ptr(k0), k0.shape[1], k0.shape[0], norm)
                out.append(d)
            return {"dst": np.stack(out)}

        def mutate():
            ks[:] = 1
        return Spec(one, {"dst": px}, lambda P, n, s: lib.gs_b200_filter_batch(
            P["dst"], P["src"], w, h, n, ks.ctypes.data, ks.shape[1], ks.shape[0], norm, s), want, mutate=mutate)
    if sym == "gs_b200_match_template_batch":
        tw, th = g["tw"], g["th"]
        rw, rh = w - tw + 1, h - th + 1

        def want(ins, bf):
            out = []
            for a in ins["src"]:
                d = np.zeros((rh, rw), np.uint8)
                O.gso_match_template(L.ptr(a), w, h, L.ptr(np.ascontiguousarray(ins["tmpl"])), tw, th, L.ptr(d))
                out.append(d)
            return {"res": np.stack(out)}
        return Spec(dict(one, tmpl=tw * th), {"res": rw * rh}, lambda P, n, s: lib.gs_b200_match_template_batch(
            P["res"], P["src"], w, h, n, P["tmpl"], tw, th, s), want, shared=("tmpl",))
    if sym == "gs_b200_find_best_match_batch":
        def best(a):
            b = O.gso_find_best_match(L.ptr(np.ascontiguousarray(a)), w, h)
            return np.array([b % w, b // w], np.uint32)
        return Spec({"res": px}, {"best": 8}, lambda P, n, s: lib.gs_b200_find_best_match_batch(
            P["best"], P["res"], w, h, n, s), lambda ins, bf: {"best": _each(best, ins["res"])})
    if sym == "gs_b200_blobs_batch":
        nb = g["nb"]

        def want(ins, bf):
            res = [o_blobs(O, a, nb) for a in ins["src"]]
            return {"labels": np.stack([lb for lb, _ in res]), "blobs": records([b for _, b in res], bf["blobs"]),
                    "counts": counts([b for _, b in res])}
        return Spec(one, {"labels": 2 * px, "blobs": 32 * nb, "counts": 4}, lambda P, n, s: lib.gs_b200_blobs_batch(
            P["src"], w, h, n, P["labels"], P["blobs"], P["counts"], nb, s), want)
    if sym == "gs_b200_blob_corners":
        def want(ins, bf):
            c = np.zeros((4, 2), np.uint32)
            O.gso_blob_corners(L.ptr(ins["src"][0]), w, h, L.ptr(ins["labels"][0]), L.ptr(ins["blob"]), L.ptr(c))
            return {"corners": c[None]}
        return Spec(dict(one, labels=2 * px, blob=32), {"corners": 32}, lambda P, n, s: lib.gs_b200_blob_corners(
            P["src"], w, h, P["labels"], P["blob"], P["corners"], s), want)
    if sym == "gs_b200_perspective_correct_batch":
        dw, dh, per_frame = g["dw"], g["dh"], g.get("per_frame", 1)
        q_host, q0 = host_quad(), host_quad()          # per_frame = 0: the corners every frame takes (mutate: q_host)

        def want(ins, bf):
            out = []
            for i, a in enumerate(ins["src"]):
                d = np.empty((dh, dw), np.uint8)
                q = np.ascontiguousarray(ins["corners"][i]) if per_frame else q0
                O.gso_perspective_correct(L.ptr(d), dw, dh, L.ptr(a), w, h, L.ptr(q))
                out.append(d)
            return {"dst": np.stack(out)}
        if per_frame:
            return Spec(dict(one, corners=32), {"dst": dw * dh}, lambda P, n, s: lib.gs_b200_perspective_correct_batch(
                P["dst"], dw, dh, P["src"], w, h, n, P["corners"], 1, s), want)

        def mutate():
            q_host[:] = 0
        return Spec(one, {"dst": dw * dh}, lambda P, n, s: lib.gs_b200_perspective_correct_batch(
            P["dst"], dw, dh, P["src"], w, h, n, q_host.ctypes.data, 0, s), want, mutate=mutate)
    if sym in ("gs_b200_fast_batch", "gs_b200_orb_extract_batch"):
        orb, nk, t, f = "orb" in sym, g["nkps"], g["t"], getattr(lib, sym)

        def want(ins, bf):
            sms, lists = [], []
            for a, sm in zip(ins["src"], ins["score"]):
                sm = np.array(sm, np.uint8).reshape(h, w)
                lists.append(L.o_orb(O, a, sm, nk, t) if orb else L.o_fast(O, a, sm, nk, t))
                sms.append(sm)
            return {"score": np.stack(sms), "kps": records(lists, bf["kps"]), "counts": counts(lists)}
        return Spec({"src": px, "score": px}, {"score": px, "kps": 48 * nk, "counts": 4}, lambda P, n, s: f(
            P["src"], w, h, n, P["score"], P["kps"], P["counts"], nk, t, s), want)
    if sym == "gs_b200_match_orb_batch":
        s1, s2, mm = g["s1"], g["s2"], g["mm"]
        md = {"max_distance": 60.0}

        def want(ins, bf):
            lists = [L.o_match(O, a[:c1], b[:c2], mm, 60.0) for a, c1, b, c2 in
                     zip(ins["kps1"], ins["n1"].reshape(-1), ins["kps2"], ins["n2"].reshape(-1))]
            return {"matches": records(lists, bf["matches"]), "counts": counts(lists)}

        def mutate():
            md["max_distance"] = 1.0
        return Spec({"kps1": 48 * s1, "n1": 4, "kps2": 48 * s2, "n2": 4}, {"matches": 12 * mm, "counts": 4},
                    lambda P, n, s: lib.gs_b200_match_orb_batch(P["kps1"], P["n1"], s1, P["kps2"], P["n2"], s2, n,
                                                                P["matches"], P["counts"], mm, md["max_distance"], s),
                    want, mutate=mutate)
    if sym == "gs_b200_lbp_detect_batch":
        # the cascade the call reads, and the one expect() reads: mutate() changes the first only
        cas = g["cascade"] if "cascade" in g else gb.load_cascade()
        cas0 = g["cascade"] if "cascade" in g else gb.load_cascade()
        mr = g["mr"]
        env = {"GS_B200_LBP_BIG": g["big"]} if "big" in g else {}
        if "chunk" in g:
            env["GS_B200_LBP_CHUNK_FRAMES"] = g["chunk"]

        def want(ins, bf):
            lists = [L.o_detect(O, cas0, ii, mr, *LBP) for ii in ins["ii"]]
            return {"rects": records(lists, bf["rects"]), "counts": counts(lists)}

        def mutate():
            cas.arrays["stage_threshold"][:] = 1e9
        return Spec({"ii": 4 * px}, {"rects": 16 * mr, "counts": 4}, lambda P, n, s: lib.gs_b200_lbp_detect_batch(
            cas.ptr, P["ii"], w, h, n, P["rects"], P["counts"], mr, *LBP, s), want, mutate=mutate, env=env)
    if sym == "gs_b200_crop_resize_batch":
        from grayskull_b200._lib import Rect
        dw, dh, roi, mode = g["dw"], g["dh"], g["roi"], g.get("mode", 1)
        return Spec(one, {"dst": dw * dh}, lambda P, n, s: lib.gs_b200_crop_resize_batch(
            P["dst"], dw, dh, P["src"], w, h, n, Rect(*roi), mode, s),
            lambda ins, bf: {"dst": _each(lambda a: L.composition(O, a, roi, dw, dh, mode), ins["src"])})
    if sym == "gs_b200_rois_resize_batch":
        dw, dh, mr, mode = g["dw"], g["dh"], g["mr"], g.get("mode", 1)

        def want(ins, bf):
            out = bf["dst"].reshape(-1, mr, dh, dw).copy()
            for i, (a, rs, c) in enumerate(zip(ins["src"], ins["rects"], ins["rcounts"].reshape(-1))):
                for j in range(int(c)):
                    out[i, j] = L.composition(O, a, tuple(rs[j]), dw, dh, mode)
            return {"dst": out}
        return Spec(dict(one, rects=16 * mr, rcounts=4), {"dst": mr * dw * dh}, lambda P, n, s: lib.gs_b200_rois_resize_batch(
            P["dst"], dw, dh, P["src"], w, h, n, P["rects"], P["rcounts"], mr, mode, s), want)
    if sym == "gs_b200_orb_pyramid_batch":
        nk, t, lv = g["nkps"], g["t"], g["levels"]
        sizes = [a * b for a, b in L.layout(w, h, lv)[0]]

        def want(ins, bf):
            k = len(ins["src"])
            kl, pyr, maps = L.pyramid_expected(O, ins["src"], nk, t, lv, flat(ins["score"], k))
            return {"pyr": unflat(pyr, sizes[1:], k), "score": unflat(maps, sizes, k), "kps": records(kl, bf["kps"]),
                    "counts": counts(kl)}
        return Spec({"src": px, "score": sizes}, {"pyr": sizes[1:], "score": sizes, "kps": 48 * nk, "counts": 4},
                    lambda P, n, s: lib.gs_b200_orb_pyramid_batch(P["src"], w, h, n, lv, P["pyr"], P["score"], P["kps"],
                                                                  P["counts"], nk, t, s), want)
    raise KeyError(sym)


# ---- the default inputs ---------------------------------------------------------------------------------------------
def _frames(w, h, k, seed):
    """gpu-harness frames; another seed than 1 reverses their kinds, so no frame of it equals the real one"""
    from _gpu import frames
    return frames(w, h, k, 1) if seed == 1 else np.ascontiguousarray(frames(w, h, k, 100 + seed)[::-1])


def lena():
    return np.load(os.path.join(L.ROOT, "tests", "golden", "lena_golden.npz"))["lena"]      # 128 x 128, faces found


def inputs(sym, g, k, seed):
    """{buffer: k frames} for spec(sym, g)"""
    from _gpu import frames
    w, h = g.get("w"), g.get("h")
    if sym == "gs_b200_threshold_each_batch":
        return {"src": _frames(w, h, k, seed), "thresh": np.random.default_rng(seed).integers(0, 256, k).astype(np.uint8)}
    if sym == "gs_b200_match_template_batch":
        fr = _frames(w, h, k, seed)
        return {"src": fr, "tmpl": np.ascontiguousarray(fr[1, 5 + seed:5 + seed + g["th"], 10 + seed:10 + seed + g["tw"]])}
    if sym == "gs_b200_find_best_match_batch":
        rng = np.random.default_rng(w * h + seed)
        return {"res": (rng.integers(0, 250, (k, w * h)) * (rng.random((k, w * h)) < 0.5)).astype(np.uint8)}
    if sym == "gs_b200_blobs_batch":
        return {"src": np.stack([L.binary_like(w, h, 50 * seed + i) for i in range(k)])}
    if sym == "gs_b200_blob_corners":
        a = L.binary_like(w, h, 7 + seed)
        labels, blobs = o_blobs(L.oracle(), a, 300)
        j = int(np.argmax(blobs["area"]))
        return {"src": a[None], "labels": labels[None], "blob": np.ascontiguousarray(blobs[j:j + 1])}
    if sym == "gs_b200_perspective_correct_batch":
        fr = _frames(w, h, k, seed)
        if not g.get("per_frame", 1):
            return {"src": fr}
        return {"src": fr, "corners": np.random.default_rng(5 + seed).integers(0, 140, (k, 4, 2)).astype(np.uint32)}
    if sym in ("gs_b200_fast_batch", "gs_b200_orb_extract_batch"):
        fr = _frames(w, h, k, seed)
        fr[seed % k] = L.natural_like(w, h, 90 + seed)                 # corners in every batch
        return {"src": fr, "score": np.full(fr.shape, 0 if "orb" in sym else POISON, np.uint8)}
    if sym == "gs_b200_match_orb_batch":
        sizes = ((120, 90), (7, 0), (130, 61), (40, 75))
        rng = np.random.default_rng(16 + seed)
        sets = [L.desc_sets(rng, *sizes[(i + seed) % 4]) for i in range(k)]
        k1, k2 = np.zeros((k, g["s1"]), L.KP_DTYPE), np.zeros((k, g["s2"]), L.KP_DTYPE)
        for i, (a, b) in enumerate(sets):
            k1[i, :len(a)], k2[i, :len(b)] = a, b
        return {"kps1": k1, "n1": counts([a for a, _ in sets]), "kps2": k2, "n2": counts([b for _, b in sets])}
    if sym == "gs_b200_lbp_detect_batch":
        fr = [np.pad(np.roll(lena(), 4 * (i + seed), axis=1), ((0, h - 128), (0, w - 128)), mode="edge")
              if (i + seed) % 2 else L.natural_like(w, h, 40 + i + 10 * seed) for i in range(k)]
        return {"ii": np.stack([L.o_integral(L.oracle(), f) for f in fr])}
    if sym == "gs_b200_crop_resize_batch":
        return {"src": frames(w, h, k, 40 + seed)}
    if sym == "gs_b200_rois_resize_batch":
        mr, dw, dh = g["mr"], g["dw"], g["dh"]
        rects = L.regions(np.random.default_rng(g.get("mode", 1)), k, mr, w, h, dw, dh, invalid=False)
        rects[:, 0] = (5, 6, dw, dh)                                    # a copy slot in each frame
        return {"src": frames(w, h, k, 40 + seed), "rects": rects, "rcounts": np.array([mr, 2, 4][:k], np.uint32)}
    if sym == "gs_b200_orb_pyramid_batch":
        sizes = [a * b for a, b in L.layout(w, h, g["levels"])[0]]
        maps = np.random.default_rng(seed).integers(0, 256, sum(sizes) * k, dtype=np.uint8)
        return {"src": frames(w, h, k, 40 + seed), "score": unflat(maps, sizes, k)}
    return {"src": _frames(w, h, k, seed)}
