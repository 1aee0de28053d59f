"""Time gs_b200_erode_n_batch / gs_b200_dilate_n_batch (one call for N passes of the 3x3 op) against N ping-ponged
gs_b200_erode_batch / gs_b200_dilate_batch calls, on one GPU, in one run.

    python tools/morph_bench.py [--reps 3] [--quick] [--json out.jsonl]

Shapes: 64 x 4096^2 and 256 x 1920x1080 (the TMA path for 2 <= N <= 16, composed TMA passes for N <= 48) and
64 x 4092x4096 (width not a multiple of 16: the row/column pass path).  N covers both sides of the TMA path's bound of 16.  Before any timing the two
methods' outputs are compared on the device at every timed shape and N.  Times are CUDA-event medians of --reps
alternated repeats, each repeat covering several calls after a warm-up; spread = (max - min) / median.  Algorithmic
bytes: 2 B/px per 3x3 call and per TMA launch, 4 B/px per row/column-pass call (src read, workspace written and
read, dst written).  A device-to-device copy of the same batch is the practical bandwidth ceiling."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DATASHEET_BPS = 3.35e12   # H100 SXM HBM3, data sheet (700 W card)
NS = [1, 2, 3, 5, 9, 10, 16, 17, 31, 64, 255]
SHAPES = [(64, 4096, 4096), (256, 1080, 1920), (64, 4096, 4092)]   # (n, h, w)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")])) if r.returncode == 0 else {}


def timed(fn, inner):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(inner):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / inner / 1e3


def stats(ts):
    ts = sorted(ts)
    med = ts[len(ts) // 2]
    return med, (ts[-1] - ts[0]) / med


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--quick", action="store_true", help="small shapes, for a rehearsal of the script")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    import grayskull_b200 as g
    from grayskull_b200 import api
    assert torch.cuda.is_available(), "morph_bench needs a CUDA device"
    g.lib().gs_b200_set_device(0)
    lib = g.lib()
    info = card()
    print(json.dumps({"card": info}), flush=True)
    rows = []
    shapes = [(2, 256, 512), (2, 256, 508)] if args.quick else SHAPES
    for n, h, w in shapes:
        gen = torch.Generator(device="cuda").manual_seed(n + h + w)
        src = torch.randint(0, 256, (n, h, w), dtype=torch.uint8, device="cuda", generator=gen)
        out, t0, t1 = torch.empty_like(src), torch.empty_like(src), torch.empty_like(src)
        px = n * h * w
        tma = bool(lib.gs_b200_uses_tma(w, h, src.data_ptr()))
        copy = [timed(lambda: out.copy_(src), 10) for _ in range(args.reps + 1)][1:]
        cmed, cspr = stats(copy)
        print(json.dumps({"shape": [n, h, w], "tma_geometry": tma, "copy_ms": cmed * 1e3, "copy_spread": cspr,
                          "copy_TBps": 2 * px / cmed / 1e12}), flush=True)

        def chain(ops):
            """ops applied one after another, ping-ponging between t0 and t1 (the N-call baseline)"""
            a = src
            for i, op in enumerate(ops):
                b = t0 if i % 2 == 0 else t1
                op(a, out=b)
                a = b
            return a

        def old(op, k):
            return lambda: chain([op] * k)

        for name, new_fn, old_op in (("erode", api.erode_n_batch, api.erode_batch),
                                     ("dilate", api.dilate_n_batch, api.dilate_batch)):
            for N in NS:
                res = old(old_op, N)()
                assert torch.equal(new_fn(src, N, out=out), res), (name, n, h, w, N)   # before any timing
                fn_new, fn_old = (lambda: new_fn(src, N, out=out)), old(old_op, N)
                fn_new(), fn_old()
                tn, to = [], []
                for _ in range(args.reps):
                    tn.append(timed(fn_new, 5))
                    to.append(timed(fn_old, max(1, 20 // N)))
                (mn, sn), (mo, so) = stats(tn), stats(to)
                steps = -(-N // 16)                       # TMA launches when 17 <= N <= 48 are composed
                path = ("3x3" if N == 1 else "A" if tma and N <= 16 else "A x %d" % steps if tma and N <= 48 else "B")
                bytes_new = px * (2 if path in ("A", "3x3") else 2 * steps if path.startswith("A") else 4)
                r = {"shape": [n, h, w], "op": name, "N": N, "path": path, "one_call_ms": mn * 1e3, "spread": sn,
                     "n_calls_ms": mo * 1e3, "n_calls_spread": so, "speedup": mo / mn,
                     "alg_TBps": bytes_new / mn / 1e12, "of_datasheet": bytes_new / mn / DATASHEET_BPS,
                     "of_copy": (bytes_new / mn) / (2 * px / cmed)}
                rows.append(r)
                print(json.dumps(r), flush=True)
        # the reference Makefile's ArUco tail: dilate 9 -> erode 10, two calls against nineteen
        def tail_new():
            api.dilate_n_batch(src, 9, out=t0)
            api.erode_n_batch(t0, 10, out=out)

        def tail_old():
            return chain([api.dilate_batch] * 9 + [api.erode_batch] * 10)

        want = tail_old().clone()
        tail_new()
        assert torch.equal(out, want), ("tail", n, h, w)
        del want
        tn, to = [], []
        for _ in range(args.reps):
            tn.append(timed(tail_new, 3))
            to.append(timed(tail_old, 1))
        (mn, sn), (mo, so) = stats(tn), stats(to)
        r = {"shape": [n, h, w], "op": "dilate9_erode10", "two_calls_ms": mn * 1e3, "spread": sn,
             "nineteen_calls_ms": mo * 1e3, "nineteen_spread": so, "speedup": mo / mn}
        rows.append(r)
        print(json.dumps(r), flush=True)
        del src, out, t0, t1
        torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            f.write(json.dumps({"card": info}) + "\n")
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
