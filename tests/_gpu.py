"""The device side of the test suite: fixtures, device buffers and the kernel witness.  Test modules import what they
use by name, fixtures included (`from _gpu import G, lib, witness  # noqa: F401`).

  * fixtures: `lib` (the ctypes library on device 0), `G` (grayskull_b200.api), `O` (the oracle), `witness` (one
    probe: whether torch.profiler sees the library's launches at all);
  * dev(), stream(), Region (a view into a guarded device allocation), frames() (a seeded batch);
  * traced() runs one call under torch.profiler and returns the kernels it launched; witnessed() checks a case's
    kernels among them."""
import ctypes as C
import os

import numpy as np
import pytest

import _libs as L
from _libs import kernel_id

# Have kineto tear CUPTI down at the end of every profiler session, so that each session starts from a fresh CUPTI.
# Without it, once a process has run some sessions, later ones intermittently deliver no kernel records or only their
# last kernels (on an H100: 3 of 3 witness probes and 443 sessions of one run of the GPU suite, with every output
# bit-exact); with it, every session of the same run recorded all its kernels.  Set at import, before the first
# session of the process: every module that traces imports this one, and every session runs through traced().
os.environ.setdefault("TEARDOWN_CUPTI", "1")


def _on_device():
    import torch
    import grayskull_b200 as g
    assert torch.cuda.is_available()
    g.lib().gs_b200_set_device(0)
    return g.lib()


@pytest.fixture(scope="module")
def lib():
    return _on_device()


@pytest.fixture(scope="module")
def G():
    from grayskull_b200 import api
    _on_device()
    return api


@pytest.fixture(scope="module")
def O():
    return L.oracle()


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class Region:
    """`nbytes` at byte `off` of a 256-byte aligned device allocation of nbytes + 32 bytes.  Everything starts as a
    seeded byte pattern (then `data`, if given, in the view); read() checks that the bytes outside the view kept it."""

    def __init__(self, nbytes, off=0, data=None, seed=0):
        import torch
        self.off, self.nbytes = off, nbytes
        self.host = np.random.default_rng(seed * 7919 + nbytes + off).integers(0, 256, nbytes + 32, dtype=np.uint8)
        if data is not None:
            b = np.frombuffer(np.ascontiguousarray(data).tobytes(), np.uint8)
            assert b.size == nbytes
            self.host[off:off + nbytes] = b
        self.t = torch.from_numpy(self.host.copy()).cuda()
        assert self.t.data_ptr() % 256 == 0
        self.ptr = self.t.data_ptr() + off

    def before(self):
        return self.host[self.off:self.off + self.nbytes].copy()

    def read(self, what):
        got = self.t.cpu().numpy()
        o, e = self.off, self.off + self.nbytes
        assert np.array_equal(got[:o], self.host[:o]) and np.array_equal(got[e:], self.host[e:]), \
            "%s: bytes outside the view changed" % what
        return got[o:e].copy()


def frames(w, h, n, seed):
    """random, natural_like and saturated (255) frames in turn"""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        out.append([rng.integers(0, 256, (h, w), dtype=np.uint8), L.natural_like(w, h, seed + i),
                    np.full((h, w), 255, np.uint8)][i % 3])
    return np.stack(out)


def traced(fn):
    """run fn (a C call returning its status) under torch.profiler with CUDA activity -> (status, launched kernels)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        rc = fn()
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if "k_" in e.name}
    mangled = sorted(nm for nm in names if nm.startswith("_Z"))
    names = (names - set(mangled)) | set(L.demangle(mangled))
    return rc, {kernel_id(nm) for nm in names if "gsb::" in nm}


@pytest.fixture(scope="module")
def witness(lib):
    """whether kineto sees the library's launches at all: one probe launch"""
    import torch
    src = torch.zeros((1, 40, 272), dtype=torch.uint8, device="cuda")
    out = torch.empty_like(src)
    rc, seen = traced(lambda: lib.gs_b200_blur_batch(out.data_ptr(), src.data_ptr(), 272, 40, 1, 5, stream()))
    assert rc == 0
    print("\nwitness probe: %s" % (sorted(seen) or "no kernel events recorded"))
    return bool(seen)


def witnessed(witness, run, kernels, what):
    """run() makes the case's calls, asserts that every output is bit-exact and returns the launched kernels; each of
    `kernels` must be among them.  The profiler sometimes loses device records, a whole session or single kernels of
    one, so while one of `kernels` is missing run() runs again, checked again, up to 3 runs in all.  Which kernel a call
    launches is a function of its host-visible inputs, so a case that takes another kernel misses it on every run."""
    for runs in range(1, 4):
        seen = run()
        if not witness or all(kernel_id(k) in seen for k in kernels):
            break
    print("\n%s: launched %s%s" % (what, " ".join(sorted(seen)), " (run %d)" % runs if runs > 1 else ""))
    if not witness:
        pytest.skip("parity holds; kineto recorded no kernel events for the probe launch, so the path is not witnessed")
    missing = [k for k in kernels if kernel_id(k) not in seen]
    assert not missing, "expected %s, launched %s" % (missing, sorted(seen))
