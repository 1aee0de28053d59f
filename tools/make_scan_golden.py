#!/usr/bin/env python
"""Generate tests/golden/scan_<name>_golden.npz for name in document, receipt: the reference's own scanner images and
what its CLI's scan verb makes of them (the reference Makefile's `nanomagick scan testdata/document.pgm ...` and
`... receipt.pgm` lines).  The verb runs as upstream builds it (oracle/_ref/nanomagick_cpu, made by oracle/Makefile
from an upstream checkout named by GS_REFERENCE); the corners come from the unmodified reference header compiled as a
library (oracle/_ref/libgs_ref.so).  The GPU machines have no reference checkout, so these fixtures are committed.

  frame          the input frame, (h, w) uint8
  scan_sha256    SHA-256 of the verb's output file (P5, 800 x 1000), 32 uint8: a byte-for-byte check at a fraction
                 of the 800 KB the output itself would add to the fixture
  scan_size      that file's length in bytes
  corners        (4, 2) uint32: the verb's corners (blur 1, Otsu + 10, gs_blobs with 1000 records, the largest with
                 the first on ties, gs_blob_corners), in tl, tr, br, bl order
"""
import ctypes as C
import hashlib
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _libs as L  # noqa: E402

REF_TREE = os.environ.get("GS_REFERENCE", "/root/reference")
CLI = os.path.join(ROOT, "oracle", "_ref", "nanomagick_cpu")
OUT = os.path.join(ROOT, "tests", "golden", "scan_%s_golden.npz")


def read_pgm(path):
    """a binary P5 file whose header is three whitespace-separated tokens on their own lines, as these files are"""
    with open(path, "rb") as f:
        assert f.readline().strip() == b"P5"
        w, h = map(int, f.readline().split())
        assert int(f.readline()) == 255
        return np.frombuffer(f.read(w * h), np.uint8).reshape(h, w).copy()


def ref_corners(a):
    """nanomagick.c:186-202 on the reference library: the corners the verb warps from"""
    R = L.ref()
    R.gs_blur.argtypes = [L.Image, L.Image, C.c_uint]
    h, w = a.shape
    t = np.zeros_like(a)
    R.gs_blur(L.img(t), L.img(a), 1)
    R.gs_threshold(L.img(t), (int(R.gs_otsu_threshold(L.img(t))) + 10) & 255)
    lab = np.zeros((h, w), np.uint16)
    b = np.zeros(1000, L.BLOB_DTYPE)
    k = R.gs_blobs(L.img(t), L.ptr(lab), L.ptr(b), 1000)
    largest = 0
    for i in range(1, k):
        if b[i]["area"] > b[largest]["area"]:
            largest = i
    c = np.zeros((4, 2), np.uint32)
    R.gs_blob_corners(L.img(t), L.ptr(lab), L.ptr(b[largest:largest + 1]), L.ptr(c))
    return c


def main():
    if not os.path.exists(CLI) or not L.have_ref():
        sys.exit("oracle/_ref is incomplete: run `make -C oracle ref` with GS_REFERENCE set to an upstream checkout")
    with tempfile.TemporaryDirectory() as d:
        for name in ("document", "receipt"):
            src = os.path.join(REF_TREE, "testdata", name + ".pgm")
            dst = os.path.join(d, name + ".pgm")
            subprocess.run([CLI, "scan", src, dst], check=True)
            out = open(dst, "rb").read()
            a = read_pgm(src)
            c = ref_corners(a)
            np.savez_compressed(OUT % name, frame=a, scan_sha256=np.frombuffer(hashlib.sha256(out).digest(), np.uint8),
                                scan_size=np.uint64(len(out)), corners=c)
            print("%s: %dx%d, output md5 %s, corners %s -> %s" % (name, a.shape[1], a.shape[0],
                  hashlib.md5(out).hexdigest(), c.tolist(), OUT % name))


if __name__ == "__main__":
    main()
