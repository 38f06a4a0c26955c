"""Diagnostic helper (not a test): build sequential JPEGs whose scans are NOT interleaved (one scan per component)
from PIL baseline files, so that the reference's "sequential, non-interleaved" branches (jpgcoder.cc:3041-3089,
recode :3512-3545) can be exercised against the reference CLI in the build container.

usage: python tests/tools_gen_nonint.py OUTDIR
"""
import io
import os
import struct
import sys

import numpy as np
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from lepton_b200 import HostJpeg  # noqa: E402
from jpegwriter import BitWriter, canonical_codes, put_block  # noqa: E402

ZZ2AL = [49, 50, 57, 58, 0, 51, 52, 1, 2, 59, 60, 3, 4, 5, 53, 54, 6, 7, 8, 9, 61, 62, 10, 11, 12, 13, 14, 55, 56, 15, 16,
         17, 18, 19, 20, 63, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32, 33, 34, 35, 36, 37, 38, 39, 40, 41, 42, 43,
         44, 45, 46, 47, 48]


def segments(data):
    pos = 2
    segs = []
    while True:
        assert data[pos] == 0xFF
        t = data[pos + 1]
        ln = 2 + struct.unpack(">H", data[pos + 2:pos + 4])[0]
        segs.append((t, data[pos:pos + ln]))
        pos += ln
        if t == 0xDA:
            break
    return segs


def dht_tables(segs):
    tabs = {}
    for t, s in segs:
        if t != 0xC4:
            continue
        p = 4
        while p < len(s):
            tc, th = s[p] >> 4, s[p] & 15
            bits = list(s[p + 1:p + 17])
            n = sum(bits)
            vals = list(s[p + 17:p + 17 + n])
            p += 17 + n
            tabs[(tc, th)] = canonical_codes(bits, vals)
    return tabs


def make(w, h, sub, q, rst, name):
    y, x = np.mgrid[0:h, 0:w]
    rng = np.random.default_rng(w * h + sub)
    a = np.clip((128 + 60 * np.sin(x / 13.0) + 50 * np.cos(y / 9.0))[..., None] + rng.normal(0, 20, (h, w, 3)), 0, 255)
    b = io.BytesIO()
    Image.fromarray(a.astype(np.uint8)).save(b, "JPEG", quality=q, subsampling=sub)
    data = b.getvalue()
    hj = HostJpeg(data)
    assert hj.status == 0
    img = hj.coef_image()
    segs = segments(data)
    tabs = dht_tables(segs)
    sof = [s for t, s in segs if t == 0xC0][0]
    nc = sof[9]
    comps = [(sof[10 + 3 * i], sof[11 + 3 * i] >> 4, sof[11 + 3 * i] & 15) for i in range(nc)]
    sos = [s for t, s in segs if t == 0xDA][0]
    tdta = {sos[5 + 2 * i]: (sos[6 + 2 * i] >> 4, sos[6 + 2 * i] & 15) for i in range(nc)}
    out = bytearray(b"\xff\xd8")
    for t, s in segs:
        if t != 0xDA:
            out += s
    if rst:
        out += b"\xff\xdd\x00\x04" + struct.pack(">H", rst)
    hm = max(c[1] for c in comps)
    vm = max(c[2] for c in comps)
    mcuh = -(-w // (8 * hm))
    for ci, (cid, H, V) in enumerate(comps):
        td, ta = tdta[cid]
        out += b"\xff\xda" + struct.pack(">HB", 8, 1) + bytes([cid, (td << 4) | ta, 0, 63, 0])
        bch = mcuh * H
        nch = -(-(-(-w * H // hm)) // 8)
        ncv = -(-(-(-h * V // vm)) // 8)
        P = np.asarray(img.planes[ci]).reshape(-1, 64)
        bw = BitWriter()
        last = 0
        cnt = 0
        nrst = 0
        dc, ac = tabs[(0, td)], tabs[(1, ta)]
        for by in range(ncv):
            for bx in range(nch):
                if rst and cnt and cnt % rst == 0:
                    bw.pad()
                    bw.out += bytes([0xFF, 0xD0 + (nrst & 7)])
                    nrst += 1
                    last = 0
                last = put_block(bw, [int(v) for v in P[by * bch + bx][ZZ2AL]], last, dc, ac)
                cnt += 1
        bw.pad()
        out += bw.out
    out += b"\xff\xd9"
    open(name, "wb").write(out)
    Image.open(name).load()


if __name__ == "__main__":
    outdir = sys.argv[1]
    os.makedirs(outdir, exist_ok=True)
    k = 0
    for (w, h) in [(64, 48), (45, 37), (200, 120)]:
        for sub in [0, 1, 2]:
            for rst in [0, 5]:
                make(w, h, sub, 85, rst, os.path.join(outdir, f"n_{w}x{h}_s{sub}_r{rst}.jpg"))
                k += 1
    print(k, "files")
