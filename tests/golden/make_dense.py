#!/usr/bin/env python
"""Regenerate tests/golden/dense/ and tests/golden/dense.json: baseline JPEGs of white noise, as dense as a JPEG gets, and
what the UNMODIFIED reference CLI makes of them.

Photos need well under 64 bytes of range-coder stream per 8x8 block; noise coded at quality 100 needs up to about 90.
Every segment of every file here has a reference stream longer than the stream slot a segment starts with in the library
(align_up(64 * blocks + 4096, 256) bytes, plan_batch in lep_plan.cuh): the library has to grow the stream to code these
files at all.  The script asserts that and records the margin of each segment.

Run where oracle/_ref/lepton exists (oracle/Makefile builds it from the reference tree):
    python tests/golden/make_dense.py
The jpegwriter files are deterministic: a second run reproduces them byte for byte.  pillow_noise_q100.jpg is the
ordinary-user case, white noise saved by Pillow at quality 100; it is committed as bytes and written again only when
missing, since another Pillow (libjpeg) version may write other bytes (dense.json records the version that wrote it).
dense.json holds per file the fields of extremes.json (make_extremes.py): path, jpg_md5, rc, exit_name, lep_md5,
plane_sha256, back_md5, status_want; for the -minencodethreads records source, flags, lep_md5, nseg; and for every .lep
  seg_blocks          blocks coded by each thread-segment
  seg_stream_bytes    length of each segment's stream in the reference's .lep
  seg_slot_bytes      the library's initial stream slot of that segment
  min_margin          min(stream / slot) over the segments (> 1)
"""
import hashlib
import io
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from jpegwriter import geometry, write_baseline  # noqa: E402
from make_extremes import LEPTON, run_reference  # noqa: E402

OUTDIR = os.path.join(HERE, "dense")
OUT = os.path.join(HERE, "dense.json")
PILLOW_FILE = "pillow_noise_q100"


def md5(b):
    return hashlib.md5(b).hexdigest()


def noise_planes(rng, w, h, sampling, kind, amp, dc_lim=600):
    """Zig-zag planes of iid AC noise (every position) and a DC random walk within +-dc_lim."""
    _, _, grid, _ = geometry(w, h, sampling)
    planes = []
    for bx, by in grid:
        if kind == "gauss":
            p = np.clip(np.rint(rng.normal(0, amp, size=(by, bx, 64))), -1023, 1023).astype(np.int64)
        else:
            p = rng.integers(-amp, amp + 1, size=(by, bx, 64)).astype(np.int64)
        dc = np.cumsum(rng.integers(-40, 41, size=by * bx))
        p[..., 0] = np.clip(dc, -dc_lim, dc_lim).reshape(by, bx)
        planes.append(p)
    return planes


def corpus():
    """-> [(name, jpeg bytes, extra -minencodethreads values)].  Each jpegwriter file has its own seed."""
    files = []

    def rng(k):
        return np.random.default_rng(20261016 + k)

    # Gaussian sigma 74 at every AC position, AC quantisers 1: just over the slot (the capacity edge)
    files.append(("grey_gauss74", write_baseline(noise_planes(rng(1), 256, 256, [(1, 1)], "gauss", 74), 256, 256, [(1, 1)],
                                                 [[4] + [1] * 63]), []))
    # uniform +-1023: far over
    files.append(("grey_uniform1023", write_baseline(noise_planes(rng(2), 192, 192, [(1, 1)], "uniform", 1023), 192, 192,
                                                     [(1, 1)], [[8] + [1] * 63]), []))
    # 4:2:0 colour, uniform +-1023, and an 8-segment record of it
    s420 = [(2, 2), (1, 1), (1, 1)]
    files.append(("color420_uniform", write_baseline(noise_planes(rng(3), 256, 256, s420, "uniform", 1023), 256, 256, s420,
                                                     [[8] + [1] * 63, [8] + [1] * 63]), [8]))
    # 4:4:4 colour, odd size (partial MCUs at the right and bottom edges), restart interval of 7 MCUs
    s444 = [(1, 1)] * 3
    files.append(("color444_odd_rst", write_baseline(noise_planes(rng(4), 139, 131, s444, "uniform", 511), 139, 131, s444,
                                                     [[8] + [1] * 63, [8] + [1] * 63], restart=7), []))
    # white noise pixels saved by Pillow at quality 100 (committed bytes; see the module docstring)
    path = os.path.join(OUTDIR, PILLOW_FILE + ".jpg")
    if os.path.exists(path):
        jpg = open(path, "rb").read()
    else:
        from PIL import Image
        px = np.random.default_rng(20261016).integers(0, 256, size=(256, 256), dtype=np.uint8)
        b = io.BytesIO()
        Image.fromarray(px, "L").save(b, "JPEG", quality=100)
        jpg = b.getvalue()
    files.append((PILLOW_FILE, jpg, []))
    return files


def segment_blocks(lf):
    """Blocks of every thread-segment of a .lep, counted like segment_blocks of lep_plan.cuh."""
    import lepfmt
    f = lf.frame
    tbcv, _ = lepfmt.truncation(lf)
    v0 = max(f.bcv[0] // f.mcuv, 1)
    out = []
    hs = lf.handoffs
    for i, h in enumerate(hs):
        last = i == len(hs) - 1
        min_y = h.luma_y_start
        max_y = f.bcv[0] if last else hs[i + 1].luma_y_start
        n = 0
        for c in range(f.ncmp):
            mult = f.bcv[c] // f.mcuv
            y0 = (min_y // v0) * mult
            y1 = tbcv[c] if last else ((max_y + v0 - 1) // v0) * mult
            y1 = min(y1, tbcv[c])
            if y1 > y0:
                n += (y1 - y0) * f.bch[c]
        out.append(n)
    return out


def stream_record(lep):
    """Per-segment blocks, reference stream bytes and the library's initial slot; asserts every stream outgrows its slot."""
    import lepfmt
    lf = lepfmt.parse_container(lep)
    streams = lepfmt.demux(lf.payload, lf.version)[:lf.nseg]
    nb = segment_blocks(lf)
    slots = [(n * 64 + 4096 + 255) // 256 * 256 for n in nb]
    lens = [len(s) for s in streams]
    assert all(n > s for n, s in zip(lens, slots)), (lens, slots)
    return {"seg_blocks": nb, "seg_stream_bytes": lens, "seg_slot_bytes": slots,
            "min_margin": round(min(n / s for n, s in zip(lens, slots)), 4)}


def main():
    import lepfmt
    import PIL
    from helpers import plane_hashes
    os.makedirs(OUTDIR, exist_ok=True)
    record = {}
    with tempfile.TemporaryDirectory() as td:
        for name, jpg, threads in corpus():
            src = os.path.join(OUTDIR, name + ".jpg")
            with open(src, "wb") as f:
                f.write(jpg)
            rc, exit_name, lep = run_reference(src, os.path.join(td, "o.lep"))
            assert rc == 0 and not exit_name and lep, (name, rc, exit_name)
            with open(os.path.join(OUTDIR, name + ".lep"), "wb") as f:
                f.write(lep)
            e = {"path": "dense/%s.jpg" % name, "jpg_md5": md5(jpg), "rc": rc, "exit_name": exit_name, "lep_md5": md5(lep)}
            ujg = os.path.join(td, "o.ujg")
            assert os.system("%s -unjailed -ujg -skipverify %s %s > /dev/null 2>&1" % (LEPTON, src, ujg)) == 0
            e["plane_sha256"] = plane_hashes(lepfmt.parse_ujg_planes(open(ujg, "rb").read())[1])
            back = os.path.join(td, "b.jpg")
            assert os.system("%s -unjailed %s %s > /dev/null 2>&1" % (LEPTON, os.path.join(OUTDIR, name + ".lep"), back)) == 0
            e["back_md5"] = md5(open(back, "rb").read())
            e["status_want"] = 0
            e.update(stream_record(lep))
            if name == PILLOW_FILE:
                e["pillow_version"] = PIL.__version__
            record[name + ".jpg"] = e
            print(name, len(jpg), len(lep), e["seg_stream_bytes"], e["seg_slot_bytes"], e["min_margin"], flush=True)
            for t in threads:
                flags = ["-minencodethreads=%d" % t]
                rc, exit_name, lep = run_reference(src, os.path.join(td, "t.lep"), flags)
                assert rc == 0 and not exit_name and lep, (name, t)
                lname = "%s_t%d.lep" % (name, t)
                with open(os.path.join(OUTDIR, lname), "wb") as f:
                    f.write(lep)
                r = {"path": "dense/" + lname, "source": name + ".jpg", "flags": flags, "lep_md5": md5(lep),
                     "nseg": lepfmt.parse_container(lep).nseg}
                r.update(stream_record(lep))
                record[lname] = r
                print(" ", lname, len(lep), r["nseg"], r["min_margin"], flush=True)
    with open(OUT, "w") as f:
        json.dump(record, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
