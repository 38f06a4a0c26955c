#!/usr/bin/env python
"""Regenerate tests/golden/geometry/ and tests/golden/geometry.json: baseline JPEGs with every sampling geometry the
reference accepts, and what the UNMODIFIED reference CLI makes of them.

The sampling factors of the components decide the MCU grid, how the rows of the components interleave in the coding
order (ImageDesc.mult, row_spec_from_index), the truncation bounds, the luma rows at which thread-segments split, the
row-buffer offsets of the range-coder kernels and the MCU walks of the Huffman kernels.  Photos are nearly always 4:2:0,
4:2:2 or 4:4:4 with 1x1 chroma; a lossless rotation or an unusual encoder gives the rest.  This corpus takes every class
of factors in {1, 2} for one and three components (GEOMETRIES) at four sizes each (sizes()):

  whole   a whole number of MCUs
  plus1   one pixel past an MCU in each direction, so that some components have nch < bch or ncv < bcv and others not
  col     one MCU column (width <= 8 * Hmax)
  odd     an odd number of MCUs across

plus restart intervals (DRI 1, and an interval that does not divide the MCU row) on six colour geometries, and files
tall enough that -minencodethreads=4 / =8 give 4 and 8 thread-segments.  Planes are photo-like (a smooth DC walk and
decaying low-frequency AC), with dense blocks and blocks holding category-11 magnitudes in the chroma planes, also at
the chroma borders; the Huffman tables give common symbols short codes, as photo encoders do, so that the sub-sequence
Huffman kernels synchronise within their iteration budget.

Run where oracle/_ref/lepton exists (oracle/Makefile builds it from the reference tree):
    python tests/golden/make_geometry.py
The output is deterministic: a second run reproduces every file byte for byte.  geometry.json holds per JPEG

  path, jpg_md5         the input, relative to tests/golden/
  cls                   the geometry class (CLASSES)
  sampling              (H, V) per component; width, height, restart (DRI interval in MCUs, 0 = none)
  mcuh, mcuv, bch, bcv  the MCU grid and the blocks of each component in it
  nch, ncv              the blocks of each component that hold image data
  rc / exit_name        as extremes.json (make_extremes.py): exit code and ExitCode name of `lepton -unjailed
                        -skipverify in.jpg out.lep`
  lep_md5               the .lep it wrote (accepted files; committed next to the JPEG)
  plane_sha256          sha256 of each coefficient plane of its `-ujg` dump (accepted files)
  back_md5              md5 of what the reference decodes that .lep to
  status_want           the status the library must report
and for the multi-segment records (NAME_tN.lep): source, flags, lep_md5, nseg, splits, back_md5.
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from jpegwriter import AC_SYMBOLS, DC_SYMBOLS, HuffTable, fit_lengths, geometry, write_baseline  # noqa: E402
from make_extremes import EXIT_CODES, LEPTON  # noqa: E402
from make_truncated import exit_name_of  # noqa: E402

OUTDIR = os.path.join(HERE, "geometry")
OUT = os.path.join(HERE, "geometry.json")

# (H, V) of Y / Cb / Cr, by class
GEOMETRIES = {
    "luma": {"y11": ((1, 1), (1, 1), (1, 1)), "y21": ((2, 1), (1, 1), (1, 1)), "y12": ((1, 2), (1, 1), (1, 1)),
             "y22": ((2, 2), (1, 1), (1, 1))},
    "alike": {"all22": ((2, 2),) * 3, "all21": ((2, 1),) * 3, "all12": ((1, 2),) * 3},
    "chroma_heavy": {"y11_c22": ((1, 1), (2, 2), (2, 2)), "y11_c21": ((1, 1), (2, 1), (2, 1)),
                     "y12_c21": ((1, 2), (2, 1), (2, 1)), "y21_c12": ((2, 1), (1, 2), (1, 2))},
    "cb_ne_cr": {"y22_cb11_cr21": ((2, 2), (1, 1), (2, 1)), "y22_cb12_cr11": ((2, 2), (1, 2), (1, 1)),
                 "y11_cb22_cr11": ((1, 1), (2, 2), (1, 1)), "y21_cb11_cr22": ((2, 1), (1, 1), (2, 2))},
    "grey": {"g11": ((1, 1),), "g21": ((2, 1),), "g12": ((1, 2),), "g22": ((2, 2),)},
}
CLASSES = sorted(GEOMETRIES)
# colour geometries that also get restart intervals (DRI 1 and 3, on a 4-MCU row), across the classes
RESTART = ["y12", "all21", "y11_c22", "y21_c12", "y22_cb12_cr11", "y21_cb11_cr22"]
# geometries that also get a tall file for -minencodethreads=4 / =8
TALL = ["y22", "y12", "all22", "y11_c22", "y12_c21", "y21_c12", "y11_cb22_cr11", "y22_cb11_cr21", "g21"]


def md5(b):
    return hashlib.md5(b).hexdigest()


def sizes(sampling):
    """-> [(size name, width, height)]: the four sizes of a geometry (module docstring)."""
    mw = 8 * max(h for h, _ in sampling)
    mh = 8 * max(v for _, v in sampling)
    return [("whole", 6 * mw, 4 * mh), ("plus1", 4 * mw + 1, 3 * mh + 1), ("col", mw - 3, 7 * mh + 5),
            ("odd", 5 * mw - 2, 3 * mh - 1)]


def photo_tables(rng):
    """DC and AC tables shaped like a photo encoder's: short codes for small categories, EOB and short runs, 16-bit
    codes for the rare symbols; the order within a length is shuffled per file."""
    dc = sorted(DC_SYMBOLS[:12], key=lambda s: (s, rng.random()))
    dct = HuffTable(fit_lengths([(s, 2 + i // 2) for i, s in enumerate(dc)]))
    ac = sorted(AC_SYMBOLS, key=lambda s: (0 if s == 0 else (s >> 4) + (s & 15) + (8 if s == 0xF0 else 0), rng.random()))
    act = HuffTable(fit_lengths([(s, 3 + i // 4) for i, s in enumerate(ac)]))
    return dct, act


def photo_planes(rng, w, h, sampling):
    """Photo-like planes over the whole MCU grid: a smooth DC walk, a few decaying low-frequency AC coefficients; in the
    chroma planes some dense blocks (every AC position set) and some with category-11 magnitudes, among them the
    corner blocks and the last column and row of the coded area."""
    _, _, grid, coded = geometry(w, h, sampling)
    planes = []
    for c, (bx, by) in enumerate(grid):
        n = by * bx
        p = np.zeros((n, 64), np.int64)
        nnz = 6 if c == 0 else 3
        pos = np.minimum(rng.geometric(0.18, size=(n, nnz)), 63)
        val = np.rint(rng.normal(0, 1, size=(n, nnz)) * 60 / np.sqrt(pos)).astype(np.int64)
        np.put_along_axis(p, pos, val, axis=1)
        p[:, 0] = np.clip(np.cumsum(rng.integers(-25, 26, size=n)), -700 if c else -900, 700 if c else 900)
        p = p.reshape(by, bx, 64)
        if c:
            nx, ny = coded[c]
            spots = {(0, 0), (ny - 1, nx - 1), (ny // 2, nx - 1), (ny - 1, nx // 2), (by - 1, bx - 1)}
            spots |= {(int(rng.integers(0, by)), int(rng.integers(0, bx))) for _ in range(max(1, n // 12))}
            for k, (y, x) in enumerate(sorted(spots)):
                if k % 2:
                    p[y, x, 1:] = rng.integers(-24, 25, size=63)                 # dense: categories up to 5 everywhere
                else:
                    at = rng.choice(np.arange(1, 64), size=3, replace=False)   # category 11 at three positions
                    p[y, x, at] = rng.integers(1024, 2048, size=3) * rng.choice([-1, 1], size=3)
        planes.append(p)
    return planes


def corpus():
    """-> [(name, cls, geometry name, sampling, width, height, restart, thread flags, jpeg bytes)]; one seed per file."""
    files = []
    k = 0
    for cls in CLASSES:
        for gname, sampling in GEOMETRIES[cls].items():
            jobs = [(sz, w, h, 0, []) for sz, w, h in sizes(sampling)]
            if gname in RESTART:
                _, w, h = sizes(sampling)[0]
                mw = 8 * max(hh for hh, _ in sampling)
                jobs += [("rst1", 4 * mw, h, 1, []), ("rst3", 4 * mw - 5, h, 3, [])]
            if gname in TALL:
                mw = 8 * max(hh for hh, _ in sampling)
                mh = 8 * max(v for _, v in sampling)
                jobs.append(("tall", 5 * mw - 3, 20 * mh - 2, 0, [4, 8]))
            for sz, w, h, restart, threads in jobs:
                k += 1
                rng = np.random.default_rng(20261016 + k)
                tabs = [photo_tables(rng), photo_tables(rng)]
                q = [[6] + [4 + i // 8 for i in range(63)], [9] + [7 + i // 6 for i in range(63)]][:min(2, len(sampling))]
                jpg = write_baseline(photo_planes(rng, w, h, sampling), w, h, list(sampling), q,
                                     dc_tables=[t[0] for t in tabs], ac_tables=[t[1] for t in tabs], restart=restart)
                files.append(("%s_%s" % (gname, sz), cls, gname, sampling, w, h, restart, threads, jpg))
    return files


def run_reference(src, dst, flags=()):
    if os.path.exists(dst):
        os.unlink(dst)
    r = subprocess.run([LEPTON, "-unjailed", "-skipverify"] + list(flags) + [src, dst], capture_output=True)
    exit_name = exit_name_of(r.stderr)
    rc = EXIT_CODES[exit_name] if exit_name else r.returncode
    out = open(dst, "rb").read() if rc == 0 and os.path.exists(dst) else b""
    return rc, exit_name, out


def decode_back(lep_path, td):
    back = os.path.join(td, "b.jpg")
    if os.path.exists(back):
        os.unlink(back)
    r = subprocess.run([LEPTON, "-unjailed", lep_path, back], capture_output=True)
    return md5(open(back, "rb").read()) if r.returncode == 0 and os.path.exists(back) else None


def check_coverage(record):
    """The corpus holds what the tests lean on; the generator fails otherwise."""
    acc = {n: e for n, e in record.items() if n.endswith(".jpg") and e["status_want"] == 0}
    for cls in CLASSES:
        assert any(e["cls"] == cls for e in acc.values()), ("no accepted file in class", cls)
    colour = [e for e in acc.values() if len(e["sampling"]) == 3]
    mult = lambda e: [bv // e["mcuv"] for bv in e["bcv"]]                     # noqa: E731
    assert any(mult(e)[1] > mult(e)[0] for e in colour), "no file with mult[1] > mult[0]"
    assert any(e["bch"][1] != e["bch"][2] for e in colour), "no file with bch[1] != bch[2]"
    partial = [[e["nch"][c] < e["bch"][c] or e["ncv"][c] < e["bcv"][c] for c in range(3)] for e in colour]
    assert any(any(p) and not all(p) for p in partial), "no file with a partial MCU in some components only"
    assert any(e["restart"] == 1 for e in colour) and any(e["restart"] and e["mcuh"] % e["restart"] for e in colour)
    recs = [e for n, e in record.items() if n.endswith(".lep")]
    for t in (4, 8):
        full = [e for e in recs if e["flags"] == ["-minencodethreads=%d" % t] and e["nseg"] == t]
        assert len(full) >= 8, ("too few files with %d segments" % t, len(full))
        heavy = [m for m in (mult(record[e["source"]]) for e in full) if len(m) == 3 and m[1] > m[0]]
        assert len(heavy) >= 2, ("too few %d-segment files with mult[1] > mult[0]" % t, len(heavy))


def main():
    import lepfmt
    from helpers import plane_hashes
    os.makedirs(OUTDIR, exist_ok=True)
    for f in os.listdir(OUTDIR):
        os.unlink(os.path.join(OUTDIR, f))
    record = {}
    with tempfile.TemporaryDirectory() as td:
        for name, cls, gname, sampling, w, h, restart, threads, jpg in corpus():
            src = os.path.join(OUTDIR, name + ".jpg")
            with open(src, "wb") as f:
                f.write(jpg)
            mcuh, mcuv, grid, coded = geometry(w, h, sampling)
            e = {"path": "geometry/%s.jpg" % name, "jpg_md5": md5(jpg), "cls": cls, "sampling": [list(s) for s in sampling],
                 "width": w, "height": h, "restart": restart, "mcuh": mcuh, "mcuv": mcuv, "bch": [g[0] for g in grid],
                 "bcv": [g[1] for g in grid], "nch": [c[0] for c in coded], "ncv": [c[1] for c in coded]}
            rc, exit_name, lep = run_reference(src, os.path.join(td, "o.lep"))
            e.update(rc=rc, exit_name=exit_name)
            if rc == 0 and lep:
                lp = os.path.join(OUTDIR, name + ".lep")
                with open(lp, "wb") as f:
                    f.write(lep)
                e["lep_md5"] = md5(lep)
                ujg = os.path.join(td, "o.ujg")
                assert subprocess.run([LEPTON, "-unjailed", "-ujg", "-skipverify", src, ujg], capture_output=True).returncode == 0
                e["plane_sha256"] = plane_hashes(lepfmt.parse_ujg_planes(open(ujg, "rb").read())[1])
                e["back_md5"] = decode_back(lp, td)
                e["status_want"] = 0
            else:
                assert rc, (name, "the reference wrote nothing and reported no error")
                e["status_want"] = rc
            record[name + ".jpg"] = e
            print(name, sampling, w, h, len(jpg), rc, exit_name, len(lep), e.get("back_md5") == e["jpg_md5"], flush=True)
            for t in threads:
                flags = ["-minencodethreads=%d" % t]
                rc, exit_name, lep = run_reference(src, os.path.join(td, "t.lep"), flags)
                assert rc == 0 and not exit_name and lep, (name, t, rc, exit_name)
                lname = "%s_t%d.lep" % (name, t)
                lp = os.path.join(OUTDIR, lname)
                with open(lp, "wb") as f:
                    f.write(lep)
                lf = lepfmt.parse_container(lep)
                record[lname] = {"path": "geometry/" + lname, "source": name + ".jpg", "flags": flags, "lep_md5": md5(lep),
                                 "nseg": lf.nseg, "splits": [hd.luma_y_start for hd in lf.handoffs],
                                 "back_md5": decode_back(lp, td)}
                print(" ", lname, len(lep), record[lname]["nseg"], record[lname]["splits"], flush=True)
    check_coverage(record)
    total = sum(os.path.getsize(os.path.join(OUTDIR, f)) for f in os.listdir(OUTDIR))
    print(len(record), "records;", total, "bytes under geometry/")
    with open(OUT, "w") as f:
        json.dump(record, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
