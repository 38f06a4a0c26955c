#!/usr/bin/env python
"""Regenerate tests/golden/extremes/ and tests/golden/extremes.json: baseline JPEGs at the coder's numeric limits and
what the UNMODIFIED reference CLI makes of them.

Every file is written by tests/jpegwriter.py from seeded coefficient planes and targets one regime where the reference's
arithmetic wraps, truncates or caps (see corpus()).  The Huffman tables give codes up to 16 bits long, shuffled
per file.  The coder has to reproduce the reference's bytes there too; the oracle's regime counters
(oracle.regime_counts) show that the corpus reaches each regime.

Run where oracle/_ref/lepton exists (oracle/Makefile builds it from the reference tree):
    python tests/golden/make_extremes.py
The output is deterministic: a second run reproduces the committed files byte for byte.  extremes.json holds per file:

  path                  the file, relative to tests/golden/
  jpg_md5               the input
  rc / exit_name        exit code of `lepton -unjailed -skipverify in.jpg out.lep` and the ExitCode name it wrote to
                        stderr when it failed.  The process status of a failing run is not stable (custom_exit ends one
                        thread, see make_refimages.py), so for those rc is the code of the name, and a run that wrote a
                        name counts as failed whatever its status
  lep_md5               the .lep it wrote (accepted files; committed next to the JPEG)
  plane_sha256          sha256 of each coefficient plane of its `-ujg` dump (accepted files)
  back_md5              md5 of what the reference decodes that .lep to
  status_want           the status the library must report: 0, or 6 (COEFFICIENT_OUT_OF_RANGE) for the refused files
and, for the multi-segment records (`-minencodethreads=N`, named NAME_tN.lep): source, flags, lep_md5, nseg.
"""
import hashlib
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from jpegwriter import AC_SYMBOLS, DC_SYMBOLS, HuffTable, fit_lengths, geometry, write_baseline  # noqa: E402

LEPTON = os.path.join(ROOT, "oracle", "_ref", "lepton")
OUTDIR = os.path.join(HERE, "extremes")
OUT = os.path.join(HERE, "extremes.json")
# ExitCode values of the reference (src/vp8/util/memory.hh); a run that prints one of these names failed with it, even
# when the process itself exits with 0
EXIT_CODES = {"ASSERTION_FAILURE": 1, "CODING_ERROR": 2, "SHORT_READ": 3, "UNSUPPORTED_4_COLORS": 4, "THREAD_PROTOCOL_ERROR": 5,
              "COEFFICIENT_OUT_OF_RANGE": 6, "STREAM_INCONSISTENT": 7, "PROGRESSIVE_UNSUPPORTED": 8,
              "SAMPLING_BEYOND_TWO_UNSUPPORTED": 10, "SAMPLING_BEYOND_FOUR_UNSUPPORTED": 11, "THREADING_PARTIAL_MCU": 12,
              "ONLY_GARBAGE_NO_JPEG": 14, "UNSUPPORTED_JPEG": 42, "UNSUPPORTED_JPEG_WITH_ZERO_IDCT_0": 43}
RASTER_OF_ZZ = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
                21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60,
                61, 54, 47, 55, 62, 63]


def md5(b):
    return hashlib.md5(b).hexdigest()


def long_tables(rng, ac_sizes=11, last_ac=0x0B):
    """DC and AC tables whose codes run from 2 to 16 bits; most symbols get 16-bit codes.  `last_ac` gets the largest
    code (fifteen 1 bits and a 0), so runs of it with all-ones magnitudes fill the scan with stuffed 0xFF bytes."""
    dc = [int(s) for s in rng.permutation(DC_SYMBOLS[:12])]
    ac = [0x00] + [int(s) for s in rng.permutation([s for s in AC_SYMBOLS if s and (s & 15) <= ac_sizes and s != last_ac])]
    ac.append(last_ac)
    dct = HuffTable(fit_lengths([(s, min(16, 4 + i)) for i, s in enumerate(dc)]))
    act = HuffTable(fit_lengths([(s, min(16, 2 + i)) for i, s in enumerate(ac)]))
    return dct, act


def magnitudes(rng, shape, cats):
    """Signed values whose magnitude category is drawn from `cats` (0 = zero), uniform inside the category."""
    c = rng.choice(cats, size=shape)
    lo = np.where(c > 0, 1 << np.maximum(c - 1, 0), 0)
    m = lo + (rng.integers(0, 1 << 16, size=shape) % np.maximum(lo, 1)) * (c > 0)
    return (m * (rng.integers(0, 2, size=shape) * 2 - 1)).astype(np.int64)


def dc_walk(rng, n, lim=1000, step=600):
    """Absolute DC values within +-lim whose successive differences stay within category 11."""
    v = np.cumsum(rng.integers(-step, step + 1, size=n))
    v = (v + lim) % (4 * lim)
    return np.where(v > 2 * lim, 4 * lim - v, v) - lim


def dense_grey(rng, cats, w=64, h=64):
    _, _, grid, _ = geometry(w, h, [(1, 1)])
    bx, by = grid[0]
    p = magnitudes(rng, (by, bx, 64), cats)
    p[..., 0] = dc_walk(rng, by * bx).reshape(by, bx)
    return [p]


def sparse_colour(rng, w, h, sampling, nnz=4, ff_rows=1):
    """Mostly-empty blocks with a few large coefficients each (every category up to 11, weighted to 11); the first
    `ff_rows` block rows of luma are all +2047 to make long runs of stuffed 0xFF bytes."""
    _, _, grid, _ = geometry(w, h, sampling)
    planes = []
    for c, (bx, by) in enumerate(grid):
        n = by * bx
        p = np.zeros((n, 64), np.int64)
        pos = rng.integers(1, 64, size=(n, nnz))
        val = magnitudes(rng, (n, nnz), [1, 2, 3, 5, 8, 10, 11, 11, 11, 11])
        np.put_along_axis(p, pos, val, axis=1)
        p[:, 0] = dc_walk(rng, n, lim=1000 if c == 0 else 400)
        p = p.reshape(by, bx, 64)
        if c == 0:
            p[:ff_rows, :, 1:] = 2047
        planes.append(p)
    return planes


def q_table(vals_raster):
    return [int(vals_raster[RASTER_OF_ZZ[k]]) for k in range(64)]


def corpus():
    """-> [(name, jpeg bytes, extra flag sets)].  Each file has its own seed."""
    files = []

    def rng(k):
        return np.random.default_rng(20261015 + k)

    # magnitudes 1024..2047 at all 63 AC positions, q = 1: length 11 everywhere, bit-length cap, threshold context 255,
    # saturated threshold context index (min_thr = 0).  The DC quantiser is 255 in these files: with q0 = 1 the DC
    # prediction of such blocks is far out of the +-1024 the reference can code, and it refuses the file.
    r = rng(1)
    dct, act = long_tables(r)
    files.append(("cat11_q1", write_baseline(dense_grey(r, [11]), 64, 64, [(1, 1)], [[255] + [1] * 63], dc_tables=[dct],
                                             ac_tables=[act]), []))
    # the same with q = 255: Lakhani sum wraps, IDCT int32 overflow, int16 pixel truncation
    r = rng(2)
    dct, act = long_tables(r)
    files.append(("cat11_q255", write_baseline(dense_grey(r, [11]), 64, 64, [(1, 1)], [[255] * 64], dc_tables=[dct], ac_tables=[act]), []))
    # 16-bit DQT, q = 65535 everywhere
    r = rng(3)
    dct, act = long_tables(r)
    files.append(("q16_max", write_baseline(dense_grey(r, list(range(12))), 64, 64, [(1, 1)], [[65535] * 64], qbits=16,
                                            dc_tables=[dct], ac_tables=[act]), []))
    # 16-bit DQT, first row and column 1, the rest near 65535: |prior| > 65535 (threshold-context mask, int16 sign context)
    r = rng(4)
    dct, act = long_tables(r)
    q = r.integers(60000, 65536, size=64)
    q[:8] = 1
    q[::8] = 1
    q[0] = 65535
    files.append(("q16_mixed", write_baseline(dense_grey(r, list(range(12))), 64, 64, [(1, 1)], [q_table(q)], qbits=16,
                                              dc_tables=[dct], ac_tables=[act]), []))
    # DC values near +-1024 with a large q0: adv_unpredict wraps both ways, q0 * dc wraps in int16
    r = rng(5)
    dct, act = long_tables(r)
    p = dense_grey(r, [0, 0, 0, 1, 2, 4, 6])
    p[0][..., 0] = r.choice([-1024, -1020, -1000, -900, 900, 1000, 1020, 1024], size=p[0].shape[:2])
    for k in range(1, p[0].shape[0] * p[0].shape[1]):      # keep DC differences within category 11
        y, x = divmod(k, p[0].shape[1])
        py, px = divmod(k - 1, p[0].shape[1])
        if abs(p[0][y, x, 0] - p[0][py, px, 0]) > 2047:
            p[0][y, x, 0] = -p[0][y, x, 0]
    q = np.full(64, 40)
    q[0] = 200
    files.append(("dc_wrap", write_baseline(p, 64, 64, [(1, 1)], [q_table(q)], dc_tables=[dct], ac_tables=[act]), []))
    # refused: one DC outside +-1024
    r = rng(6)
    p = dense_grey(r, [0, 0, 1, 3, 5])
    p[0][..., 0] = np.clip(p[0][..., 0], -300, 300)
    p[0][3, 4, 0] = 1500
    files.append(("dc_out_of_range", write_baseline(p, 64, 64, [(1, 1)], [[16] * 64]), []))
    # refused: q0 = 1 under category-11 magnitudes puts the DC prediction thousands away; the residual round-trips through
    # adv_unpredict's single wrap but needs more than 11 bits
    r = rng(11)
    dct, act = long_tables(r)
    files.append(("dc_residual_long", write_baseline(dense_grey(r, [11]), 64, 64, [(1, 1)], [[1] * 64], dc_tables=[dct],
                                                     ac_tables=[act]), []))
    # refused: one AC coefficient of category 12
    r = rng(7)
    dct, act = long_tables(r, ac_sizes=12)
    p = dense_grey(r, [0, 0, 1, 3, 5, 11])
    p[0][5, 2, 9] = -3000
    files.append(("cat12", write_baseline(p, 64, 64, [(1, 1)], [[8] * 64], dc_tables=[dct], ac_tables=[act]), []))
    # colour, large enough for many Huffman sub-sequences and several thread-segments
    r = rng(8)
    tabs = [long_tables(r), long_tables(r)]
    qs = [list(r.integers(1, 256, size=64)), list(r.integers(1, 256, size=64))]
    files.append(("color420_long", write_baseline(sparse_colour(r, 512, 512, [(2, 2), (1, 1), (1, 1)]), 512, 512,
                                                  [(2, 2), (1, 1), (1, 1)], qs, dc_tables=[t[0] for t in tabs],
                                                  ac_tables=[t[1] for t in tabs]), [4, 8]))
    r = rng(9)
    tabs = [long_tables(r), long_tables(r)]
    q = r.integers(1, 65536, size=(3, 64))
    q[:, 0] = r.integers(1, 64, size=3)
    files.append(("color444_long", write_baseline(sparse_colour(r, 352, 352, [(1, 1)] * 3, nnz=3), 352, 352, [(1, 1)] * 3,
                                                  [list(t) for t in q], qbits=16, dc_tables=[t[0] for t in tabs],
                                                  ac_tables=[t[1] for t in tabs]), [4, 8]))
    # partial MCUs (odd size, 4:2:2) and restart markers every 5 MCUs
    r = rng(10)
    tabs = [long_tables(r), long_tables(r)]
    files.append(("odd_rst", write_baseline(sparse_colour(r, 203, 141, [(2, 1), (1, 1), (1, 1)], nnz=12), 203, 141,
                                            [(2, 1), (1, 1), (1, 1)], [[255] * 64, [255] + [3] * 63], dc_tables=[t[0] for t in tabs],
                                            ac_tables=[t[1] for t in tabs], restart=5), [4]))
    return files


def run_reference(src, dst, flags=()):
    if os.path.exists(dst):
        os.unlink(dst)
    r = subprocess.run([LEPTON, "-unjailed", "-skipverify"] + list(flags) + [src, dst], capture_output=True)
    names = re.findall(rb"^([A-Z][A-Z0-9_]{3,})$", r.stderr, re.M)
    out = open(dst, "rb").read() if os.path.exists(dst) else b""
    return r.returncode, names[-1].decode() if names else None, out


def main():
    import lepfmt
    from helpers import plane_hashes
    os.makedirs(OUTDIR, exist_ok=True)
    record = {}
    with tempfile.TemporaryDirectory() as td:
        for name, jpg, threads in corpus():
            src = os.path.join(OUTDIR, name + ".jpg")
            with open(src, "wb") as f:
                f.write(jpg)
            rc, exit_name, lep = run_reference(src, os.path.join(td, "o.lep"))
            if exit_name:
                rc = EXIT_CODES[exit_name]
            e = {"path": "extremes/%s.jpg" % name, "jpg_md5": md5(jpg), "rc": rc, "exit_name": exit_name}
            if rc == 0 and lep:
                with open(os.path.join(OUTDIR, name + ".lep"), "wb") as f:
                    f.write(lep)
                e["lep_md5"] = md5(lep)
                ujg = os.path.join(td, "o.ujg")
                assert subprocess.run([LEPTON, "-unjailed", "-ujg", "-skipverify", src, ujg], capture_output=True).returncode == 0
                e["plane_sha256"] = plane_hashes(lepfmt.parse_ujg_planes(open(ujg, "rb").read())[1])
                back = os.path.join(td, "b.jpg")
                assert subprocess.run([LEPTON, "-unjailed", os.path.join(OUTDIR, name + ".lep"), back], capture_output=True).returncode == 0
                e["back_md5"] = md5(open(back, "rb").read())
                e["status_want"] = 0
            else:
                assert rc, (name, "the reference wrote nothing and reported no error")
                e["status_want"] = rc
            record[name + ".jpg"] = e
            print(name, len(jpg), rc, exit_name, len(lep), flush=True)
            for t in threads:
                flags = ["-minencodethreads=%d" % t]
                rc, exit_name, lep = run_reference(src, os.path.join(td, "t.lep"), flags)
                assert rc == 0 and not exit_name and lep, (name, t)
                lname = "%s_t%d.lep" % (name, t)
                with open(os.path.join(OUTDIR, lname), "wb") as f:
                    f.write(lep)
                record[lname] = {"path": "extremes/" + lname, "source": name + ".jpg", "flags": flags, "lep_md5": md5(lep),
                                 "nseg": lepfmt.parse_container(lep).nseg}
                print(" ", lname, len(lep), record[lname]["nseg"], flush=True)
    with open(OUT, "w") as f:
        json.dump(record, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
