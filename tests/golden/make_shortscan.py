#!/usr/bin/env python
"""Regenerate tests/golden/shortscan/ and tests/golden/shortscan.json: complete baseline JPEGs (EOI present) whose scan
is short, damaged or oddly padded, and what the UNMODIFIED reference CLI makes of them.

A JPEG can end in EOI and still have less entropy-coded data than its frame needs: a writer that stopped early, a file
spliced together.  The reference reads zeros past the end of the data, finishes the block it is in and stops, and the
file is coded like any other (jpgcoder.cc, decode_jpeg: huffr->eof ends the scan).  The same decoder refuses a zero
run past the end of a block when the data did not run out (ASSERTION_FAILURE), padding that changes between restart
intervals and bytes left over behind the last block (UNSUPPORTED_JPEG).  Every file here is written by
tests/jpegwriter.py from seeded planes, then:

  full        the complete file, untouched (one per source, for comparison)
  cut_block   the scan cut in the middle of a block (at half its bytes), then FF D9
  cut_row     the scan of the first MCU rows only, ending at an MCU-row border with its pad bits, then FF D9
  cut_rst     the scan cut right after its first RST marker, then FF D9 (restart sources)
  cut_1       the last byte of the scan removed
  pad0        every interval padded with 0 bits instead of 1 (where the scan has pad bits)
  padmix      the restart intervals padded with 1 and 0 bits in turn (restart sources)
  junk        three bytes behind the coded data, in front of EOI
  flip_S      one bit of the scan flipped, at the first position (from a seeded order) where the product's host decoder
              reports status S: 0 (other coefficients), 1 (a zero run past the end of a block) or 42 (a bad code, an
              EOB after a zero); flips that make or break an FF byte are skipped, so the file stays parseable
plus the committed badzerorun.jpg (a zero run past the end of a block in complete data).

Run where oracle/_ref/lepton exists (oracle/Makefile builds it from the reference tree):
    python tests/golden/make_shortscan.py
The output is deterministic: a second run reproduces every file byte for byte.  shortscan.json holds per file:

  path            relative to tests/golden/
  kind, source    the variant above and the source it was made from
  jpg_md5
  rc_skipverify   exit code of `lepton -unjailed -skipverify in.jpg out.lep`, and exit_name, the ExitCode name it wrote to
  exit_name       stderr (a run that printed a name failed with it, see make_extremes.py)
  rc_verify       the same run without -skipverify (the reference decodes the .lep again and compares)
  status_want     the status the library must report: rc_skipverify (the library does not verify by default), or 1
                  (ASSERTION_FAILURE) where the reference died on an assert (rc_skipverify -6, SIGABRT)
  lep_md5         the .lep of an accepted file (committed as shortscan/NAME.lep)
  back_md5        md5 of what the reference decodes that .lep to
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
sys.path.insert(0, ROOT)
from jpegwriter import geometry, write_baseline  # noqa: E402
from make_extremes import EXIT_CODES, LEPTON  # noqa: E402
from make_truncated import GREY, S420, S444, smooth_planes, sos_end  # noqa: E402

OUTDIR = os.path.join(HERE, "shortscan")
OUT = os.path.join(HERE, "shortscan.json")
Q = [6] + [4 + i // 8 for i in range(63)]
CODES = dict(EXIT_CODES, ROUNDTRIP_FAILURE=41)


def exit_name_of(stderr):
    """The first ExitCode name the run printed on a line of its own: the error it stopped with (a verifying run goes on
    to print ROUNDTRIP_FAILURE and SHORT_READ behind it)."""
    for line in stderr.decode("latin-1").splitlines():
        if line.strip() in CODES:
            return line.strip()
    return None


def md5(b):
    return hashlib.md5(b).hexdigest()


# name, seed, width, height, sampling, restart interval (MCUs)
SOURCES = [("grey", 1, 64, 48, GREY, 0), ("c420", 2, 48, 40, S420, 0), ("c444", 3, 40, 32, S444, 0),
           ("c420_rst2", 4, 48, 48, S420, 2), ("c444_rst3", 5, 40, 40, S444, 3)]


def scan_span(jpg):
    """[first, end) of the entropy-coded bytes (restart markers included) of a file written by write_baseline."""
    assert jpg[-2:] == b"\xff\xd9"
    return sos_end(jpg), len(jpg) - 2


def cut_at(jpg, k):
    """The file with its scan ending before file byte k, then EOI; k moves back so that no FF is left dangling."""
    while jpg[k - 1] == 0xFF:
        k -= 1
    return jpg[:k] + b"\xff\xd9"


def flips(jpg, seed):
    """Scan bit flips that keep the file parseable, in a seeded order: (file offset, bit)."""
    a, b = scan_span(jpg)
    order = np.random.default_rng(seed).permutation((b - a) * 8)
    for q in order:
        off, bit = a + int(q) // 8, int(q) % 8
        v = jpg[off] ^ (1 << bit)
        if jpg[off] == 0xFF or v == 0xFF or jpg[off - 1] == 0xFF:
            continue
        yield off, bit


def variants():
    """-> [(file name, kind, source, jpeg bytes)]."""
    from lepton_b200 import HostJpeg
    out = []
    for name, seed, w, h, sampling, rst in SOURCES:
        rng = np.random.default_rng(20261018 + seed)
        planes = smooth_planes(rng, w, h, sampling)
        q = [Q] * (1 if len(sampling) == 1 else 2)

        def write(pl=planes, hh=h, **kw):
            return write_baseline(pl, w, hh, sampling, q, restart=rst, **kw)
        full = write()
        a, b = scan_span(full)
        add = lambda kind, data: out.append(("%s_%s.jpg" % (name, kind), kind, name, data))   # noqa: E731
        add("full", full)
        add("cut_block", cut_at(full, (a + b) // 2))
        # the first MCU rows of the same planes: their scan is a prefix of the full one, up to the row border and padded
        mcuh, mcuv, grid, _ = geometry(w, h, sampling)
        vmax = max(v for _, v in sampling)
        rows = mcuv // 2
        part = write([p[:rows * sampling[c][1]] for c, p in enumerate(planes)], rows * 8 * vmax)
        pa, pb = scan_span(part)
        add("cut_row", full[:a] + part[pa:pb] + b"\xff\xd9")
        if rst:
            k = full.index(b"\xff\xd0", a)
            add("cut_rst", full[:k + 2] + b"\xff\xd9")
        add("cut_1", cut_at(full, b - 1))
        pad0 = write(padbit=0)
        if pad0 != full:                  # a scan that ends on a byte border has no pad bits
            add("pad0", pad0)
        if rst:
            add("padmix", write(padbit=[k & 1 for k in range(mcuh * mcuv + 1)]))
        add("junk", full[:b] + b"\x5a\xa5\x33" + full[b:])
        want = {0: None, 1: None, 42: None}
        for off, bit in flips(full, seed):
            d = bytearray(full)
            d[off] ^= 1 << bit
            st = HostJpeg(bytes(d)).status
            if st in want and want[st] is None:
                want[st] = bytes(d)
            if all(v is not None for v in want.values()):
                break
        for st, d in sorted(want.items()):
            if d is not None:
                add("flip_%d" % st, d)
    return out


def run_reference(jpg):
    """-> (rc_skipverify, exit name, rc_verify, lep bytes, bytes the reference decodes the .lep to)."""
    with tempfile.TemporaryDirectory() as td:
        src, dst, back = (os.path.join(td, f) for f in ("in.jpg", "out.lep", "back.jpg"))
        with open(src, "wb") as f:
            f.write(jpg)
        res = []
        for fl in (["-skipverify"], []):
            if os.path.exists(dst):
                os.unlink(dst)
            r = subprocess.run([LEPTON, "-unjailed"] + fl + [src, dst], capture_output=True)
            name = exit_name_of(r.stderr)
            res.append((CODES[name] if name else r.returncode, name))
            if not fl:
                continue
            lep = open(dst, "rb").read() if res[0][0] == 0 and os.path.exists(dst) else b""
        out = b""
        if lep:
            with open(dst, "wb") as f:
                f.write(lep)
            subprocess.run([LEPTON, "-unjailed", dst, back], capture_output=True)
            out = open(back, "rb").read() if os.path.exists(back) else b""
    return res[0][0], res[0][1], res[1][0], lep, out


def main():
    os.makedirs(OUTDIR, exist_ok=True)
    for f in os.listdir(OUTDIR):
        os.unlink(os.path.join(OUTDIR, f))
    files = [(fn, kind, src, data) for fn, kind, src, data in variants()]
    files.append(("badzerorun.jpg", "zerorun", "badzerorun", open(os.path.join(HERE, "badzerorun.jpg"), "rb").read()))
    record = {}
    for fn, kind, src, jpg in files:
        path = fn if fn == "badzerorun.jpg" else "shortscan/" + fn
        if path != fn:
            with open(os.path.join(HERE, path), "wb") as f:
                f.write(jpg)
        rc, name, rcv, lep, back = run_reference(jpg)
        e = {"path": path, "kind": kind, "source": src, "jpg_md5": md5(jpg), "rc_skipverify": rc, "exit_name": name,
             "rc_verify": rcv, "status_want": 1 if rc == -6 else rc, "lep_md5": None, "back_md5": None}
        if lep:
            with open(os.path.join(OUTDIR, fn[:-4] + ".lep"), "wb") as f:
                f.write(lep)
            e["lep_md5"], e["back_md5"] = md5(lep), md5(back)
        record[fn] = e
        print("%-22s %-9s rc %3d %-24s verify %3d %s" % (fn, kind, rc, name or "", rcv, "" if not lep else
                                                       ("restores the input" if back == jpg else "restores other bytes")))
    with open(OUT, "w") as f:
        f.write(json.dumps(record, indent=1, sort_keys=True) + "\n")


if __name__ == "__main__":
    main()
