#!/usr/bin/env python
"""Regenerate tests/golden/permissive.json: what the UNMODIFIED reference CLI does with -permissive (jpgcoder.cc:1111,
process_file :1603-1655, validation.cc:25-218, generic_compress.cc:60-200).  A file the coder cannot take -- not a JPEG,
damaged, arithmetic-coded, one whose .lep would not restore it byte for byte, a .lep itself -- is stored in the generic
'Y' container (a fixed 1x1 grey header, the whole input in the PGE section, no coded blocks) and restored byte for byte;
a file the coder takes gives its ordinary .lep; an empty input fails with UNSUPPORTED_JPEG.

Every case is a file made again from case_bytes() (committed fixtures, or deterministic bytes for the non-JPEG blobs)
and the reference's flags for it.  Per case and run the record holds the exit code, the ExitCode names printed on
stderr, the md5 and size of the .lep and, for every .lep written, the exit code, md5 and size of what the reference
restores from it, plainly and with -zlib0.  Runs: "verify" (-permissive alone), "skipverify" (-permissive -skipverify:
the reference verifies every file under -permissive all the same) and "t1" (-skipverify -maxencodethreads=1).

A few generic .lep files of the skipverify run are kept under tests/golden/permissive/ (LEP_FIXTURES) so that restoring
files the reference wrote is tested as well as writing them; every other case is checked through its recorded md5.

Run where oracle/_ref/lepton exists (oracle/Makefile builds it from the reference tree):
    python tests/golden/make_permissive.py
"""
import hashlib
import json
import os
import re
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_extremes import LEPTON  # noqa: E402

OUT = os.path.join(HERE, "permissive.json")
FIXDIR = os.path.join(HERE, "permissive")
RUNS = {"verify": [], "skipverify": ["-skipverify"], "t1": ["-skipverify", "-maxencodethreads=1"]}
LEP_FIXTURES = ["one_byte", "two_bytes", "arithmetic_head", "badzerorun", "blob70k"]

# name -> (source, extra flags)
CASES = {
    "badzerorun": ("badzerorun.jpg", []),                    # the reference's coder asserts on a zero run
    "roundtripfail": ("legacy/roundtripfail.jpg", []),       # its .lep does not restore the file
    "nofsync": ("nofsync.jpg", []),
    "arithmetic_head": ("arithmetic_head.jpg", []),          # arithmetic-coded (SOF10)
    "trunc_head": ("trunc_head.jpg", []),                    # a truncated JPEG the coder takes
    "androidcrop": ("androidcrop.jpg", []),                  # a good JPEG: the plain .lep
    "gold_legacy_lep": ("legacy/gold-legacy.lep", []),       # .lep files are inputs like any other
    "android_lep": ("android.lep", []),
    "empty": (None, []),
    "one_byte": (None, []),
    "two_bytes": (None, []),
    "blob70k": (None, []),
    "blob1m": (None, []),
    "d_androidcropoptions": ("androidcropoptions.jpg", ["-d"]),           # -d: the restored JPEG differs -> generic
    "emb5_androidcrop": ("androidcrop.jpg", ["-embedding=5"]),            # the SOI is not at byte 5 -> generic
    "emb1001_android": (None, ["-embedding=1001"]),                       # a real embedded JPEG: the PGE .lep
}


def md5(b):
    return hashlib.md5(b).hexdigest()


def read(rel):
    with open(os.path.join(HERE, rel), "rb") as f:
        return f.read()


def blob(n, seed):
    """n deterministic bytes that deflate neither trivially nor not at all: words of a small vocabulary (long matches,
    skewed literals) broken up by runs of noise (literals of every value), from a 32-bit LCG."""
    words = [b"lepton", b"jpeg", b"container", b" ", b"\n", b"0123456789", b"\xff\xd8", b"\xcf\x84", b"generic", b"PGE"]
    out = bytearray()
    x = seed & 0xFFFFFFFF
    while len(out) < n:
        x = (x * 1664525 + 1013904223) & 0xFFFFFFFF
        if (x >> 28) < 3:
            for _ in range(1 + ((x >> 16) & 63)):
                x = (x * 1664525 + 1013904223) & 0xFFFFFFFF
                out.append(x >> 24)
        else:
            out += words[(x >> 16) % len(words)]
    return bytes(out[:n])


def case_bytes(name):
    src = CASES[name][0]
    if src:
        return read(src)
    if name == "empty":
        return b""
    if name == "one_byte":
        return b"a"
    if name == "two_bytes":
        return b"bc"
    if name == "blob70k":
        return blob(70000, 70)
    if name == "blob1m":
        return blob(1 << 20, 1)
    if name == "emb1001_android":
        return blob(1001, 3) + read("android.jpg")
    raise KeyError(name)


def run(args):
    r = subprocess.run([LEPTON, "-unjailed"] + args, capture_output=True)
    return r.returncode, [n.decode() for n in re.findall(rb"^([A-Z][A-Z0-9_]{3,})$", r.stderr, re.M)]


def main():
    os.makedirs(FIXDIR, exist_ok=True)
    res = {"runs": RUNS, "cases": {}}
    with tempfile.TemporaryDirectory() as tmp:
        src, lep, back = os.path.join(tmp, "in.bin"), os.path.join(tmp, "o.lep"), os.path.join(tmp, "b.jpg")
        for name in sorted(CASES):
            data = case_bytes(name)
            with open(src, "wb") as f:
                f.write(data)
            e = {"flags": CASES[name][1], "md5": md5(data), "size": len(data)}
            for key, extra in RUNS.items():
                for f in (lep, back):
                    if os.path.exists(f):
                        os.unlink(f)
                rc, names = run(["-permissive"] + CASES[name][1] + extra + [src, lep])
                out = open(lep, "rb").read() if os.path.exists(lep) else b""
                r = {"rc": rc, "names": names, "lep_md5": md5(out) if out else None, "lep_size": len(out),
                     "flag": chr(out[3]) if len(out) > 3 else None}
                if rc == 0 and out:
                    for rk, rflags in (("restore", []), ("restore_zlib0", ["-zlib0"])):
                        if os.path.exists(back):
                            os.unlink(back)
                        brc, bnames = run(rflags + [lep, back])
                        b = open(back, "rb").read() if os.path.exists(back) and brc == 0 else b""
                        r[rk] = {"rc": brc, "names": bnames, "md5": md5(b) if b else None, "size": len(b)}
                    if key == "skipverify" and name in LEP_FIXTURES:
                        with open(os.path.join(FIXDIR, name + ".lep"), "wb") as f:
                            f.write(out)
                e[key] = r
            res["cases"][name] = e
            print(name, {k: (e[k]["rc"], e[k]["flag"], e[k]["lep_size"]) for k in RUNS}, flush=True)
    with open(OUT, "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
