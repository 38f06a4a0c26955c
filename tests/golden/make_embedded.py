#!/usr/bin/env python
"""Regenerate tests/golden/embedded.json: what the UNMODIFIED reference CLI does with JPEGs embedded in larger files
(-embedding=N: the SOI sits at byte N; jpgcoder.cc:1135-1137, read_jpeg :2275-2282, PGE section :4009-4017, restore
recoder.cc:449-456) and with -d (discard metadata, rebuild_header_jpg :4848-4888).

Every case is a file made again from case_bytes() (committed fixtures behind and in front of deterministic bytes) and the
reference's flags for it.  Per case and run the record holds the exit code, the ExitCode names printed on stderr (the
first one is the coder's: the process status of a failed run is not stable), the md5 and size of the .lep, and for a
.lep written with -skipverify the md5 and size of what the reference restores from it, plainly and with -zlib0.
Runs: "verify" (the reference's default), "skipverify", "t4" / "t8" (-skipverify -minencodethreads=4 / 8).

A few of the reference's .lep files are kept under tests/golden/embedded/ (LEP_FIXTURES) so that restoring files the
reference wrote is tested as well as writing them.

Run where oracle/_ref/lepton exists (oracle/Makefile builds it from the reference tree):
    python tests/golden/make_embedded.py
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

OUT = os.path.join(HERE, "embedded.json")
FIXDIR = os.path.join(HERE, "embedded")
BASELINE = ["android.jpg", "grayscale.jpg", "trailingrst.jpg", "geometry/all22_tall.jpg"]   # 4:2:0, grey, restarts, 8 segments
PREFIXES = [1, 2, 3, 255, 4096, 70000]
RUNS = {"verify": [], "skipverify": ["-skipverify"], "t4": ["-skipverify", "-minencodethreads=4"],
        "t8": ["-skipverify", "-minencodethreads=8"]}
LEP_FIXTURES = ["all22_tall.jpg_p1_t0", "all22_tall.jpg_p70000_t1", "trailingrst.jpg_p255_t1", "trunc_p1001",
                "d_emb_androidcropoptions"]


def md5(b):
    return hashlib.md5(b).hexdigest()


def filler(n, seed):
    """n deterministic bytes, different for every seed (prefixes and trailers)."""
    return bytes((seed * i * i + 7 * i + seed) & 0xFF for i in range(n))


def read(rel):
    with open(os.path.join(HERE, rel), "rb") as f:
        return f.read()


def cases():
    """name -> (source description, flags that shape the bytes: -embedding= / -d).  The bytes come from case_bytes(name)."""
    out = {}
    for src in BASELINE:
        for p in PREFIXES:
            for t in (0, 1):
                out["%s_p%d_t%d" % (src.split("/")[-1], p, t)] = ["-embedding=%d" % p]
    out["android.jpg_e0"] = ["-embedding=0"]               # offset 0: the plain .lep
    out["trunc_p1001"] = ["-embedding=1001"]               # a truncated JPEG behind a prefix
    out["prog_p500"] = ["-embedding=500"]                  # progressive: the reference's restore drops the prefix
    out["notsoi_p1001"] = ["-embedding=1000"]              # the offset is not at the SOI
    out["past_end"] = ["-embedding=200000"]                # the offset lies past the end of the input
    out["plain_e2"] = ["-embedding=2"]                     # -embedding=2 on a plain JPEG
    out["lep_e0"] = ["-embedding=0"]                       # a .lep taken as a JPEG: every input is one with -embedding
    out["lep_e5"] = ["-embedding=5"]
    for src in ("android.jpg", "androidcropoptions.jpg", "grayscale.jpg", "iphonecrop2.jpg"):
        out["d_" + src[:-4]] = ["-d"]                      # APPn / COM segments dropped
    out["d_emb_androidcropoptions"] = ["-d", "-embedding=4096"]
    return out


def case_bytes(name):
    if name == "android.jpg_e0" or name == "plain_e2":
        return read("android.jpg")
    if name == "trunc_p1001":
        j = read("android.jpg")
        return filler(1001, 3) + j[:len(j) * 3 // 5]
    if name == "prog_p500":
        return filler(500, 5) + read("androidprogressive.jpg")
    if name in ("notsoi_p1001", "past_end"):
        return filler(1001, 3) + read("android.jpg") + filler(777, 5)
    if name.startswith("lep_"):
        return read("android.lep")
    if name.startswith("d_emb_"):
        return filler(4096, 9) + read(name[6:] + ".jpg")
    if name.startswith("d_"):
        return read(name[2:] + ".jpg")
    src, p, t = name.rsplit("_", 2)
    rel = [b for b in BASELINE if b.split("/")[-1] == src][0]
    return filler(int(p[1:]), 3) + read(rel) + (filler(777, 5) if t == "t1" else b"")


def embedding_of(flags):
    """The -embedding= offset of a case's flags (None without one) and whether -d is among them."""
    off = [int(f.split("=")[1]) for f in flags if f.startswith("-embedding=")]
    return (off[0] if off else None), "-d" in flags


def expected_status(r):
    """The status this build gives where the reference made the run record `r`: 0 for a .lep written, else the code of the
    first ExitCode name the coder printed, or ASSERTION_FAILURE (1) when an always_assert aborted it without a name."""
    from make_extremes import EXIT_CODES
    if r["rc"] == 0 and r["lep_md5"]:
        return 0
    if r["names"]:
        return 41 if r["names"][0] == "ROUNDTRIP_FAILURE" else EXIT_CODES[r["names"][0]]
    assert r["rc"] == -6, r
    return 1


def run(args):
    r = subprocess.run([LEPTON, "-unjailed"] + args, capture_output=True)
    return r.returncode, [n.decode() for n in re.findall(rb"^([A-Z][A-Z0-9_]{3,})$", r.stderr, re.M)]


def main():
    os.makedirs(FIXDIR, exist_ok=True)
    res = {"runs": RUNS, "cases": {}}
    with tempfile.TemporaryDirectory() as tmp:
        src, lep, back = os.path.join(tmp, "in.bin"), os.path.join(tmp, "o.lep"), os.path.join(tmp, "b.jpg")
        for name, flags in sorted(cases().items()):
            data = case_bytes(name)
            with open(src, "wb") as f:
                f.write(data)
            e = {"flags": flags, "md5": md5(data), "size": len(data)}
            for key, extra in RUNS.items():
                for f in (lep, back):
                    if os.path.exists(f):
                        os.unlink(f)
                rc, names = run(flags + extra + [src, lep])
                out = open(lep, "rb").read() if os.path.exists(lep) else b""
                r = {"rc": rc, "names": names, "lep_md5": md5(out) if out else None, "lep_size": len(out)}
                if key != "verify" and rc == 0 and out:
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
            print(name, {k: (e[k]["rc"], e[k]["names"][:1], e[k]["lep_size"]) for k in RUNS}, flush=True)
    with open(OUT, "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
