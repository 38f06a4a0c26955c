#!/usr/bin/env python
"""Regenerate tests/golden/concat.json and tests/golden/concat/: what the UNMODIFIED reference CLI restores from streams of
concatenated .lep files (process_file, jpgcoder.cc:1867-1898; prep_for_new_file :1508-1524) and from -lepcat files
(concat.cc; the CNT marker of read_ujpg :4187-4189, :4328-4330).

Members are written by the reference with -brotliheader (container version 2: the mux ends in an EOF marker, so the
reader knows where a member ends).  Every case is a stream of bytes built from the members (case_bytes()), restored by
`lepton -` from stdin to stdout, plainly and with -zlib0.  Per case and run the record holds the exit code, the ExitCode
names printed on stderr (the first one is the coder's), and the md5 and length of stdout.  The JPEGs behind the members
are recorded too (jpeg_md5: the concatenation of the members' sources, what a complete restore gives).

Every member and every -lepcat file is committed under tests/golden/concat/, so the streams are rebuilt from the
repository alone.  Run where oracle/_ref/lepton exists (oracle/Makefile builds it from the reference tree):
    python tests/golden/make_concat.py
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

OUT = os.path.join(HERE, "concat.json")
FIXDIR = os.path.join(HERE, "concat")

# member name -> (source bytes maker, reference flags besides -brotliheader)
SMALL = ["trailingrst2", "androidtrail", "androidcrop", "narrowrst", "colorswap"]     # test_concat.sh's images


def md5(b):
    return hashlib.md5(b).hexdigest()


def read(rel):
    with open(os.path.join(HERE, rel), "rb") as f:
        return f.read()


def filler(n, seed):
    return bytes((seed * i * i + 7 * i + seed) & 0xFF for i in range(n))


def members():
    """member name -> (source bytes, extra reference flags)."""
    out = {s: (read(s + ".jpg"), []) for s in SMALL}
    out["tall_t1"] = (read("geometry/all22_tall.jpg"), ["-maxencodethreads=1"])
    out["tall_t4"] = (read("geometry/all22_tall.jpg"), ["-minencodethreads=4"])
    out["tall_t8"] = (read("geometry/all22_tall.jpg"), ["-minencodethreads=8"])
    out["progressive"] = (read("androidprogressive.jpg"), [])
    a = read("android.jpg")
    out["truncated"] = (a[:len(a) * 3 // 5], [])
    out["embedded"] = (filler(1001, 3) + a + filler(777, 5), ["-embedding=1001"])
    return out


def member(name):
    return read("concat/%s.lep" % name)


def legacy():
    """A version-1 container (zlib header blob, no EOF marker): the committed golden .lep of narrowrst."""
    return read("narrowrst.lep")


def cases():
    """case name -> (member names in stream order, or a -lepcat file name; what the bytes are)"""
    out = {}
    for i in ("androidcrop", "narrowrst"):
        for j in ("trailingrst2", "androidtrail"):
            out["pair_%s_%s" % (i, j)] = [i, j]
    for i in ("colorswap", "trailingrst2"):
        for j in ("androidtrail", "androidcrop"):
            for k in ("narrowrst", "trailingrst2"):
                out["triple_%s_%s_%s" % (i, j, k)] = [i, j, k]
    for t in ("tall_t4", "tall_t8"):
        out["t1_then_%s" % t] = ["colorswap", t]
        out["%s_then_t1" % t] = [t, "colorswap"]
    out["tall_t1_then_t8"] = ["tall_t1", "tall_t8"]
    out["baseline_then_progressive"] = ["androidcrop", "progressive"]
    out["progressive_then_baseline"] = ["progressive", "androidcrop"]
    out["truncated_then_baseline"] = ["truncated", "narrowrst"]
    out["baseline_then_truncated"] = ["narrowrst", "truncated"]
    out["embedded_doubled"] = ["embedded", "embedded"]
    out["single_androidcrop"] = ["androidcrop"]
    out["lepcat2"] = ["@lepcat2"]
    out["lepcat3"] = ["@lepcat3"]
    for g in range(1, 8):
        out["garbage%d" % g] = ["androidcrop", "narrowrst", "#garbage%d" % g]
    out["zeta_second"] = ["androidcrop", "!zeta:narrowrst"]
    out["zeta_first"] = ["!zeta:androidcrop", "narrowrst"]
    out["cut_in_second"] = ["androidcrop", "!cut:narrowrst"]
    out["v1_then_v2"] = ["!v1", "narrowrst"]
    out["v2_then_v1"] = ["narrowrst", "!v1"]
    return out


LEPCAT = {"lepcat2": ["androidcrop", "trailingrst2"], "lepcat3": ["colorswap", "androidtrail", "narrowrst"]}


def part_bytes(p):
    if p.startswith("@"):
        return read("concat/%s.lep" % p[1:])
    if p.startswith("#garbage"):
        return filler(int(p[8:]), 11)
    if p.startswith("!zeta:"):
        m = member(p[6:])
        return b"\xce\xb6" + m[2:]
    if p.startswith("!cut:"):
        m = member(p[5:])
        return m[:len(m) // 2]
    if p == "!v1":
        return legacy()
    return member(p)


def case_bytes(parts):
    return b"".join(part_bytes(p) for p in parts)


def part_source(p, src):
    """The JPEG a part would restore to on its own (None for garbage and cut members)."""
    if p.startswith("@"):
        return b"".join(src[m][0] for m in LEPCAT[p[1:]])
    if p.startswith("#") or p.startswith("!cut:"):
        return None
    if p.startswith("!zeta:"):
        return src[p[6:]][0]
    if p == "!v1":
        return read("narrowrst.jpg")
    return src[p][0]


# Where this build differs from the reference on purpose (DESIGN.md section 6): the status it gives instead.  A stream cut
# inside a member is SHORT_READ, as a cut single file is; the reference writes what it restored of it and exits 0.  A
# version-1 member has no EOF marker, so the member behind it is read as its mux packets, and they run past the end of
# the stream; the reference ignores them and restores the first member only.
DIFFERENCES = {"cut_in_second": 3, "v1_then_v2": 3}


def expected(name, e, key):
    """(status, md5 of the output or None) this build gives for case `name` (record `e`), restored plainly ("plain") or
    as a zlib stream ("zlib0"): the reference's output, or ASSERTION_FAILURE (1) where an always_assert aborted it."""
    if name in DIFFERENCES:
        return DIFFERENCES[name], None
    r = e[key]
    if r["rc"] == 0:
        return 0, r["md5"]
    assert r["rc"] == -6 and not r["names"], (name, r)
    return 1, None


def run(args, stdin):
    r = subprocess.run([LEPTON, "-unjailed"] + args, input=stdin, capture_output=True)
    return r.returncode, [n.decode() for n in re.findall(rb"^([A-Z][A-Z0-9_]{3,})$", r.stderr, re.M)], r.stdout


def main():
    os.makedirs(FIXDIR, exist_ok=True)
    src = members()
    with tempfile.TemporaryDirectory() as tmp:
        for name, (data, flags) in sorted(src.items()):
            i, o = os.path.join(tmp, "in.jpg"), os.path.join(FIXDIR, name + ".lep")
            with open(i, "wb") as f:
                f.write(data)
            if os.path.exists(o):
                os.unlink(o)
            r = subprocess.run([LEPTON, "-unjailed", "-skipverify", "-brotliheader"] + flags + [i, o], capture_output=True)
            assert r.returncode == 0 and os.path.exists(o), (name, r.returncode, r.stderr[-300:])
        for name, ms in LEPCAT.items():
            r = subprocess.run([LEPTON, "-unjailed", "-lepcat"] + [os.path.join(FIXDIR, m + ".lep") for m in ms], capture_output=True)
            assert r.returncode == 0 and r.stdout, (name, r.returncode, r.stderr[-300:])
            with open(os.path.join(FIXDIR, name + ".lep"), "wb") as f:
                f.write(r.stdout)
    res = {"members": {k: {"flags": v[1], "jpeg_md5": md5(v[0]), "jpeg_len": len(v[0])} for k, v in src.items()},
           "lepcat": LEPCAT, "cases": {}}
    for name, parts in sorted(cases().items()):
        data = case_bytes(parts)
        whole = [part_source(p, src) for p in parts]
        e = {"parts": parts, "md5": md5(data), "size": len(data)}
        if all(w is not None for w in whole):
            e["jpeg_md5"] = md5(b"".join(whole))
        for key, flags in (("plain", []), ("zlib0", ["-zlib0"])):
            rc, names, out = run(flags + ["-"], data)
            e[key] = {"rc": rc, "names": names, "md5": md5(out), "len": len(out)}
        res["cases"][name] = e
        print(name, e["plain"]["rc"], e["plain"]["names"][:1], e["plain"]["len"], e["zlib0"]["rc"], e["zlib0"]["len"],
              "= sources" if e.get("jpeg_md5") == e["plain"]["md5"] else "", flush=True)
    with open(OUT, "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
