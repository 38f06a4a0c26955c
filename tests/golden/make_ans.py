#!/usr/bin/env python
"""Regenerate tests/golden/ans.json and tests/golden/ans/: .lep files of container version 3 (the reference's -ans option:
the two-state rANS coder instead of the bool coder, brotli header blob; jpgcoder.cc:1120-1122, ans_bool_writer.hh), written
by the UNMODIFIED reference built with -DENABLE_ANS_EXPERIMENTAL (oracle/_ref/lepton-ans, built by oracle/Makefile.ans).

Every case is an input made from committed fixtures (a JPEG, a cut of one, or one behind a prefix of deterministic bytes) and
the reference's flags for it.  Per case the record holds the flags, the encoder's exit code, the md5 and size of the .lep,
and the exit code and md5 of what lepton-ans restores from it, plainly and with -zlib0.  Each .lep that was written goes to
tests/golden/ans/<case>.lep, together with its version-1 twin <case>.v1.lep: the same input and flags through
oracle/_ref/lepton.  The twin has the same segments and the same decisions; its zlib header blob gives the tests the
geometry and the handoffs without a brotli decoder.

Run where oracle/_ref/lepton-ans exists (oracle/Makefile.ans builds it from the reference tree):
    python tests/golden/make_ans.py
"""
import hashlib
import json
import os
import re
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
LEPTON = os.path.join(ROOT, "oracle", "_ref", "lepton")
LEPTON_ANS = os.path.join(ROOT, "oracle", "_ref", "lepton-ans")
OUT = os.path.join(HERE, "ans.json")
FIXDIR = os.path.join(HERE, "ans")

# case name -> (source, how the input is made from it, flags besides -ans)
CASES = {
    "android": ("android.jpg", None, []),                                  # baseline 4:2:0
    "androidcrop": ("androidcrop.jpg", None, []),
    "iphonecrop2": ("iphonecrop2.jpg", None, []),
    "colorswap": ("colorswap.jpg", None, []),
    "androidprogressive": ("androidprogressive.jpg", None, []),            # progressive
    "narrowrst": ("narrowrst.jpg", None, []),                              # restart intervals
    "trailingrst": ("trailingrst.jpg", None, []),
    "androidtrail": ("androidtrail.jpg", None, []),                        # trailing garbage
    "iphonecrop2_t2": ("iphonecrop2.jpg", None, ["-minencodethreads=2"]),
    "iphonecrop2_t4": ("iphonecrop2.jpg", None, ["-minencodethreads=4"]),
    "iphonecrop2_t8": ("iphonecrop2.jpg", None, ["-minencodethreads=8"]),
    "all22_tall_t8": ("geometry/all22_tall.jpg", None, ["-minencodethreads=8"]),
    "dense_color420_uniform": ("dense/color420_uniform.jpg", None, []),   # streams longer than the first stream slot
    "dense_grey_gauss74": ("dense/grey_gauss74.jpg", None, []),
    "dense_color444_odd_rst_t4": ("dense/color444_odd_rst.jpg", None, ["-minencodethreads=4"]),
    "cut_android_40000": ("android.jpg", ("cut", 40000), []),              # truncated JPEGs
    "cut_iphonecrop2_9001": ("iphonecrop2.jpg", ("cut", 9001), []),
    "cut_grayscale_30000_t4": ("grayscale.jpg", ("cut", 30000), ["-minencodethreads=4"]),     # grey
    "emb_androidcrop_p1001": ("androidcrop.jpg", ("prefix", 1001), ["-embedding=1001"]),   # PGE container
    "d_androidcropoptions": ("androidcropoptions.jpg", None, ["-d", "-skipverify"]),     # metadata discarded
}
# one file of every sampling class of the geometry corpus (tests/golden/geometry)
for cls in ("all12", "all21", "all22", "g11", "g12", "g21", "g22", "y11", "y12", "y21", "y22"):
    CASES["geo_%s_odd" % cls] = ("geometry/%s_odd.jpg" % cls, None, [])


def md5(b):
    return hashlib.md5(b).hexdigest()


def case_bytes(name):
    src, how, _ = CASES[name]
    data = open(os.path.join(HERE, src), "rb").read()
    if how and how[0] == "cut":
        data = data[:how[1]]
    elif how and how[0] == "prefix":
        data = bytes((i * 37 + 11) & 255 for i in range(how[1])) + data
    return data


def run(exe, args):
    r = subprocess.run([exe, "-unjailed"] + args, capture_output=True)
    return r.returncode, [n.decode() for n in re.findall(rb"^([A-Z][A-Z0-9_]{3,})$", r.stderr, re.M)]


def main():
    os.makedirs(FIXDIR, exist_ok=True)
    res = {}
    with tempfile.TemporaryDirectory() as tmp:
        src, lep, twin, back = (os.path.join(tmp, n) for n in ("in.bin", "o.lep", "o1.lep", "b.jpg"))
        for name in sorted(CASES):
            data = case_bytes(name)
            with open(src, "wb") as f:
                f.write(data)
            flags = CASES[name][2]
            for f in (lep, twin):
                if os.path.exists(f):
                    os.unlink(f)
            rc, names = run(LEPTON_ANS, ["-ans"] + flags + [src, lep])
            out = open(lep, "rb").read() if rc == 0 and os.path.exists(lep) else b""
            e = {"source": CASES[name][0], "flags": flags, "input_md5": md5(data), "input_size": len(data),
                 "rc": rc, "names": names, "lep_md5": md5(out) if out else None, "lep_size": len(out)}
            if out:
                assert out[2] == 3, name
                for rk, rflags in (("restore", []), ("restore_zlib0", ["-zlib0"])):
                    if os.path.exists(back):
                        os.unlink(back)
                    brc, bnames = run(LEPTON_ANS, rflags + [lep, back])
                    b = open(back, "rb").read() if os.path.exists(back) and brc == 0 else b""
                    e[rk] = {"rc": brc, "names": bnames, "md5": md5(b) if b else None, "size": len(b)}
                trc, _ = run(LEPTON, flags + [src, twin])
                assert trc == 0, (name, trc)
                with open(os.path.join(FIXDIR, name + ".lep"), "wb") as f:
                    f.write(out)
                with open(os.path.join(FIXDIR, name + ".v1.lep"), "wb") as f:
                    f.write(open(twin, "rb").read())
            res[name] = e
            print(name, rc, names[:1], len(out), e.get("restore", {}).get("rc"), flush=True)
    with open(OUT, "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
