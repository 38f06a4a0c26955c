#!/usr/bin/env python
"""Regenerate tests/golden/zlib0.json: what the UNMODIFIED reference CLI writes when it restores .lep files as zlib streams.

`lepton -zlib0 in.lep out` writes the JPEG as a zlib stream of stored deflate blocks (jpgcoder.cc:2089, check_file
:2200-2220, src/io/Zlib0.cc), and a container whose magic is CE B6 (zeta) instead of CF 84 (tau) is restored that way
without the flag.  Two sets are recorded:

  leps    every committed .lep under tests/golden/ (golden, extremes, dense, geometry, truncated, legacy, future), restored
          with -zlib0 ("plain") and as a zeta copy (the same bytes with CE B6 in front, "zeta"): exit code, exit name
          printed on stderr, output size and md5 of each run
  sweep   one committed baseline JPEG brought to total lengths around the 65535-byte block size by deterministic bytes
          after its EOI (the container keeps them as trailing garbage): the md5 of the JPEG, of the reference's .lep of it
          (-skipverify) and of that .lep restored with -zlib0.  The unpadded file is the one under one block.

Run where oracle/_ref/lepton exists (oracle/Makefile builds it from the reference tree):
    python tests/golden/make_zlib0.py
Only the JSON is written; the sweep's files are made again from sweep_jpeg() wherever they are needed.
"""
import hashlib
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_extremes import LEPTON, run_reference  # noqa: E402

OUT = os.path.join(HERE, "zlib0.json")
SWEEP_SOURCE = "androidcropoptions.jpg"
SWEEP_LENGTHS = [None, 65534, 65535, 65536, 131069, 131070, 131071, 196605]     # None: the JPEG as committed (one block)


def md5(b):
    return hashlib.md5(b).hexdigest()


def zeta(lep):
    """The zeta-headed twin of a .lep: the same container with CE B6 in front."""
    return b"\xce\xb6" + lep[2:]


def sweep_jpeg(total):
    """The sweep file of `total` bytes: the source JPEG, then bytes (37 i + 11) mod 256 up to that length."""
    src = open(os.path.join(HERE, SWEEP_SOURCE), "rb").read()
    if total is None:
        return src
    assert total >= len(src)
    return src + bytes((37 * i + 11) & 0xFF for i in range(total - len(src)))


def committed_leps():
    out = []
    for d, _, files in os.walk(HERE):
        for f in files:
            if f.endswith(".lep"):
                out.append(os.path.relpath(os.path.join(d, f), HERE))
    return sorted(out)


def restore(tmp, lep, flags):
    src, dst = os.path.join(tmp, "in.lep"), os.path.join(tmp, "out.jpg.z")
    with open(src, "wb") as f:
        f.write(lep)
    rc, name, out = run_reference(src, dst, flags)
    return {"rc": rc, "exit_name": name, "size": len(out), "md5": md5(out) if out else None}


def main():
    res = {"source": SWEEP_SOURCE, "leps": {}, "sweep": []}
    with tempfile.TemporaryDirectory() as tmp:
        for rel in committed_leps():
            lep = open(os.path.join(HERE, rel), "rb").read()
            res["leps"][rel] = {"plain": restore(tmp, lep, ["-zlib0"]), "zeta": restore(tmp, zeta(lep), [])}
        for total in SWEEP_LENGTHS:
            jpg = sweep_jpeg(total)
            src, dst = os.path.join(tmp, "s.jpg"), os.path.join(tmp, "s.lep")
            with open(src, "wb") as f:
                f.write(jpg)
            rc, name, lep = run_reference(src, dst)
            assert rc == 0 and name is None and lep, (total, rc, name)
            z = restore(tmp, lep, ["-zlib0"])
            assert z["rc"] == 0 and z["exit_name"] is None, (total, z)
            res["sweep"].append({"total": total, "jpg_len": len(jpg), "jpg_md5": md5(jpg), "lep_md5": md5(lep),
                                 "zlib0_size": z["size"], "zlib0_md5": z["md5"]})
    with open(OUT, "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)
        f.write("\n")
    ok = sum(e["plain"]["rc"] == 0 and e["plain"]["exit_name"] is None for e in res["leps"].values())
    print("%d .lep files (%d restored by the reference), %d sweep records -> %s" % (len(res["leps"]), ok, len(res["sweep"]), OUT))


if __name__ == "__main__":
    main()
