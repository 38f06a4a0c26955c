#!/usr/bin/env python
"""Regenerate tests/golden/ans_damaged.json: what the UNMODIFIED reference built with -DENABLE_ANS_EXPERIMENTAL
(oracle/_ref/lepton-ans, built by oracle/Makefile.ans) restores from damaged .lep files of container version 3 and from
their version-1 twins damaged at the same places.

The inputs are the fixtures of tests/golden/ans (tests/golden/make_ans.py) with bytes of their mux packets XORed: the
container (header, brotli / zlib header blob, packet headers, size trailer) stays intact, only stream bytes change.  Each
case picks one segment and one to three offsets inside its stream (some inside the 16 state bytes of the rANS stream), and
the same segment and stream offsets are damaged in the version-1 twin, so the two coders meet damage at the same places.
The damage is recorded as (file offset, XOR value) pairs on the committed fixture, with the md5 of the damaged file, so
the tests rebuild the inputs; no damaged file is committed.

Per case the record holds the reference's exit code and, where it is 0, the md5 of what it wrote.  Every case runs RUNS
times under a timeout; a case whose runs differ, or that times out, is left out and listed under "left_out" with the
reason, as are the cases of LEFT_OUT (below) with theirs.

Run where oracle/_ref/lepton-ans exists:
    python tests/golden/make_ans_damaged.py
"""
import hashlib
import json
import os
import random
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
LEPTON_ANS = os.path.join(ROOT, "oracle", "_ref", "lepton-ans")
ANS_DIR = os.path.join(HERE, "ans")
OUT = os.path.join(HERE, "ans_damaged.json")
TIMEOUT = 60
RUNS = 10


# Cases left out for a cause found by comparing with the oracle (oracle/oracle_ans.py, oracle/oracle.py) and by running
# the reference 30 to 40 times, which RUNS runs need not show.  The reference's custom_exit ends a thread with the SYS_exit
# system call, which on Linux ends the calling thread alone: an error met by one of the decoding threads of a
# multi-segment file reaches the process's exit code only as the threads' timing allows, and the bytes left behind are no
# restoration of the file.  The library reports the segment's status, as the oracle does.
LEFT_OUT = {
    "all22_tall_t8": "the last segment fails (oracle: 7 at decision 15214 of segment 7); the reference exits 0 or 7 from "
                     "run to run",
    "all22_tall_t8.v1": "the last segment fails (oracle: 7 in segment 7); the reference exits 0 with no bytes, or 7, from "
                        "run to run",
    "androidprogressive": "segment 0 fails; the reference exits 7 or 5 (THREAD_PROTOCOL_ERROR) from run to run",
    "androidprogressive.v1": "segment 0 fails; the reference exits 7, 5 (THREAD_PROTOCOL_ERROR) or 0 with no bytes "
                             "from run to run",
    "cut_grayscale_30000_t4": "the last segment fails (oracle: 7 at decision 121 of segment 3); the reference exits 0",
    "cut_grayscale_30000_t4.v1": "the last segment fails (oracle: 7 at decision 376 of segment 3); the reference exits 0 "
                                 "and writes no bytes",
}


def md5(b):
    return hashlib.md5(b).hexdigest()


def stream_positions(data):
    """File offset of every byte of every segment stream of a .lep of container version 1 or 3: the mux packets behind
    "CMP" (src/io/MuxReader.hh:230-283), up to the size trailer (or the end-of-file marker)."""
    zlen = int.from_bytes(data[24:28], "little")
    p, end = 31 + zlen, len(data) - 4
    assert data[p - 3:p] == b"CMP"
    pos = [[] for _ in range(16)]
    while p < end:
        if data[2] > 1 and data[p:p + 3] == b"\xff\xfe\xff":
            break
        h = data[p]
        sid, flags = h & 15, (h >> 4) & 3
        if flags == 0:
            ln, p = data[p + 1] + 256 * data[p + 2] + 1, p + 3
        else:
            ln, p = 1024 << (2 * flags), p + 1
        pos[sid] += range(p, min(p + ln, end))
        p += ln
    return pos[:data[4]]


def cases():
    """case name -> (fixture file, [(file offset, XOR value)]), a version-3 case and its version-1 twin for each of 20
    fixtures"""
    ans = json.load(open(os.path.join(HERE, "ans.json")))
    names = sorted(n for n, e in ans.items() if e["rc"] == 0 and not n.startswith("dense_"))[:20]
    rng = random.Random(2024)
    out = {}
    for n in names:
        v3, v1 = (open(os.path.join(ANS_DIR, n + ext), "rb").read() for ext in (".lep", ".v1.lep"))
        p3, p1 = stream_positions(v3), stream_positions(v1)
        seg = rng.randrange(len(p3))
        room = min(len(p3[seg]), len(p1[seg]))
        offs = sorted(rng.sample(range(room), min(room, 1 + rng.randrange(3))))
        if rng.random() < 0.3:
            offs = sorted(set(offs[1:] + [rng.randrange(min(16, room))]))     # one inside the rANS state bytes
        xors = [rng.randrange(1, 256) for _ in offs]
        out[n] = (n + ".lep", [(p3[seg][o], x) for o, x in zip(offs, xors)], seg, offs)
        out[n + ".v1"] = (n + ".v1.lep", [(p1[seg][o], x) for o, x in zip(offs, xors)], seg, offs)
    return out


def damaged(fixture, flips):
    b = bytearray(open(os.path.join(ANS_DIR, fixture), "rb").read())
    for off, x in flips:
        b[off] ^= x
    return bytes(b)


def restore(data, tmp):
    src, dst = os.path.join(tmp, "in.lep"), os.path.join(tmp, "out.jpg")
    with open(src, "wb") as f:
        f.write(data)
    if os.path.exists(dst):
        os.unlink(dst)
    try:
        r = subprocess.run([LEPTON_ANS, "-unjailed", src, dst], capture_output=True, timeout=TIMEOUT)
    except subprocess.TimeoutExpired:
        return None
    out = open(dst, "rb").read() if r.returncode == 0 and os.path.exists(dst) else b""
    return r.returncode, md5(out) if r.returncode == 0 else None


def main():
    res, left_out = {}, {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, (fixture, flips, seg, offs) in sorted(cases().items()):
            data = damaged(fixture, flips)
            got = [restore(data, tmp) for _ in range(RUNS)]
            if name in LEFT_OUT:
                left_out[name] = LEFT_OUT[name]
            elif None in got:
                left_out[name] = "the reference did not finish within %d s" % TIMEOUT
            elif len(set(got)) > 1:
                left_out[name] = "the reference's runs differ: %s" % sorted(set(got))
            else:
                res[name] = {"fixture": fixture, "flips": flips, "segment": seg, "stream_offsets": offs,
                             "input_md5": md5(data), "rc": got[0][0], "md5": got[0][1]}
            print(name, sorted(set(got), key=str), flush=True)
    with open(OUT, "w") as f:
        json.dump({"cases": res, "left_out": left_out}, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
