"""Shared helpers of the rANS (container version 3) tests: the fixtures of tests/golden/ans (tests/golden/make_ans.py).

Each fixture <case>.lep has a version-1 twin <case>.v1.lep, written by the reference from the same input and flags: same
segments, same decisions.  The twin's zlib header blob gives the geometry and the handoffs, so nothing here needs a brotli
decoder; the rANS streams are demuxed from the version-3 file itself."""
import json
import os
import struct

import lepfmt
from helpers import GOLDEN, oracle_decode_planes

ANS = json.load(open(os.path.join(GOLDEN, "ans.json")))
ANS_DIR = os.path.join(GOLDEN, "ans")


def ans_cases():
    """The cases the reference wrote a version-3 file for."""
    return sorted(n for n, e in ANS.items() if e["rc"] == 0)


def ans_streams(data):
    """The per-segment streams of a version-3 .lep (the mux packets behind CMP, up to the EOF marker)."""
    assert data[2] == 3
    zlen = struct.unpack("<I", data[24:28])[0]
    assert data[28 + zlen:31 + zlen] == b"CMP"
    return lepfmt.demux(data[31 + zlen:-4], 3)[:data[4]]


def load_ans_case(name):
    """(twin LepFile, the oracle's planes of the twin, its bool streams, the version-3 file's rANS streams, its bytes)"""
    ans = open(os.path.join(ANS_DIR, name + ".lep"), "rb").read()
    lf = lepfmt.parse_container(open(os.path.join(ANS_DIR, name + ".v1.lep"), "rb").read())
    planes, bool_streams = oracle_decode_planes(lf)
    assert lf.nseg == ans[4]
    return lf, planes, bool_streams[:lf.nseg], ans_streams(ans), ans
