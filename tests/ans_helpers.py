"""Shared helpers of the rANS (container version 3) tests: the fixtures of tests/golden/ans (tests/golden/make_ans.py), and
the oracle's streams, decodes and per-decision traces of synthetic images that the emulator and device tests judge with.

Each fixture <case>.lep has a version-1 twin <case>.v1.lep, written by the reference from the same input and flags: same
segments, same decisions.  The twin's zlib header blob gives the geometry and the handoffs, so nothing here needs a brotli
decoder; the rANS streams are demuxed from the version-3 file itself."""
import json
import os
import struct

import numpy as np

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


# ---------------------------------------------------------------------------------------------------- random images
def image_geometry(img):
    """The oracle's geometry of a lepton_b200.CoefImage, truncation included."""
    import oracle
    return oracle.make_geometry(img.ncmp, list(img.bch), list(img.bcv), img.mcuv, img.qtables_zigzag,
                                list(img.trunc_bcv) if img.trunc_bcv is not None else None,
                                list(img.trunc_bc) if img.trunc_bc is not None else None)


def image_segments(img):
    """(min_y, max_y, is_last) of every thread-segment of a CoefImage"""
    starts = list(img.luma_y_start)
    return [(y0, img.bcv[0] if i == len(starts) - 1 else starts[i + 1], i == len(starts) - 1) for i, y0 in enumerate(starts)]


def oracle_ans_streams(imgs):
    """The oracle's rANS streams of every image's segments (each must code with status 0)."""
    import oracle_ans
    out = []
    for img in imgs:
        g = image_geometry(img)
        ref = [oracle_ans.encode_segment(g, img.planes, *seg) for seg in image_segments(img)]
        assert all(rc == 0 for rc, _, _ in ref)
        out.append([s for _, s, _ in ref])
    return out


def oracle_decode_image(img, streams, coder=1, trace=False):
    """What the oracle decodes from an image's segment streams with the bool coder (coder 0) or the rANS coder (coder 1)
    -> (status, decision count of every segment, planes[, traces of the rANS decisions]).  A segment that fails leaves its
    blocks as far as the oracle wrote them, and the next segment is decoded all the same (as the kernels do); blocks
    nothing codes stay zero."""
    import oracle
    import oracle_ans
    g = image_geometry(img)
    planes = [np.zeros_like(p) for p in img.planes]
    status, nd, traces = [], [], []
    for seg, s in zip(image_segments(img), streams):
        if trace:
            assert coder == 1
            rc, n, t = oracle_ans.decode_segment_trace(g, planes, *seg, s)
            traces.append(t)
        else:
            rc, n = (oracle_ans if coder == 1 else oracle).decode_segment(g, planes, *seg, s)
        status.append(rc)
        nd.append(n)
    return (status, nd, planes, traces) if trace else (status, nd, planes)


def blank_like(img, fill=-5):
    """A CoefImage of img's geometry whose planes hold `fill`, for a decode to write into."""
    from lepton_b200 import CoefImage
    return CoefImage(ncmp=img.ncmp, mcuv=img.mcuv, bch=img.bch, bcv=img.bcv, qtables_zigzag=img.qtables_zigzag,
                     planes=[np.full_like(p, fill) for p in img.planes], luma_y_start=img.luma_y_start,
                     trunc_bcv=img.trunc_bcv, trunc_bc=img.trunc_bc)


ZERO_IDCT_0 = 43        # status of a segment the host refuses: a zero quantiser in the first row or column (model.hh:257-262)


def judge(run, imgs, streams, coders=None, refused=()):
    """Decodes one batch with run(out_images, streams, coders) -> (status, decision count per segment) and holds every
    segment's status and decision count, and every image's planes, to the oracle of the image's coder (coders: per image,
    0 bool / 1 rANS; None = all bool, passed on as it is).  The planes are compared whether the segments end well or not:
    the kernels write the blocks a failing segment reached, as the oracle does.  The images of `refused` have a zero
    quantiser: the host refuses their segments with ZERO_IDCT_0 before any decision and their planes stay zero (the
    oracle cannot judge them: like the reference's decoder it does not check, and divides by zero).  -> the statuses."""
    out = [blank_like(i) for i in imgs]
    st, nd = run(out, streams, coders)
    assert len(st) == len(nd) == sum(i.nseg for i in imgs)
    k, all_st = 0, []
    for i, (img, o, ss) in enumerate(zip(imgs, out, streams)):
        c = coders[i] if coders is not None else 0
        if i in refused:
            want_st, want_nd, want = [ZERO_IDCT_0] * img.nseg, [0] * img.nseg, [np.zeros_like(p) for p in img.planes]
        else:
            want_st, want_nd, want = oracle_decode_image(img, ss, c)
        n = img.nseg
        assert (st[k:k + n], nd[k:k + n]) == (want_st, want_nd), (i, c, st[k:k + n], want_st, nd[k:k + n], want_nd)
        for ci in range(img.ncmp):
            assert np.array_equal(o.planes[ci], want[ci]), (i, c, ci, np.nonzero(np.any(o.planes[ci] != want[ci], axis=1))[0][:8])
        all_st += want_st
        k += n
    return all_st


def traces(imgs, streams):
    """The oracle's per-decision traces of every segment of rANS-coded images, concatenated (oracle_ans.TRACE_DTYPE),
    with the length of each decision's stream in a field of its own (`len`)."""
    import numpy.lib.recfunctions as rf
    out = []
    for img, ss in zip(imgs, streams):
        for t, s in zip(oracle_decode_image(img, ss, 1, trace=True)[3], ss):
            out.append(rf.append_fields(t, "len", np.full(len(t), len(s), np.int64), usemask=False))
    return np.concatenate(out)


def advanced(t):
    """The state each traced decision advanced to, before its refill."""
    return np.where(t["word_off"] >= 0, t["x_after"] >> np.uint64(32), t["x_after"])
