"""The rANS decode kernels (container version 3) on the device at the coder's own edges: stream tails next to stale bytes,
the renormalisation boundary, saturated models, batches whose bool and rANS parts take different kernels, and one context
reused across batches of both coders.

The batches are the builders of tests/test_emu_ans.py, whose twins run them on the CPU warp emulator; each builder's
coverage assertion (through the oracle's per-decision trace) shows the batch reaches its edge.  Every batch is judged by
ans_helpers.judge: status, decision count and planes of every segment against the oracle of its coder.  What only the
device shows: the stream arena and the pinned staging buffer behind each stream hold whatever earlier batches left there,
CTAs run together on shared queues, and the library's own launch code picks each part's kernel and resets its counter.
"""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import test_emu_ans as edges  # noqa: E402
from ans_helpers import judge  # noqa: E402
from test_gpu_kernel_edges import DEC_FORMS, ONE_LAUNCH_FORMS, codec_with, device_run  # noqa: E402

pytestmark = pytest.mark.gpu

ANS, BOOL = edges.ANS, edges.BOOL


@pytest.fixture(params=list(DEC_FORMS))
def decoder(request, monkeypatch):
    c = codec_with(monkeypatch, DEC_FORMS[request.param])
    yield c
    c.close()


def stale_batch():
    """One-segment rANS images with long 0xFF streams: decoded first, they leave 0xFF in the staging buffer and the
    device stream arena where the next batch's short streams and their padding lie."""
    imgs, _, _ = edges.stream_length_batch()
    return imgs, [[b"\xff" * (600 + 8 * (i % 5))] for i in range(len(imgs))], [ANS] * len(imgs)


def gather_run(codec, rng):
    """judge's run through lepb200_decode_upload_gather_coded: every stream handed over in spans of 1..40 bytes, as the
    mux packets of a file lie."""
    from lepton_b200.codec import _Buffer, _Stream
    L = codec._L
    L.lepb200_decode_upload_gather_coded.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                                     ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    L.lepb200_decode_upload_gather_coded.restype = ctypes.c_int

    def run(out, streams, coders):
        segs = [s for ss in streams for s in ss]
        pieces, first = [], [0]
        for s in segs:
            o = 0
            while o < len(s):
                n = int(rng.integers(1, 41))
                pieces.append(s[o:o + n])
                o += n
            first.append(len(pieces))
        keep = [np.frombuffer(p, np.uint8) for p in pieces]
        spans = (_Buffer * max(1, len(pieces)))()
        for k, p in enumerate(keep):
            spans[k].data, spans[k].len = p.ctypes.data, len(p)
        ins = (_Stream * len(segs))()
        for k, s in enumerate(segs):
            ins[k].data, ins[k].len = None, len(s)
        span_first = (ctypes.c_uint32 * len(first))(*first)
        cod = (ctypes.c_uint8 * len(out))(*coders)
        codec._dec_imgs, codec._dec_c = out, codec._c_images(out)
        codec._check(L.lepb200_decode_upload_gather_coded(codec._ctx, codec._dec_c, len(out), ins, spans, span_first, cod),
                     "decode_upload_gather_coded")
        codec.decode_launch()
        st = codec.decode_fetch()
        return st, codec.decode_decisions()
    return run


def test_streams_of_every_length_next_to_stale_bytes(decoder):
    """The stream-length batch after a batch of long 0xFF streams in the same context, through both upload paths: a
    partial last word must be masked against whatever lies behind it, not only against zeros."""
    imgs, streams, coders = edges.stream_length_batch()
    edges.assert_stream_tails(imgs, streams)
    rng = np.random.default_rng(12)
    for run in (device_run(decoder), gather_run(decoder, rng)):
        judge(device_run(decoder), *stale_batch())
        judge(run, imgs, streams, coders)


def test_renormalisation_boundary(decoder):
    imgs, streams, coders = edges.renorm_boundary_batch()
    edges.assert_renorm_edges(imgs, streams)
    judge(device_run(decoder), imgs, streams, coders)


@pytest.mark.parametrize("form", list(ONE_LAUNCH_FORMS))
def test_saturated_models(monkeypatch, form):
    imgs, streams, coders = edges.saturated_batch()
    edges.assert_saturation(imgs, streams)
    c = codec_with(monkeypatch, ONE_LAUNCH_FORMS[form])
    try:
        judge(device_run(c), imgs, streams, coders)
    finally:
        c.close()


# (environment, bool segments, rANS segments): the library's size switch sends each part to its own kernel
SPLITS = {
    "bool-group+ans-warp": ({"LEPB200_DEC_GROUP_MIN": "64"}, 70, 9),
    "bool-warp+ans-group": ({"LEPB200_DEC_GROUP_MIN": "64"}, 9, 70),
    "bool-warp+ans-group-default-switch": ({}, 7, 6145),
    "both-group-several-launches": ({"LEPB200_DEC_MODE": "2", "LEPB200_DEC_THREADS": "32"}, 75, 70),
    "ans-part-of-one-segment-warp": ({"LEPB200_DEC_MODE": "1"}, 20, 1),
    "ans-part-of-one-segment-group": ({"LEPB200_DEC_MODE": "2", "LEPB200_DEC_THREADS": "32"}, 20, 1),
    "coders-all-bool": ({"LEPB200_DEC_GROUP_MIN": "64"}, 70, 0),
}


@pytest.mark.parametrize("split", list(SPLITS))
def test_coder_parts_on_different_kernels(monkeypatch, split):
    """Mixed batches, the two coders' images interleaved in batch order: every image equals its own coder's oracle
    whichever kernel each part takes, however many launches it needs, and when the rANS part is the second launch that
    resets the work counter itself."""
    env, n_bool, n_ans = SPLITS[split]
    imgs, streams, coders = edges.split_batch(n_bool, n_ans)
    c = codec_with(monkeypatch, env)
    try:
        judge(device_run(c), imgs, streams, coders)
    finally:
        c.close()


def test_context_reused_across_coders_sizes_and_kernels(monkeypatch):
    """One context decodes rANS, bool, rANS and mixed batches of different sizes in turn, so the warp and the group
    kernel alternate on its model pool, row pool, work counter and stream arena: every batch decodes as on a fresh
    context (the oracle's results)."""
    c = codec_with(monkeypatch, {"LEPB200_DEC_GROUP_MIN": "64"})
    try:
        for n_bool, n_ans in ((0, 70), (9, 0), (0, 9), (70, 9), (0, 70), (9, 70), (70, 0)):
            judge(device_run(c), *edges.split_batch(n_bool, n_ans, seed=90))
    finally:
        c.close()
