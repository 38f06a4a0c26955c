"""The encode side of container version 3 (rANS) on the CPU warp emulator (test infrastructure): the harness
emu_ans_encode.cc, built like emu.py's -- kernel A with the rANS model, the rANS pass, their launches per coder, and the
pass's division and output bound."""
import ctypes
import os
import subprocess

import numpy as np

import emu

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_build", "libemu_ans_encode.so")
SOURCES = [os.path.join(HERE, "emu_ans_encode.cc")] + emu.SOURCES

CODER_BOOL, CODER_ANS = 0, 1          # LEPB200_CODER_BOOL / LEPB200_CODER_ANS

_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        if not (os.path.exists(OUT) and all(os.path.getmtime(OUT) >= os.path.getmtime(s) for s in SOURCES)):
            os.makedirs(os.path.dirname(OUT), exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", "-I", os.path.join(HERE, "fake"),
                                   "-Wno-unknown-pragmas", "-o", OUT, os.path.join(HERE, "emu_ans_encode.cc")])
        L = ctypes.CDLL(OUT)
        L.emu_encode_images_coded.restype = ctypes.c_int
        L.emu_ans_pass.restype = ctypes.c_int
        L.emu_ans_divide.restype = None
        L.emu_ans_stream_bound.restype = ctypes.c_uint64
        L.emu_ans_stream_bound.argtypes = [ctypes.c_uint64]
        L.emu_ans_slot_fits.restype = ctypes.c_int
        L.emu_ans_slot_fits.argtypes = [ctypes.c_uint64, ctypes.c_uint64]
        _LIB = L
    return _LIB


def encode_images(images, coders=None, kernel=0, grid_cap=0, reverse=False, token_bounds=None):
    """emu.encode_images with the coder of every image (CODER_BOOL, CODER_ANS; None = all bool): per image a list of
    (status, bytes, ndecisions) per segment, and the token slot of every segment.  token_bounds: per image, the caller's
    token bound of every segment (lepb200_image::seg_token_bound; then no counting pre-pass)."""
    from lepton_b200.codec import _Image, _Stream
    n = sum(im.nseg for im in images)
    cim = (_Image * len(images))(*[im.to_c() for im in images])
    for i, tb in enumerate(token_bounds or []):
        for k, v in enumerate(tb):
            cim[i].seg_token_bound[k] = int(v)
    cod = None if coders is None else (ctypes.c_uint8 * len(images))(*[int(c) for c in coders])
    out = (_Stream * n)()
    cap = sum(im.blocks() for im in images) * 128 + 8192 * n
    arena = (ctypes.c_uint8 * cap)()
    tc = (ctypes.c_uint32 * n)()
    rc = lib().emu_encode_images_coded(int(kernel), int(grid_cap), int(bool(reverse)), cim, len(images), cod, out, arena,
                                       ctypes.c_size_t(cap), tc)
    if rc != 0:
        raise RuntimeError("emu_encode_images_coded failed with %d" % rc)
    res, k = [], 0
    for im in images:
        segs = []
        for _ in range(im.nseg):
            o = out[k]
            segs.append((o.status, ctypes.string_at(o.data, o.len) if o.len else b"", int(o.ndecisions)))
            k += 1
        res.append(segs)
    return res, list(tc)


def ans_pass(streams, tok_caps=None, reverse=False):
    """The rANS pass alone: streams = uint16 token arrays (prob | bit << 8); tok_caps = token slot of each (None or 0: the
    library's token_slot).  -> (per segment (status, bytes), canary tokens behind the slots that changed)."""
    toks = [np.ascontiguousarray(t, dtype=np.uint16) for t in streams]
    n = len(toks)
    flat = np.concatenate(toks + [np.zeros(1, np.uint16)])
    nt = (ctypes.c_uint32 * n)(*[len(t) for t in toks])
    tc = (ctypes.c_uint32 * n)(*[int(c or 0) for c in (tok_caps or [0] * n)])
    st = (ctypes.c_int32 * n)()
    ln = (ctypes.c_uint32 * n)()
    out_cap = sum(len(t) for t in toks) + 64 * n + 64
    out = (ctypes.c_uint8 * out_cap)()
    bad = ctypes.c_uint64(0)
    rc = lib().emu_ans_pass(int(bool(reverse)), n, flat.ctypes.data_as(ctypes.c_void_p), nt, tc, st, ln, out, ctypes.c_size_t(out_cap),
                            ctypes.byref(bad))
    if rc != 0:
        raise RuntimeError("emu_ans_pass failed with %d" % rc)
    raw, res, pos = bytes(out), [], 0
    for s in range(n):
        res.append((st[s], raw[pos:pos + ln[s]]))
        pos += ln[s]
    return res, bad.value


def ans_divide(x, f):
    """The pass's division: (x // f, x % f) for uint64 arrays x (< 2^63) and f (1..256)."""
    x = np.ascontiguousarray(x, dtype=np.uint64)
    f = np.ascontiguousarray(f, dtype=np.uint32)
    q = np.zeros(len(x), np.uint64)
    r = np.zeros(len(x), np.uint32)
    lib().emu_ans_divide(len(x), x.ctypes.data_as(ctypes.c_void_p), f.ctypes.data_as(ctypes.c_void_p),
                         q.ctypes.data_as(ctypes.c_void_p), r.ctypes.data_as(ctypes.c_void_p))
    return q, r


def stream_bound(ntok):
    return int(lib().emu_ans_stream_bound(int(ntok)))


def slot_fits(ntok, tok_cap):
    return bool(lib().emu_ans_slot_fits(int(ntok), int(tok_cap)))


def ans_put(x, tok):
    """One decision of the pass on states x (uint64) with tokens tok (prob | bit << 8) -> (states after, words, emitted)."""
    x = np.ascontiguousarray(x, dtype=np.uint64)
    tok = np.ascontiguousarray(tok, dtype=np.uint16)
    xo = np.zeros(len(x), np.uint64)
    w = np.zeros(len(x), np.uint32)
    e = np.zeros(len(x), np.uint8)
    lib().emu_ans_put(len(x), x.ctypes.data_as(ctypes.c_void_p), tok.ctypes.data_as(ctypes.c_void_p), xo.ctypes.data_as(ctypes.c_void_p),
                      w.ctypes.data_as(ctypes.c_void_p), e.ctypes.data_as(ctypes.c_void_p))
    return xo, w, e.astype(bool)
