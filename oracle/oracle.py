"""TEST INFRASTRUCTURE ONLY -- ctypes binding of oracle/_build/liblepton_oracle.so (oracle/lepton_oracle.c).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import this module; the product
(lepton_b200/) never does.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


class Geometry(ctypes.Structure):
    _fields_ = [
        ("ncmp", ctypes.c_int32),
        ("bch", ctypes.c_int32 * 3),
        ("bcv", ctypes.c_int32 * 3),
        ("trunc_bcv", ctypes.c_int32 * 3),
        ("trunc_bc", ctypes.c_int32 * 3),
        ("mcuv", ctypes.c_int32),
        ("q_zigzag", (ctypes.c_uint16 * 64) * 3),
    ]


def build():
    subprocess.check_call(["make", "-s", "-C", HERE, os.path.join(HERE, "_build", "liblepton_oracle.so")])


def lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(HERE, "_build", "liblepton_oracle.so")
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(os.path.join(HERE, "lepton_oracle.c")):
            build()
        L = ctypes.CDLL(path)
        P3 = ctypes.c_void_p * 3
        L.lo_encode_segment.argtypes = [ctypes.POINTER(Geometry), P3, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                        ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t),
                                        ctypes.POINTER(ctypes.c_uint64)]
        L.lo_encode_segment.restype = ctypes.c_int
        L.lo_decode_segment.argtypes = [ctypes.POINTER(Geometry), P3, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                        ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint64)]
        L.lo_decode_segment.restype = ctypes.c_int
        _LIB = L
    return _LIB


def make_geometry(ncmp, bch, bcv, mcuv, qtables_zigzag, trunc_bcv=None, trunc_bc=None) -> Geometry:
    g = Geometry()
    g.ncmp = ncmp
    g.mcuv = mcuv
    for c in range(ncmp):
        g.bch[c] = bch[c]
        g.bcv[c] = bcv[c]
        g.trunc_bcv[c] = trunc_bcv[c] if trunc_bcv else bcv[c]
        g.trunc_bc[c] = trunc_bc[c] if trunc_bc else bch[c] * bcv[c]
        for i in range(64):
            g.q_zigzag[c][i] = int(qtables_zigzag[c][i])
    return g


def _ptrs(planes):
    P3 = ctypes.c_void_p * 3
    arr = P3()
    for i, p in enumerate(planes):
        assert p.dtype == np.int16 and p.flags["C_CONTIGUOUS"]
        arr[i] = p.ctypes.data
    return arr


def encode_segment(g: Geometry, planes, min_y, max_y, is_last, cap=None):
    """-> (exit_code, stream bytes, ndecisions)"""
    nbytes = sum(p.nbytes for p in planes)
    cap = cap or max(1 << 16, nbytes)
    out = np.zeros(cap, dtype=np.uint8)
    n = ctypes.c_size_t(0)
    nd = ctypes.c_uint64(0)
    rc = lib().lo_encode_segment(ctypes.byref(g), _ptrs(planes), min_y, max_y, int(is_last), out.ctypes.data, cap,
                                 ctypes.byref(n), ctypes.byref(nd))
    return rc, out[:n.value].tobytes(), nd.value


def decode_segment(g: Geometry, planes, min_y, max_y, is_last, stream: bytes):
    """Decodes in place into planes (list of int16 [nblocks,64] arrays). -> (exit_code, ndecisions)"""
    buf = np.frombuffer(stream, dtype=np.uint8)
    nd = ctypes.c_uint64(0)
    rc = lib().lo_decode_segment(ctypes.byref(g), _ptrs(planes), min_y, max_y, int(is_last),
                                 buf.ctypes.data if len(buf) else None, len(buf), ctypes.byref(nd))
    return rc, nd.value


def bool_encode(tokens, cap=None):
    """The bool coder alone over `tokens` (uint16: prob | bit << 8), marker bit and stop rule included.
    -> (exit_code, stream bytes); exit code 100 when the stream does not fit `cap` bytes (default: always fits)."""
    L = lib()
    L.lo_bool_encode.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t)]
    L.lo_bool_encode.restype = ctypes.c_int
    t = np.ascontiguousarray(tokens, dtype=np.uint16)
    cap = cap or len(t) + 64          # a decision shifts at most 7 bits: < 1 byte each
    out = np.zeros(cap, dtype=np.uint8)
    n = ctypes.c_size_t(0)
    rc = L.lo_bool_encode(t.ctypes.data if len(t) else None, len(t), out.ctypes.data, cap, ctypes.byref(n))
    return rc, out[:n.value].tobytes()


def bool_counts(reset=False):
    """Bool-coder regimes reached since the last reset, by bool_encode and encode_segment alike: longest carry walk
    (bytes a carry changed), carry walks of 64 bytes or more, streams that ended with the extra zero byte of the stop rule."""
    L = lib()
    out = (ctypes.c_uint64 * 3)()
    L.lo_bool_counts(out)
    if reset:
        L.lo_bool_counts_reset()
    return dict(walk_max=int(out[0]), walks_64=int(out[1]), stop_zero=int(out[2]))


def regime_counts(reset=False):
    """{site: count} since the last reset: how often each place where the reference's arithmetic wraps, truncates or
    caps (int32 IDCT, int16 pixels and edges, uint32 Lakhani sum, context masks and caps, DC wrap, status 6) produced a
    value different from the exact one, over every segment the oracle coded.  reset=True clears them afterwards."""
    L = lib()
    L.lo_regime_name.restype = ctypes.c_char_p
    L.lo_regime_value.restype = ctypes.c_uint64
    out = {L.lo_regime_name(i).decode(): int(L.lo_regime_value(i)) for i in range(L.lo_regime_count())}
    if reset:
        L.lo_regime_reset()
    return out
