"""TEST INFRASTRUCTURE ONLY: ctypes bindings of the oracle with the rANS coder of container version 3
(oracle/_build/liblepton_oracle_ans.so, built by oracle/Makefile.ans).  Same geometry and plane conventions as oracle.py."""
import ctypes
import os
import subprocess

import numpy as np

from oracle import Geometry, _ptrs, make_geometry  # noqa: F401  (make_geometry: the geometry this module takes)

HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
_SOURCES = ["lepton_oracle.c", "lepton_oracle_ans.c", "lepton_oracle_ans.h", "Makefile.ans"]


def lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(HERE, "_build", "liblepton_oracle_ans.so")
        if not os.path.exists(path) or any(os.path.getmtime(path) < os.path.getmtime(os.path.join(HERE, s)) for s in _SOURCES):
            subprocess.check_call(["make", "-s", "-f", os.path.join(HERE, "Makefile.ans"), path])
        L = ctypes.CDLL(path)
        P3 = ctypes.c_void_p * 3
        L.lo_encode_segment_ans.argtypes = [ctypes.POINTER(Geometry), P3, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                            ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t),
                                            ctypes.POINTER(ctypes.c_uint64)]
        L.lo_encode_segment_ans.restype = ctypes.c_int
        L.lo_decode_segment_ans.argtypes = [ctypes.POINTER(Geometry), P3, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                            ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint64)]
        L.lo_decode_segment_ans.restype = ctypes.c_int
        L.lo_decode_segment_ans_trace.argtypes = L.lo_decode_segment_ans.argtypes + [ctypes.c_void_p, ctypes.c_size_t]
        L.lo_decode_segment_ans_trace.restype = ctypes.c_int
        L.lo_ans_encode.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t)]
        L.lo_ans_encode.restype = ctypes.c_int
        _LIB = L
    return _LIB


def encode_segment(g: Geometry, planes, min_y, max_y, is_last, cap=None):
    """One thread-segment coded with the rANS coder -> (exit_code, stream bytes, ndecisions)."""
    cap = cap or 4 * sum(p.size for p in planes) + 4096        # at most one 4-byte word per decision
    out = np.zeros(cap, dtype=np.uint8)
    n = ctypes.c_size_t(0)
    nd = ctypes.c_uint64(0)
    rc = lib().lo_encode_segment_ans(ctypes.byref(g), _ptrs(planes), min_y, max_y, int(is_last), out.ctypes.data, cap,
                                     ctypes.byref(n), ctypes.byref(nd))
    return rc, out[:n.value].tobytes(), nd.value


def decode_segment(g: Geometry, planes, min_y, max_y, is_last, stream: bytes):
    """Decodes an rANS-coded segment stream in place into planes. -> (exit_code, ndecisions)"""
    buf = np.frombuffer(stream, dtype=np.uint8)
    nd = ctypes.c_uint64(0)
    rc = lib().lo_decode_segment_ans(ctypes.byref(g), _ptrs(planes), min_y, max_y, int(is_last),
                                     buf.ctypes.data if len(buf) else None, len(buf), ctypes.byref(nd))
    return rc, nd.value


# lo_ans_step (lepton_oracle_ans.h): one decision of a decode
TRACE_DTYPE = np.dtype([("x_before", "<u8"), ("x_after", "<u8"), ("word_off", "<i8"), ("prob", "u1"), ("bit", "u1"),
                        ("c0", "u1"), ("c1", "u1"), ("pad", "u1", 4)])
assert TRACE_DTYPE.itemsize == 32


def decode_segment_trace(g: Geometry, planes, min_y, max_y, is_last, stream: bytes):
    """decode_segment with a record of every decision -> (exit_code, ndecisions, trace): trace is a TRACE_DTYPE array, one
    entry per decision: the probability, the bit, the branch counts before the update (c0, c1), the state the decision
    reads (x_before) and that state advanced and refilled (x_after), and the stream offset of the word the refill took
    (word_off, -1 without a refill)."""
    rc, nd = decode_segment(g, planes, min_y, max_y, is_last, stream)     # sizes the trace; decoding again writes the same
    buf = np.frombuffer(stream, dtype=np.uint8)
    trace = np.zeros(max(nd, 1), TRACE_DTYPE)
    n = ctypes.c_uint64(0)
    rc2 = lib().lo_decode_segment_ans_trace(ctypes.byref(g), _ptrs(planes), min_y, max_y, int(is_last),
                                            buf.ctypes.data if len(buf) else None, len(buf), ctypes.byref(n),
                                            trace.ctypes.data, len(trace))
    assert (rc2, n.value) == (rc, nd)
    return rc, nd, trace[:nd]


def ans_encode(tokens, cap=None):
    """The rANS writer alone over `tokens` (uint16: prob | bit << 8), coded in reverse like the reference's
    ANSBoolWriter::finish.  -> (exit_code, stream bytes); 1 for a token of probability 0, 100 when the stream does not
    fit `cap` bytes (default: always fits)."""
    t = np.ascontiguousarray(tokens, dtype=np.uint16)
    cap = cap or 4 * len(t) + 64
    out = np.zeros(cap, dtype=np.uint8)
    n = ctypes.c_size_t(0)
    rc = lib().lo_ans_encode(t.ctypes.data if len(t) else None, len(t), out.ctypes.data, cap, ctypes.byref(n))
    return rc, out[:n.value].tobytes()
