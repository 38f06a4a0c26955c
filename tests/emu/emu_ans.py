"""The decode kernels with the rANS coder of container version 3 on the CPU warp emulator (test infrastructure): the
harness emu_ans_kernels.cc, built like emu.py's, with a coder per image."""
import ctypes
import os
import subprocess

import numpy as np

import emu

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_build", "libemu_ans_kernels.so")
SOURCES = [os.path.join(HERE, "emu_ans_kernels.cc")] + emu.SOURCES[1:]

CODER_BOOL, CODER_ANS = 0, 1          # LEPB200_CODER_BOOL / LEPB200_CODER_ANS
KERNEL_WARP, KERNEL_G2 = emu.KERNEL_WARP, emu.KERNEL_G2

_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        if not (os.path.exists(OUT) and all(os.path.getmtime(OUT) >= os.path.getmtime(s) for s in SOURCES)):
            os.makedirs(os.path.dirname(OUT), exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", "-I", os.path.join(HERE, "fake"),
                                   "-Wno-unknown-pragmas", "-o", OUT, os.path.join(HERE, "emu_ans_kernels.cc")])
        _LIB = ctypes.CDLL(OUT)
        _LIB.emu_decode_images_coded.restype = ctypes.c_int
    return _LIB


def decode_images(kernel, images, streams, coders, grid_cap=0, reverse=False):
    """emu.decode_images with the entropy coder of every image's streams (CODER_BOOL, CODER_ANS): decodes into
    images[i].planes, returns (status, ndecisions) per segment."""
    from lepton_b200.codec import _Image, _Stream
    assert len(coders) == len(images)
    n = sum(im.nseg for im in images)
    arr = (_Stream * n)()
    keep, k = [], 0
    for im, segs in zip(images, streams):
        assert len(segs) == im.nseg
        for s in segs:
            buf = np.frombuffer(bytes(s), dtype=np.uint8)
            keep.append(buf)
            arr[k].data = buf.ctypes.data if len(buf) else None
            arr[k].len = len(buf)
            k += 1
    cim = (_Image * len(images))(*[im.to_c() for im in images])
    cod = (ctypes.c_uint8 * len(images))(*[int(c) for c in coders])
    st = (ctypes.c_int32 * n)()
    nd = (ctypes.c_uint64 * n)()
    rc = lib().emu_decode_images_coded(int(kernel), int(grid_cap), int(bool(reverse)), cim, len(images), arr, cod, st, nd)
    if rc != 0:
        raise RuntimeError("emu_decode_images_coded failed with %d" % rc)
    return list(st), list(nd)
