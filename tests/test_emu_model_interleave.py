"""The interleaved model pool of the group decode kernel (lep_common.cuh: mi_offset, mi_model, mi_width), on the
CPU warp emulator (tests/emu) against the oracle.

The models of MI_K consecutive jobs share one block, unit by unit, and the groups of a warp claim their jobs together.
A job's model must still be its own: the offset function has to be a bijection over a pool of any size (a partial last
block holds only the models that are left, so the pool stays n models long), and a group that takes a second job, at
whatever position in a block, must start from a zero model and leave its neighbours' words alone.
"""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")
sys.path.insert(0, EMU)
import emu  # noqa: E402
from helpers import oracle_encode_image, random_coef_image  # noqa: E402


HOST_SRC = r"""
#include "cuda_shim.h"
#include "%s"
using namespace lepb200;
// Places every word of every model of a pool of n jobs (mi_model, mi_width, mi_offset) and records, at each u16 offset of the
// pool, the job and the word stored there (job_at / word_at: n * M_TOTAL entries, -1 on entry).  Returns MI_K, or -1 when an
// offset falls outside the pool or is produced twice.
extern "C" int place_pool(int n, int32_t* job_at, int32_t* word_at) {
    for (int j = 0; j < n; ++j) {
        const size_t base = mi_model((size_t)j, (size_t)n);
        const uint32_t width = mi_width((size_t)j, (size_t)n);
        for (uint32_t w = 0; w < M_TOTAL; ++w) {
            const size_t off = base + mi_offset(w, 0, width);
            if (off >= (size_t)n * M_TOTAL || job_at[off] != -1) return -1;
            job_at[off] = j; word_at[off] = (int32_t)w;
        }
    }
    return (int)MI_K;
}
extern "C" uint32_t model_words() { return M_TOTAL; }
"""


@pytest.fixture(scope="module")
def placement(tmp_path_factory):
    """place_pool of lep_common.cuh compiled for the host, as shipped and with -DLEPB200_MODEL_INTERLEAVE=1"""
    tmp = tmp_path_factory.mktemp("interleave")
    src = tmp / "place.cc"
    src.write_text(HOST_SRC % os.path.join(ROOT, "lepton_b200", "csrc", "lep_common.cuh"))
    libs = {}
    for name, defs in (("shipped", []), ("k1", ["-DLEPB200_MODEL_INTERLEAVE=1"])):
        so = str(tmp / ("place_%s.so" % name))
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", "-I", EMU, "-I", os.path.join(EMU, "fake"),
                               "-Wno-unknown-pragmas"] + defs + ["-o", so, str(src)])
        libs[name] = ctypes.CDLL(so)
        libs[name].model_words.restype = ctypes.c_uint32

    def place(name, n):
        lib = libs[name]
        m = lib.model_words()
        job = np.full(n * m, -1, np.int32)
        word = np.full(n * m, -1, np.int32)
        k = lib.place_pool(n, job.ctypes.data_as(ctypes.c_void_p), word.ctypes.data_as(ctypes.c_void_p))
        assert k > 0, "an offset lies outside the pool or is produced twice"
        return k, m, job, word
    return place


@pytest.mark.parametrize("n", [8, 13, 3])
def test_offset_function_is_a_bijection_over_a_pool(placement, n):
    """Whole blocks and a partial last one: every offset of the n-model pool holds exactly one word of one model, word
    pairs stay together, and a block of W models puts unit u of model k at unit u * W + k."""
    k, m, job, word = placement("shipped", n)
    assert k == 8
    assert np.all(job >= 0)                                              # onto: the pool is exactly n models long
    for j in range(n):
        assert np.array_equal(np.sort(word[job == j]), np.arange(m, dtype=np.int32))
    off = np.arange(n * m)
    blk = off // (k * m)
    width = np.minimum(k, n - blk * k)
    rel = off - blk * k * m
    assert np.array_equal(job, blk * k + rel // 2 % width)
    assert np.array_equal(word, rel // (2 * width) * 2 + rel % 2)


def test_one_model_per_block_is_the_private_layout(placement):
    _, m, job, word = placement("k1", 5)
    off = np.arange(5 * m)
    assert np.array_equal(job, off // m) and np.array_equal(word, off % m)


def batch(sizes, seed):
    """Random images with the given thread-segment counts, their oracle streams and the planes they decode to."""
    from lepton_b200 import CoefImage
    rng = np.random.default_rng(seed)
    imgs, streams, want = [], [], []
    for i, nseg in enumerate(sizes):
        cfg = [dict(ncmp=3, mcuh=3 + i % 4, mcuv=max(nseg, 2), sf=((2, 2), (1, 1), (1, 1))),
               dict(ncmp=1, mcuh=4 + i % 5, mcuv=max(nseg, 3), sf=((1, 1),), density=0.5)][i % 2]
        img = random_coef_image(rng, nseg=nseg, **cfg)
        ref = oracle_encode_image(img)
        assert all(rc == 0 for rc, _, _ in ref)
        imgs.append(CoefImage(ncmp=img.ncmp, mcuv=img.mcuv, bch=img.bch, bcv=img.bcv, qtables_zigzag=img.qtables_zigzag,
                              planes=[np.full_like(p, -9) for p in img.planes], luma_y_start=img.luma_y_start))
        streams.append([s for _, s, _ in ref])
        want.append((img.planes, [n for _, _, n in ref]))
    return imgs, streams, want


def check(kernel, sizes, seed, grid_cap):
    imgs, streams, want = batch(sizes, seed)
    st, nd = emu.decode_images(kernel, imgs, streams, grid_cap=grid_cap)
    assert all(s == 0 for s in st), st
    assert nd == [n for _, ns in want for n in ns]
    for img, (planes, _) in zip(imgs, want):
        for c in range(img.ncmp):
            assert np.array_equal(img.planes[c], planes[c])


@pytest.mark.parametrize("lanes", [4, 8])
def test_segment_count_not_a_multiple_of_the_block(lanes):
    """13 segments: one whole block of 8 models and a partial one of 5, in a pool of exactly 13 models."""
    check(emu.KERNEL_G2(lanes), [3, 1, 5, 4], seed=5, grid_cap=0)


@pytest.mark.parametrize("lanes", [4, 8])
def test_groups_take_second_jobs_at_any_place_in_a_block(lanes):
    """One CTA (32 groups at G = 4, 16 at G = 8) for 45 segments of different lengths: groups that finish early claim
    again, alone or a few at a time, so later jobs start anywhere in a block and share it with jobs of other warps."""
    check(emu.KERNEL_G2(lanes), [8, 2, 7, 1, 6, 3, 5, 4, 9], seed=11, grid_cap=1)
