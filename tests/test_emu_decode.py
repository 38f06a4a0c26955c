"""The decode kernels, compiled as host C++ and run with real 32-lane warps by the CPU warp emulator (tests/emu), against
the oracle.

`lep_decode.cu` (one warp per thread-segment; small batches) and `lep_decode_g2.cu` (G lanes per segment, 32 / G segments
per warp in lock step; large batches) run here exactly as written -- divergence, votes, shuffles, shared memory and the
persistent work queues included -- so their logic is pinned without a GPU; the GPU parity tests run the same sources on
the device.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu  # noqa: E402
import oracle  # noqa: E402
from helpers import (EXTREMES, coef_image_from_lep, extreme_leps, geometry_of, golden_leps, load_extreme_lep, load_lep,
                     oracle_decode_planes, oracle_encode_image, plane_hashes, random_coef_image, segments_of)

KERNELS = [emu.KERNEL_WARP]
GROUPS = [emu.KERNEL_G2(g) for g in (1, 2, 4, 8, 16, 32)]       # lep_decode_g2_kernel<G>; the library ships G = 4, 8, 32
SCHEDULES = [False, True]                                       # reverse: CTAs and threads in reverse order


@pytest.mark.parametrize("kernel", KERNELS + [emu.KERNEL_G2(4)])
def test_golden_files_decode_to_the_reference_planes(kernel):
    for name in golden_leps():
        lf = load_lep(name)
        planes, streams = oracle_decode_planes(lf)
        img = coef_image_from_lep(lf, [np.full_like(p, 77) for p in planes])
        st, _ = emu.decode_images(kernel, [img], [streams[:lf.nseg]])
        assert all(s == 0 for s in st), (name, st)
        for c in range(img.ncmp):
            assert np.array_equal(img.planes[c], planes[c]), "%s component %d" % (name, c)


@pytest.mark.parametrize("kernel", KERNELS + [emu.KERNEL_G2(8)])
def test_one_launch_with_more_segments_than_a_warp(kernel):
    """All golden files in one batch: > 32 segments, so several warps and a partly filled last one.  Under both schedules
    of the emulator (the threads of each CTA in order and in reverse order): this is the golden decode case that runs
    reversed, the test above decodes the same files one launch each."""
    for reverse in SCHEDULES:
        imgs, streams_all, want = [], [], []
        for name in golden_leps():
            lf = load_lep(name)
            planes, streams = oracle_decode_planes(lf)
            imgs.append(coef_image_from_lep(lf, [np.full_like(p, -3) for p in planes]))
            streams_all.append(streams[:lf.nseg])
            want.append(planes)
        assert sum(im.nseg for im in imgs) > 32
        st, _ = emu.decode_images(kernel, imgs, streams_all, grid_cap=3, reverse=reverse)     # warp kernel: 12 persistent warps share the queue
        assert all(s == 0 for s in st), st
        for name, img, planes in zip(golden_leps(), imgs, want):
            for c in range(img.ncmp):
                assert np.array_equal(img.planes[c], planes[c]), "%s component %d reverse %s" % (name, c, reverse)


@pytest.mark.parametrize("kernel", KERNELS + GROUPS)
@pytest.mark.parametrize("cfg", [
    dict(ncmp=3, mcuh=5, mcuv=4, sf=((2, 2), (1, 1), (1, 1)), nseg=1),
    dict(ncmp=3, mcuh=7, mcuv=6, sf=((2, 2), (1, 1), (1, 1)), nseg=3),
    dict(ncmp=3, mcuh=9, mcuv=5, sf=((1, 1), (1, 1), (1, 1)), nseg=2),
    dict(ncmp=3, mcuh=6, mcuv=4, sf=((2, 1), (1, 1), (1, 1)), nseg=2),
    dict(ncmp=1, mcuh=11, mcuv=7, sf=((1, 1),), nseg=4),
    dict(ncmp=1, mcuh=1, mcuv=1, sf=((1, 1),), nseg=1),        # single block
    dict(ncmp=1, mcuh=1, mcuv=9, sf=((1, 1),), nseg=2),        # one block wide
    dict(ncmp=3, mcuh=1, mcuv=3, sf=((2, 2), (1, 1), (1, 1)), nseg=1),
    dict(ncmp=3, mcuh=12, mcuv=8, sf=((2, 2), (1, 1), (1, 1)), nseg=8, density=0.9, amp=100, qscale=0.3),   # dense, large coefficients (threshold bits)
    dict(ncmp=3, mcuh=8, mcuv=8, sf=((2, 2), (1, 1), (1, 1)), nseg=1, density=0.0, amp=1),     # (almost) empty blocks
])
def test_random_planes_oracle_streams_decode_back(kernel, cfg):
    from lepton_b200 import CoefImage
    rng = np.random.default_rng(1234)
    img = random_coef_image(rng, **cfg)
    ref = oracle_encode_image(img)
    assert all(rc == 0 for rc, _, _ in ref)
    out = CoefImage(ncmp=img.ncmp, mcuv=img.mcuv, bch=img.bch, bcv=img.bcv, qtables_zigzag=img.qtables_zigzag,
                    planes=[np.full_like(p, -5) for p in img.planes], luma_y_start=img.luma_y_start)
    st, nd = emu.decode_images(kernel, [out], [[s for _, s, _ in ref]])
    assert all(s == 0 for s in st), st
    assert nd == [n for _, _, n in ref]                       # one get per put
    for c in range(img.ncmp):
        assert np.array_equal(out.planes[c], img.planes[c])


def test_damaged_streams_end_the_same_way_in_all_kernels_and_the_oracle():
    """Truncated / bit-flipped streams: whatever comes out (status 7 for an impossible non-zero count, or garbage
    coefficients), the two kernels under both schedules and the oracle must agree on status, decision count and every
    stored block."""
    rng = np.random.default_rng(99)
    lf = load_lep("androidcrop_t2.lep")
    planes, streams = oracle_decode_planes(lf)
    g, _, _ = geometry_of(lf)
    segs = segments_of(lf)
    seen_bad = 0
    for trial in range(6):
        bad = []
        for s in streams[:lf.nseg]:
            b = bytearray(s[:max(8, len(s) // (2 + trial))])
            for _ in range(1 + trial):
                b[int(rng.integers(4, len(b)))] ^= int(rng.integers(1, 256))
            bad.append(bytes(b))
        want = [np.zeros_like(p) for p in planes]
        want_rc = []
        for i, (y0, y1, last) in enumerate(segs):
            rc, _ = oracle.decode_segment(g, want, y0, y1, last, bad[i])
            want_rc.append(rc)
        got = {}
        for kernel in KERNELS + [emu.KERNEL_G2(4), emu.KERNEL_G2(8), emu.KERNEL_G2(32)]:
            for reverse in SCHEDULES:
                img = coef_image_from_lep(lf, [np.full_like(p, 11) for p in planes])
                st, nd = emu.decode_images(kernel, [img], [bad], reverse=reverse)
                got[kernel, reverse] = (st, nd, [p.copy() for p in img.planes])
        a = got[emu.KERNEL_WARP, False]
        for b in (v for k, v in got.items() if k != (emu.KERNEL_WARP, False)):
            assert a[0] == b[0] == want_rc and a[1] == b[1]
            for c in range(len(planes)):
                assert np.array_equal(a[2][c], b[2][c])
        seen_bad += sum(1 for s in a[0] if s != 0)
        if all(s == 0 for s in want_rc):
            for c in range(len(planes)):
                assert np.array_equal(a[2][c], want[c])
    assert seen_bad > 0       # the damage was enough to hit the inconsistent-stream exit at least once


@pytest.mark.parametrize("kernel", KERNELS + GROUPS)
def test_extreme_corpus_decodes_to_the_reference_planes(kernel):
    """Every reference-written .lep of the extreme corpus (1, 4 and 8 thread-segments) in one launch: the planes of the
    reference's -ujg dump, from the streams the reference wrote.  The group kernels skip the 4-segment records (the
    8-segment ones cover the handoffs) to keep the emulated run short."""
    imgs, streams_all, names = [], [], []
    for name, source in extreme_leps():
        if kernel != emu.KERNEL_WARP and "_t4." in name:
            continue
        lf = load_extreme_lep(name)
        planes, streams = oracle_decode_planes(lf)
        imgs.append(coef_image_from_lep(lf, [np.full_like(p, 77) for p in planes]))
        streams_all.append(streams[:lf.nseg])
        names.append((name, source))
    st, _ = emu.decode_images(kernel, imgs, streams_all, grid_cap=3)
    assert all(s == 0 for s in st), st
    for (name, source), img in zip(names, imgs):
        assert plane_hashes(img.planes) == EXTREMES[source]["plane_sha256"], name


@pytest.mark.parametrize("kernel", KERNELS + GROUPS)
@pytest.mark.parametrize("cfg", [
    dict(ncmp=3, mcuh=6, mcuv=4, sf=((2, 2), (1, 1), (1, 1)), nseg=3, q16=True, max_cat=11),
    dict(ncmp=3, mcuh=5, mcuv=5, sf=((2, 1), (1, 1), (1, 1)), nseg=2, q16=True, max_cat=11, density=0.9),
    dict(ncmp=1, mcuh=8, mcuv=8, sf=((1, 1),), nseg=4, q16=True, max_cat=11, density=0.9),
])
def test_random_extreme_planes_decode_back(kernel, cfg):
    """16-bit quantisers and magnitudes uniform over the categories 0..11 (the oracle codes every segment of these)."""
    from lepton_b200 import CoefImage
    rng = np.random.default_rng(1234)
    img = random_coef_image(rng, **cfg)
    ref = oracle_encode_image(img)
    assert all(rc == 0 for rc, _, _ in ref)
    out = CoefImage(ncmp=img.ncmp, mcuv=img.mcuv, bch=img.bch, bcv=img.bcv, qtables_zigzag=img.qtables_zigzag,
                    planes=[np.full_like(p, -5) for p in img.planes], luma_y_start=img.luma_y_start)
    st, nd = emu.decode_images(kernel, [out], [[s for _, s, _ in ref]])
    assert all(s == 0 for s in st), st
    assert nd == [n for _, _, n in ref]
    for c in range(img.ncmp):
        assert np.array_equal(out.planes[c], img.planes[c])
