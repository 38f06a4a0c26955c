"""The encode kernels -- count pre-pass, token offsets, kernel A (symbolise + adaptive model), kernel B (range coder) --
compiled as host C++ and run with real 32-lane warps by the CPU warp emulator (tests/emu), against the reference's streams and the
oracle.  Same cases as the GPU parity tests of the encoder; the GPU tests run the same sources on the device."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu  # noqa: E402
from helpers import (EXTREMES, coef_image_from_lep, extreme_jpegs, extreme_leps, golden_leps, load_extreme_lep, load_lep,
                     oracle_decode_planes, oracle_encode_image, random_coef_image, read_golden)


# range coder: 0 = range-only pass + parallel pieces + carry pass (the default), 1 = one serial chain per segment,
# 2 = as 0 with the range pass's tokens fed through registers instead of the cp.async ring (LEPB200_RC_FEED=0)
KERNELS = [0, 1, 2]


@pytest.mark.parametrize("kernel", KERNELS)
def test_golden_batch_encode_matches_reference_streams(kernel):
    """All committed reference-written .lep files in ONE batch, three persistent CTAs sharing the work queue: emulated GPU
    streams == the reference's streams.  With the parallel range coder (kernel 0) also with the CTAs and threads of every
    launch in reverse order: kernel A and its shared queue are the same for every range coder, whose forms
    test_emu_rangecoder.py runs reversed on their own."""
    imgs, want = [], []
    for name in golden_leps():
        lf = load_lep(name)
        planes, streams = oracle_decode_planes(lf)
        imgs.append(coef_image_from_lep(lf, planes))
        want.append(streams[:lf.nseg])
    for reverse in (False, True) if kernel == 0 else (False,):
        got = emu.encode_images(imgs, grid_cap=3, kernel=kernel, reverse=reverse)
        for name, g, w in zip(golden_leps(), got, want):
            assert [x[0] for x in g] == [0] * len(w), (name, reverse)
            assert [x[1] for x in g] == list(w), (name, reverse)


@pytest.mark.parametrize("cfg", [
    dict(ncmp=3, mcuh=5, mcuv=4, sf=((2, 2), (1, 1), (1, 1)), nseg=1),
    dict(ncmp=3, mcuh=7, mcuv=6, sf=((2, 2), (1, 1), (1, 1)), nseg=3),
    dict(ncmp=3, mcuh=9, mcuv=5, sf=((1, 1), (1, 1), (1, 1)), nseg=2),
    dict(ncmp=3, mcuh=6, mcuv=4, sf=((2, 1), (1, 1), (1, 1)), nseg=2),
    dict(ncmp=1, mcuh=11, mcuv=7, sf=((1, 1),), nseg=4),
    dict(ncmp=1, mcuh=1, mcuv=1, sf=((1, 1),), nseg=1),        # single block
    dict(ncmp=1, mcuh=1, mcuv=9, sf=((1, 1),), nseg=2),        # one block wide
    dict(ncmp=3, mcuh=1, mcuv=3, sf=((2, 2), (1, 1), (1, 1)), nseg=1),
    dict(ncmp=3, mcuh=12, mcuv=8, sf=((2, 2), (1, 1), (1, 1)), nseg=8, density=0.9, amp=100, qscale=0.3),   # dense, large coefficients
    dict(ncmp=3, mcuh=8, mcuv=8, sf=((2, 2), (1, 1), (1, 1)), nseg=1, density=0.0, amp=1),     # (almost) empty blocks
])
@pytest.mark.parametrize("kernel", KERNELS)
def test_random_planes_encode_vs_oracle_and_decode_back(kernel, cfg):
    from lepton_b200 import CoefImage
    rng = np.random.default_rng(1234)
    img = random_coef_image(rng, **cfg)
    ref = oracle_encode_image(img)
    got = emu.encode_images([img], kernel=kernel)[0]
    assert [(g[0], g[1], g[2]) for g in got] == [(rc, s, nd) for rc, s, nd in ref]
    out = CoefImage(ncmp=img.ncmp, mcuv=img.mcuv, bch=img.bch, bcv=img.bcv, qtables_zigzag=img.qtables_zigzag,
                    planes=[np.full_like(p, -5) for p in img.planes], luma_y_start=img.luma_y_start)
    st, _ = emu.decode_images(emu.KERNEL_WARP, [out], [[g[1] for g in got]])
    assert all(s == 0 for s in st)
    for c in range(img.ncmp):
        assert np.array_equal(out.planes[c], img.planes[c])


@pytest.mark.parametrize("kernel", KERNELS)
def test_out_of_range_coefficient_status(kernel):
    """COEFFICIENT_OUT_OF_RANGE (reference exit code 6, src/vp8/encoder/encoder.cc:124,265,343)."""
    rng = np.random.default_rng(5)
    img = random_coef_image(rng, ncmp=1, mcuh=4, mcuv=4, sf=((1, 1),), nseg=2)
    img.planes[0][3, 7] = 4096          # 13-bit magnitude in the first segment only
    ref = oracle_encode_image(img)
    got = emu.encode_images([img], kernel=kernel)[0]
    assert [g[0] for g in got] == [r[0] for r in ref] == [6, 0]
    assert got[1][1] == ref[1][1]


@pytest.mark.parametrize("kernel", KERNELS)
def test_branch_saturation_long_run(kernel):
    """Long constant runs drive branch counts through the 255 overflow / 'neverseen' paths (branch.hh:82-100): the
    closed-form conflict resolution of kernel A has to fall back to its rank loop there."""
    from lepton_b200 import CoefImage
    n = 40 * 40
    p = np.zeros((n, 64), dtype=np.int16)
    p[:, 0] = 1
    p[::7, 1] = -3
    p[:, 49] = 5
    img = CoefImage(ncmp=1, mcuv=40, bch=[40], bcv=[40], qtables_zigzag=[[8] * 64], planes=[p], luma_y_start=[0])
    (rc, s, nd), = oracle_encode_image(img)
    got = emu.encode_images([img], kernel=kernel)[0][0]
    assert rc == 0 and got == (0, s, nd)


@pytest.mark.parametrize("kernel", KERNELS)
def test_mixed_batch_many_images(kernel):
    """A batch of different geometries in one launch: per-image results must not depend on batching."""
    rng = np.random.default_rng(99)
    imgs = []
    for k in range(24):
        ncmp = 1 if k % 5 == 0 else 3
        sf = ((1, 1),) if ncmp == 1 else (((2, 2), (1, 1), (1, 1)) if k % 2 else ((1, 1), (1, 1), (1, 1)))
        imgs.append(random_coef_image(rng, ncmp=ncmp, mcuh=2 + k % 7, mcuv=2 + (k * 3) % 5, sf=sf, nseg=1 + k % 3))
    got = emu.encode_images(imgs, grid_cap=2, kernel=kernel)
    for img, g in zip(imgs, got):
        ref = oracle_encode_image(img)
        assert [x[1] for x in g] == [r[1] for r in ref]


def test_zero_quantiser_status_both_directions():
    """UNSUPPORTED_JPEG_WITH_ZERO_IDCT_0 (reference exit code 43): set_quantization_table refuses a table whose first row /
    column entries make an IDCT base of zero (src/vp8/model/model.hh:257-262).  Every segment of such an image reports 43 in
    the oracle, in kernel A and in both decode kernels; nothing is coded."""
    from lepton_b200 import CoefImage
    rng = np.random.default_rng(3)
    img = random_coef_image(rng, ncmp=3, mcuh=4, mcuv=4, sf=((2, 2), (1, 1), (1, 1)), nseg=2)
    q = [list(t) for t in img.qtables_zigzag]
    q[1][0] = 0                                  # chroma DC quantiser 0
    bad = CoefImage(ncmp=img.ncmp, mcuv=img.mcuv, bch=img.bch, bcv=img.bcv, qtables_zigzag=q, planes=img.planes, luma_y_start=img.luma_y_start)
    ref = oracle_encode_image(bad)
    assert [r[0] for r in ref] == [43, 43]
    for kernel in KERNELS:
        got = emu.encode_images([bad], kernel=kernel)[0]
        assert [g[0] for g in got] == [43, 43] and all(g[1] == b"" for g in got), kernel
    good = oracle_encode_image(img)
    for dk in (emu.KERNEL_WARP, emu.KERNEL_G2(4)):
        out = CoefImage(ncmp=bad.ncmp, mcuv=bad.mcuv, bch=bad.bch, bcv=bad.bcv, qtables_zigzag=q,
                        planes=[np.zeros_like(p) for p in bad.planes], luma_y_start=bad.luma_y_start)
        st, _ = emu.decode_images(dk, [out], [[s for _, s, _ in good]])
        assert list(st) == [43, 43], (dk, st)


def extreme_batch():
    """Every image of the extreme corpus as the encoder gets it: the reference's .lep records (their geometry and splits,
    planes from the oracle's decode) and the refused JPEGs (front end's planes).  -> images, per image a list of expected
    (status, stream or None) per segment."""
    from lepton_b200 import HostJpeg
    imgs, want = [], []
    for name, _ in extreme_leps():
        lf = load_extreme_lep(name)
        planes, streams = oracle_decode_planes(lf)
        imgs.append(coef_image_from_lep(lf, planes))
        want.append([(0, s) for s in streams[:lf.nseg]])
    for n in extreme_jpegs():
        if EXTREMES[n]["status_want"]:
            img = HostJpeg(read_golden(EXTREMES[n]["path"])).coef_image()
            imgs.append(img)
            want.append([(rc, s if rc == 0 else None) for rc, s, _ in oracle_encode_image(img)])
            assert EXTREMES[n]["status_want"] in [w[0] for w in want[-1]], n
    return imgs, want


@pytest.mark.parametrize("kernel", KERNELS)
def test_extreme_corpus_batch_encode_matches_reference_streams(kernel):
    """The extreme corpus in ONE batch (16-bit quantisers, category-11 magnitudes at every position, DC wrap, 4- and
    8-segment records, two files the reference refuses): the reference's streams, and status 6 where it refused."""
    imgs, want = extreme_batch()
    got = emu.encode_images(imgs, grid_cap=3, kernel=kernel)
    for k, (g, w) in enumerate(zip(got, want)):
        assert [x[0] for x in g] == [s for s, _ in w], k
        for (st, data, _), (_, ws) in zip(g, w):
            if st == 0:
                assert data == ws, k


# coefficient regimes photos never reach: 16-bit quantisers, magnitudes uniform over the categories 0..11, DC over +-2047
EXTREME_CFGS = [
    dict(ncmp=3, mcuh=6, mcuv=4, sf=((2, 2), (1, 1), (1, 1)), nseg=3, q16=True, max_cat=11),
    dict(ncmp=1, mcuh=8, mcuv=8, sf=((1, 1),), nseg=4, q16=True, max_cat=11, density=0.9),
    dict(ncmp=3, mcuh=6, mcuv=4, sf=((2, 1), (1, 1), (1, 1)), nseg=3, max_cat=11),
    dict(ncmp=1, mcuh=8, mcuv=8, sf=((1, 1),), nseg=8, max_cat=11, density=0.9),
    dict(ncmp=3, mcuh=5, mcuv=4, sf=((1, 1), (1, 1), (1, 1)), nseg=2, q16=True, max_cat=11, dc_max=2047),
    dict(ncmp=1, mcuh=6, mcuv=8, sf=((1, 1),), nseg=8, dc_max=2047),
]


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("cfg", EXTREME_CFGS)
def test_random_extreme_planes_encode_vs_oracle(kernel, cfg):
    """Status segment by segment as the oracle (6 where a coefficient or a DC residual cannot be coded), and the oracle's
    stream and decision count for every segment it codes."""
    rng = np.random.default_rng(4321)
    img = random_coef_image(rng, **cfg)
    ref = oracle_encode_image(img)
    got = emu.encode_images([img], kernel=kernel)[0]
    assert [g[0] for g in got] == [r[0] for r in ref]
    for g, r in zip(got, ref):
        if r[0] == 0:
            assert (g[1], g[2]) == (r[1], r[2])
