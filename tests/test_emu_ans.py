"""The rANS form of both decode kernels (container version 3), compiled as host C++ and run with real 32-lane warps by the
CPU warp emulator (tests/emu), against the oracle: the reference's -ans fixtures (tests/golden/ans), random geometries coded
by the oracle's rANS writer, damaged streams, and batches that mix bool- and rANS-coded images.  The streams come from the
version-3 files' mux packets and the geometry from their version-1 twins, so nothing here needs a brotli decoder."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu  # noqa: E402
import emu_ans  # noqa: E402
import oracle  # noqa: E402
import oracle_ans  # noqa: E402
from ans_helpers import ans_cases, load_ans_case  # noqa: E402
from helpers import coef_image_from_lep, geometry_of, random_coef_image, segments_of  # noqa: E402

ANS, BOOL = emu_ans.CODER_ANS, emu_ans.CODER_BOOL
KERNELS = [emu.KERNEL_WARP] + [emu.KERNEL_G2(g) for g in (1, 2, 4, 8, 16, 32)]
SMALL = [n for n in ans_cases() if n.startswith("geo_") or n in ("colorswap", "all22_tall_t8", "cut_iphonecrop2_9001")]


def oracle_decisions(lf, streams):
    g, _, _ = geometry_of(lf)
    planes = [np.zeros((lf.frame.bch[c] * lf.frame.bcv[c], 64), np.int16) for c in range(lf.frame.ncmp)]
    out = []
    for i, (y0, y1, last) in enumerate(segments_of(lf)):
        out.append(oracle_ans.decode_segment(g, planes, y0, y1, last, streams[i]))
    return [rc for rc, _ in out], [nd for _, nd in out], planes


@pytest.mark.parametrize("kernel", [emu.KERNEL_WARP, emu.KERNEL_G2(4)])
def test_every_fixture_decodes_to_the_reference_planes(kernel):
    """All fixtures in one batch, decision counts included."""
    imgs, streams, want = [], [], []
    for name in ans_cases():
        lf, planes, _, st, _ = load_ans_case(name)
        imgs.append(coef_image_from_lep(lf, [np.full_like(p, 77) for p in planes]))
        streams.append(st)
        want.append((planes, oracle_decisions(lf, st)[1]))
    status, nd = emu_ans.decode_images(kernel, imgs, streams, [ANS] * len(imgs))
    assert status == [0] * len(status)
    k = 0
    for name, img, (planes, decisions) in zip(ans_cases(), imgs, want):
        assert nd[k:k + img.nseg] == decisions, name
        k += img.nseg
        for c in range(img.ncmp):
            # blocks a truncated image does not code are zero in the device arena
            assert np.array_equal(img.planes[c], planes[c]), (name, c)


@pytest.mark.parametrize("kernel", KERNELS)
def test_small_fixtures_in_every_kernel_shape(kernel):
    for reverse in (False, True):
        imgs, streams, want = [], [], []
        for name in SMALL:
            lf, planes, _, st, _ = load_ans_case(name)
            imgs.append(coef_image_from_lep(lf, [np.full_like(p, -9) for p in planes]))
            streams.append(st)
            want.append((planes, oracle_decisions(lf, st)[1]))
        status, nd = emu_ans.decode_images(kernel, imgs, streams, [ANS] * len(imgs), grid_cap=2, reverse=reverse)
        assert status == [0] * len(status)
        assert nd == [d for _, ds in want for d in ds]
        for name, img, (planes, _) in zip(SMALL, imgs, want):
            for c in range(img.ncmp):
                assert np.array_equal(img.planes[c], planes[c]), (name, c, reverse)


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("cfg", [
    dict(ncmp=3, mcuh=5, mcuv=4, sf=((2, 2), (1, 1), (1, 1)), nseg=1),
    dict(ncmp=3, mcuh=7, mcuv=6, sf=((2, 2), (1, 1), (1, 1)), nseg=3),
    dict(ncmp=3, mcuh=9, mcuv=5, sf=((1, 1), (1, 1), (1, 1)), nseg=2),
    dict(ncmp=1, mcuh=11, mcuv=7, sf=((1, 1),), nseg=4),
    dict(ncmp=1, mcuh=1, mcuv=1, sf=((1, 1),), nseg=1),        # single block: a handful of decisions
    dict(ncmp=3, mcuh=12, mcuv=8, sf=((2, 2), (1, 1), (1, 1)), nseg=8, density=0.9, amp=100, qscale=0.3),   # dense: counts saturate
    dict(ncmp=3, mcuh=8, mcuv=8, sf=((2, 2), (1, 1), (1, 1)), nseg=1, density=0.0, amp=1),
])
def test_random_planes_oracle_ans_streams_decode_back(kernel, cfg):
    from lepton_b200 import CoefImage
    rng = np.random.default_rng(4321)
    img = random_coef_image(rng, **cfg)
    g = oracle.make_geometry(img.ncmp, list(img.bch), list(img.bcv), img.mcuv, img.qtables_zigzag)
    starts = list(img.luma_y_start)
    ref = []
    for i, y0 in enumerate(starts):
        last = i == len(starts) - 1
        ref.append(oracle_ans.encode_segment(g, img.planes, y0, img.bcv[0] if last else starts[i + 1], last))
    assert all(rc == 0 for rc, _, _ in ref)
    out = CoefImage(ncmp=img.ncmp, mcuv=img.mcuv, bch=img.bch, bcv=img.bcv, qtables_zigzag=img.qtables_zigzag,
                    planes=[np.full_like(p, -5) for p in img.planes], luma_y_start=img.luma_y_start)
    st, nd = emu_ans.decode_images(kernel, [out], [[s for _, s, _ in ref]], [ANS])
    assert st == [0] * img.nseg
    assert nd == [n for _, _, n in ref]
    for c in range(img.ncmp):
        assert np.array_equal(out.planes[c], img.planes[c])


def test_damaged_streams_end_like_the_oracle():
    """Cut and bit-flipped rANS streams: status and decision count of every kernel shape equal the oracle's, and the
    planes agree among the kernels (and with the oracle where every segment ends well)."""
    rng = np.random.default_rng(17)
    lf, planes, _, streams, _ = load_ans_case("iphonecrop2_t4")
    seen_bad = 0
    for trial in range(5):
        bad = []
        for s in streams:
            b = bytearray(s[:max(8, len(s) // (2 + trial))])
            for _ in range(1 + trial):
                b[int(rng.integers(0, len(b)))] ^= int(rng.integers(1, 256))
            bad.append(bytes(b))
        want_rc, want_nd, want = oracle_decisions(lf, bad)
        first = None
        for kernel in [emu.KERNEL_WARP, emu.KERNEL_G2(4), emu.KERNEL_G2(8), emu.KERNEL_G2(32)]:
            img = coef_image_from_lep(lf, [np.full_like(p, 11) for p in planes])
            st, nd = emu_ans.decode_images(kernel, [img], [bad], [ANS])
            assert st == want_rc and nd == want_nd, (trial, kernel, st, want_rc)
            got = [p.copy() for p in img.planes]
            if first is None:
                first = got
            for c in range(len(planes)):
                assert np.array_equal(got[c], first[c])
                if all(s == 0 for s in want_rc):
                    assert np.array_equal(got[c], want[c])
        seen_bad += sum(1 for s in want_rc if s != 0)
    assert seen_bad > 0


@pytest.mark.parametrize("kernel", [emu.KERNEL_WARP, emu.KERNEL_G2(4), emu.KERNEL_G2(8)])
def test_mixed_batch_of_bool_and_rans_images(kernel):
    """Version-1 and version-3 images of the same JPEGs in one batch, interleaved: the segments of each coder go to a launch
    of their own, and every image comes back as when it is decoded alone."""
    names = ["iphonecrop2_t4", "geo_y22_odd", "all22_tall_t8", "colorswap"]
    imgs, streams, coders, want = [], [], [], []
    for name in names:
        lf, planes, bool_streams, st, _ = load_ans_case(name)
        for coder, s in ((ANS, st), (BOOL, bool_streams)):
            imgs.append(coef_image_from_lep(lf, [np.full_like(p, 3) for p in planes]))
            streams.append(s)
            coders.append(coder)
            want.append(planes)
    status, _ = emu_ans.decode_images(kernel, imgs, streams, coders, grid_cap=2)
    assert status == [0] * len(status)
    for img, planes, coder in zip(imgs, want, coders):
        for c in range(img.ncmp):
            assert np.array_equal(img.planes[c], planes[c]), coder
