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
from ans_helpers import (advanced, ans_cases, judge, load_ans_case, oracle_ans_streams, oracle_decode_image,  # noqa: E402
                         traces)
from helpers import coef_image_from_lep, geometry_of, oracle_encode_image, random_coef_image, segments_of  # noqa: E402

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


# ---------------------------------------------------------------------------------------------------- edges of the coder
# Builders of one batch each -> (imgs, streams, coders), and what its oracle traces must show, so that a batch cannot
# silently stop reaching the edge it is named for.  tests/test_gpu_ans_edges.py decodes the same batches on the device.
# The emulator's stream arena holds 0xA5 behind every stream, so a partial last word is masked against that pattern here.
L31 = 1 << 31


def stream_length_batch(seed=5):
    """One-segment images whose streams end anywhere: a small image's oracle stream cut at every length (0 to all of it),
    all-zero, all-0xFF and random streams of every length 0..40 (shorter than the 16 state bytes, a partial last word,
    a last word whose refill leaves the group kernel's preload at the end of the stream), the stream with 1..7 junk bytes
    behind it, and a larger image's stream cut near its end and at a few hundred bytes."""
    rng = np.random.default_rng(seed)
    small = random_coef_image(rng, ncmp=1, mcuh=2, mcuv=1, sf=((1, 1),), nseg=1, density=0.4)
    big = random_coef_image(rng, ncmp=3, mcuh=6, mcuv=2, sf=((2, 2), (1, 1), (1, 1)), nseg=1, density=0.4)
    (s_small,), (s_big,) = oracle_ans_streams([small, big])
    assert len(s_big) > 320
    imgs, streams = [], []
    for n in range(len(s_small) + 1):
        imgs.append(small), streams.append([s_small[:n]])
    for n in range(41):
        for s in (bytes(n), b"\xff" * n, rng.bytes(n)):
            imgs.append(small), streams.append([s])
    for n in range(1, 8):
        imgs.append(small), streams.append([s_small + rng.bytes(n)])
    for n in list(range(len(s_big) - 8, len(s_big) + 1)) + [255, 256, 257, 258, 299, 300, 301, 302, 303]:
        imgs.append(big), streams.append([s_big[:n]])
    return imgs, streams, [ANS] * len(imgs)


def assert_stream_tails(imgs, streams):
    t = traces(imgs, streams)
    took = t[t["word_off"] >= 0]
    left = took["len"] - took["word_off"]
    for r in (1, 2, 3):
        assert np.any(left == r), r                       # the refill takes a partial last word
    assert np.any(left == 4)                              # the last whole word: the group kernel preloads at the end
    assert np.any(left <= 0)                              # refills past the end read zero
    assert any(0 < len(s[0]) < 16 for s in streams)


def steer(img, stream, k, target):
    """`stream` with the state words of decision k % 2 changed so that decision k advances its state to `target`, every
    decision up to k taking the bit (and so the probability) it took before.  The states of the decisions k - 2, k - 4, ..
    of that state's chain are solved backwards; none of them takes a word."""
    t = oracle_decode_image(img, [stream], trace=True)[3][0]
    x = target
    for j in range(k, -1, -2):
        assert j == k or x >= L31
        p, b = int(t["prob"][j]), int(t["bit"][j])
        start, freq = (p, 256 - p) if b else (0, p)
        x = (x // freq) << 8 | (x % freq + start)
    assert x < 1 << 64
    s = bytearray(stream)
    s[8 * (k % 2):8 * (k % 2) + 8] = x.to_bytes(8, "little")
    return bytes(s)


RENORM_TARGETS = (L31 - 1, L31, L31 + 1)


def renorm_boundary_batch(seed=6):
    """Streams whose decisions 0..3 advance their state to exactly 2^31 - 1 (a word is taken), 2^31 and 2^31 + 1 (none
    is), state words 0 and 2^64 - 1, and the oracle stream cut so that its last refill takes a partial word."""
    rng = np.random.default_rng(seed)
    imgs = [random_coef_image(rng, ncmp=1, mcuh=3, mcuv=2, sf=((1, 1),), nseg=1, density=0.4),
            random_coef_image(rng, ncmp=3, mcuh=2, mcuv=2, sf=((2, 2), (1, 1), (1, 1)), nseg=1, density=0.5)]
    base = [s[0] for s in oracle_ans_streams(imgs)]
    out_imgs, streams = [], []
    for img, s in zip(imgs, base):
        for k in range(4):
            for target in RENORM_TARGETS:
                out_imgs.append(img), streams.append([steer(img, s, k, target)])
        for x0, x1 in ((0, (1 << 64) - 1), ((1 << 64) - 1, 0), (0, 0), ((1 << 64) - 1, (1 << 64) - 1)):
            out_imgs.append(img), streams.append([x0.to_bytes(8, "little") + x1.to_bytes(8, "little") + s[16:]])
        for cut in (1, 2, 3, 5, 6, 7):
            out_imgs.append(img), streams.append([s[:len(s) - cut]])
    return out_imgs, streams, [ANS] * len(out_imgs)


def assert_renorm_edges(imgs, streams):
    t = traces(imgs, streams)
    adv = advanced(t)
    assert np.all((adv < L31) == (t["word_off"] >= 0))    # the oracle refills exactly below 2^31
    for target in RENORM_TARGETS:
        assert np.count_nonzero(adv == target) >= 8, target
    assert np.any(t["x_before"] == 0) and np.any(t["x_before"] == np.uint64((1 << 64) - 1))
    took = t[t["word_off"] >= 0]
    assert np.any((took["len"] - took["word_off"] > 0) & (took["len"] - took["word_off"] < 4))


SATURATED = [dict(ncmp=3, mcuh=12, mcuv=8, sf=((2, 2), (1, 1), (1, 1)), nseg=8, density=0.9, amp=100, qscale=0.3),
             dict(ncmp=3, mcuh=8, mcuv=8, sf=((2, 2), (1, 1), (1, 1)), nseg=1, density=0.0, amp=1),
             dict(ncmp=3, mcuh=24, mcuv=16, sf=((2, 2), (1, 1), (1, 1)), nseg=2, density=0.0, amp=1)]


def saturated_batch(seed=4321):
    """Dense and empty images whose branch counts saturate: decisions at probability 1 and 255, and counts restarting
    at 129 from 255 on either side."""
    rng = np.random.default_rng(seed)
    imgs = [random_coef_image(rng, **cfg) for cfg in SATURATED]
    return imgs, oracle_ans_streams(imgs), [ANS] * len(imgs)


def assert_saturation(imgs, streams):
    t = traces(imgs, streams)
    assert np.any(t["prob"] == 1) and np.any(t["prob"] == 255)
    assert np.count_nonzero((t["bit"] == 0) & (t["c0"] == 255)) > 10          # c0 restarts at 129
    assert np.count_nonzero((t["bit"] == 1) & (t["c1"] == 255)) > 10          # c1 restarts at 129
    assert np.any((t["c0"] == 129) & (t["c1"] < 129)) and np.any((t["c1"] == 129) & (t["c0"] < 129))


def split_batch(n_bool, n_ans, seed=8):
    """Images of 1..16 one-row segments, n_bool bool-coded and n_ans rANS-coded segments in all, the two coders' images
    interleaved in batch order."""
    rng = np.random.default_rng(seed + 7 * n_bool + n_ans)
    parts = {}
    for coder, n in ((BOOL, n_bool), (ANS, n_ans)):
        imgs, left = [], n
        while left:
            nseg = min(left, int(rng.integers(1, 17)))
            imgs.append(random_coef_image(rng, ncmp=1, mcuh=int(rng.integers(1, 4)), mcuv=nseg, sf=((1, 1),), nseg=nseg, density=0.4))
            left -= nseg
        streams = oracle_ans_streams(imgs) if coder == ANS else [[s for _, s, _ in oracle_encode_image(i)] for i in imgs]
        parts[coder] = list(zip(imgs, streams))
    imgs, streams, coders = [], [], []
    for k in range(max(len(parts[BOOL]), len(parts[ANS]))):
        for coder in (ANS, BOOL) if k % 2 else (BOOL, ANS):
            if k < len(parts[coder]):
                imgs.append(parts[coder][k][0]), streams.append(parts[coder][k][1]), coders.append(coder)
    return imgs, streams, coders


def emu_run(kernel, kernel_ans=None, grid_cap=0):
    """judge's run on the emulator: the bool part on `kernel`, the rANS part on kernel_ans (default the same)"""
    return lambda out, streams, coders: emu_ans.decode_images(kernel, out, streams, coders if coders is not None else [BOOL] * len(out),
                                                              grid_cap=grid_cap, kernel_ans=kernel_ans)


EDGE_KERNELS = [emu.KERNEL_WARP, emu.KERNEL_G2(4), emu.KERNEL_G2(8), emu.KERNEL_G2(32)]


@pytest.mark.parametrize("kernel", EDGE_KERNELS)
def test_streams_of_every_length_and_content(kernel):
    imgs, streams, coders = stream_length_batch()
    assert_stream_tails(imgs, streams)
    judge(emu_run(kernel, grid_cap=2), imgs, streams, coders)


@pytest.mark.parametrize("kernel", EDGE_KERNELS)
def test_renormalisation_boundary(kernel):
    imgs, streams, coders = renorm_boundary_batch()
    assert_renorm_edges(imgs, streams)
    judge(emu_run(kernel, grid_cap=2), imgs, streams, coders)


@pytest.mark.slow
@pytest.mark.parametrize("kernel", EDGE_KERNELS)
def test_saturated_models(kernel):
    imgs, streams, coders = saturated_batch()
    assert_saturation(imgs, streams)
    judge(emu_run(kernel), imgs, streams, coders)


@pytest.mark.parametrize("kernels", [(emu.KERNEL_WARP, emu.KERNEL_G2(4)), (emu.KERNEL_G2(4), emu.KERNEL_WARP),
                                     (emu.KERNEL_G2(8), emu.KERNEL_G2(32))], ids=["warp+group4", "group4+warp", "group8+group32"])
@pytest.mark.parametrize("sizes", [(40, 9), (9, 40), (20, 1), (17, 0)], ids=lambda s: "%d+%d" % s)
def test_coder_parts_on_different_kernels(kernels, sizes):
    """Mixed batches whose bool part and rANS part take different kernels; a rANS part of one segment; a coder array of
    bool alone."""
    imgs, streams, coders = split_batch(*sizes)
    judge(emu_run(kernels[0], kernels[1], grid_cap=1), imgs, streams, coders)
