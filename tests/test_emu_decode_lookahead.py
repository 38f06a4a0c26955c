"""Branch words read ahead of their write-backs in lep_decode_g2_kernel<G>, on the CPU warp emulator, against the oracle,
at every G.

The coefficient loops of the group kernel load the word of decision k+1 before decision k writes its own word back, and
forward the written value when both use the same branch.  The count trees are read as whole rows before their first
bit, the 7x7 tree of the next block of a row at the end of the block before it.  Each input below is built so that one
of those hazards provably occurs, and is decoded from the oracle's streams back to the oracle's planes with the oracle's
decision counts.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu  # noqa: E402
from helpers import oracle_decode_image, oracle_encode_image, random_coef_image  # noqa: E402

GROUPS = [emu.KERNEL_G2(g) for g in (1, 2, 4, 8, 16, 32)]
EDGE = list(range(50, 64))          # aligned indices of the 14 edge coefficients (raster 1..7, then 8, 16, .., 56)
Q = 20                              # every quantiser: (freqmax + Q - 1) // Q <= (1024 + 19) // 20 = 52 < 128, so the
                                    # min_threshold of every position (bit length - 7, lep_plan.cuh fill_quant) is 0


def with_quant(img, q):
    img.qtables_zigzag = [[q] * 64 for _ in range(img.ncmp)]
    return img


def decode_vs_oracle(kernel, imgs, grid_cap=0, reverse=False):
    from lepton_b200 import CoefImage
    refs = [oracle_encode_image(img) for img in imgs]
    for r in refs:
        assert all(rc == 0 for rc, _, _ in r), [rc for rc, _, _ in r]
    out = [CoefImage(ncmp=i.ncmp, mcuv=i.mcuv, bch=i.bch, bcv=i.bcv, qtables_zigzag=i.qtables_zigzag,
                     planes=[np.full_like(p, -5) for p in i.planes], luma_y_start=i.luma_y_start, trunc_bcv=i.trunc_bcv,
                     trunc_bc=i.trunc_bc) for i in imgs]
    st, nd = emu.decode_images(kernel, out, [[s for _, s, _ in r] for r in refs], grid_cap=grid_cap, reverse=reverse)
    assert all(s == 0 for s in st), st
    assert nd == [n for r in refs for _, _, n in r]             # one get per put
    for k, (img, o, r) in enumerate(zip(imgs, out, refs)):
        want = oracle_decode_image(img, [s for _, s, _ in r])
        for c in range(img.ncmp):
            assert np.array_equal(o.planes[c], want[c]), (k, c)
    return nd


def both_schedules(kernel, imgs, grid_cap=0):
    """decode_vs_oracle with the threads of each CTA in order and in reverse order -> decision counts"""
    nd = decode_vs_oracle(kernel, imgs, grid_cap)
    assert decode_vs_oracle(kernel, imgs, grid_cap, reverse=True) == nd
    return nd


# The hazard batches: (images, CTA cap of the emulated launch).  test_gpu_kernel_edges.py decodes the same batches on the
# device.
def saturated_threshold_batch():
    """(a) Decisions k, k+1 and k+2 on the same branch word.  Every edge coefficient is +-2047: bit length 11, and with a
    min_threshold of 0 the sign state goes to the threshold state for bits 9..0, ten threshold decisions.  Their index
    starts at 1 and takes (index << 1) | bit capped at 127; all bits of 2047 are ones, so the index is 127 from the
    seventh decision on and decisions 7, 8, 9 and 10 of every edge coefficient use the same branch."""
    rng = np.random.default_rng(71)
    img = with_quant(random_coef_image(rng, ncmp=3, mcuh=3, mcuv=2, sf=((2, 2), (1, 1), (1, 1)), nseg=2), Q)
    for p in img.planes:
        p[:, EDGE] = np.where(rng.random((p.shape[0], len(EDGE))) < 0.5, 2047, -2047)
    return [img], 0


def word_in_flight_batch():
    """(b) Both candidate addresses of the next decision equal the word being written back.  In this grammar the
    threshold index grows strictly until it saturates and every other address moves with the position, the bit index or
    the tree level, so the saturated index is where it happens.  Edge magnitudes 1024..2047 (bit length 11, ten
    threshold bits at min_threshold 0) with random low bits: once the index is 127, the next decision uses the word in
    flight whatever the bit, and the run ends on bits of either value."""
    rng = np.random.default_rng(72)
    img = with_quant(random_coef_image(rng, ncmp=3, mcuh=3, mcuv=2, sf=((2, 1), (1, 1), (1, 1)), nseg=1), Q)
    for p in img.planes:
        n = p.shape[0]
        mag = rng.integers(1024, 2048, size=(n, len(EDGE)))
        p[:, EDGE] = np.where(rng.random((n, len(EDGE))) < 0.5, mag, -mag)
    return [img], 0


def special_state_batch():
    """(c) Branch words driven through count saturation into the special (1,255) state.  All 7x7 coefficients of the
    grey image are positive, and the sign of every 7x7 coefficient of a component is one branch (m_sign(ci, 0, 0)): it
    sees only ones, so its one-count reaches 255 with the zero-count still 1 and stays in the special state, p = 0, for
    the rest of the segment.  The edge coefficients are +2047 (the four saturated threshold decisions of (a) each, all
    ones, on a few contexts), and the many zero positions push exponent branches of fixed contexts through the
    renormalisation of a count at 255."""
    rng = np.random.default_rng(73)
    img = with_quant(random_coef_image(rng, ncmp=1, mcuh=16, mcuv=12, sf=((1, 1),), nseg=1, density=0.3), Q)
    p = img.planes[0]
    p[:, :49] = np.abs(p[:, :49])
    p[:, EDGE] = 2047
    assert np.count_nonzero(p[:, :49] > 0) > 254 and not np.any(p[:, :49] < 0)
    return [img], 0


def uneven_segments_batch():
    """(d) Groups of one warp whose segments end at different rounds.  One launch holds a single-block image, images of
    one block row, truncated scans that end inside a row (where no count tree of a next block may be read ahead for the
    next row) and long dense segments, more segments than a warp has groups at G >= 4; every group that ends next to one
    that goes on leaves its read-ahead registers behind, and the next segment it takes starts from its own model."""
    rng = np.random.default_rng(74)
    imgs = [
        random_coef_image(rng, ncmp=1, mcuh=1, mcuv=1, sf=((1, 1),), nseg=1),
        random_coef_image(rng, ncmp=3, mcuh=9, mcuv=1, sf=((1, 1), (1, 1), (1, 1)), nseg=1),
        random_coef_image(rng, ncmp=3, mcuh=6, mcuv=6, sf=((2, 2), (1, 1), (1, 1)), nseg=3, density=0.9, amp=100, qscale=0.3),
        random_coef_image(rng, ncmp=3, mcuh=5, mcuv=4, sf=((2, 2), (1, 1), (1, 1)), nseg=2, trunc=True),
        random_coef_image(rng, ncmp=3, mcuh=4, mcuv=5, sf=((2, 1), (1, 1), (1, 1)), nseg=2, trunc="any"),
        random_coef_image(rng, ncmp=1, mcuh=7, mcuv=8, sf=((1, 1),), nseg=4, trunc=True),
        random_coef_image(rng, ncmp=1, mcuh=1, mcuv=6, sf=((1, 1),), nseg=2),
    ]
    imgs.append(with_quant(random_coef_image(rng, ncmp=1, mcuh=4, mcuv=3, sf=((1, 1),), nseg=1), Q))
    imgs[-1].planes[0][:, EDGE] = -2047
    assert any(i.trunc_bc[c] % i.bch[c] for i in imgs[3:6] for c in range(i.ncmp))        # a cut inside a row
    return imgs, 1


HAZARD_BATCHES = [saturated_threshold_batch, word_in_flight_batch, special_state_batch, uneven_segments_batch]


@pytest.mark.parametrize("kernel", GROUPS)
def test_saturated_threshold_index_three_decisions_in_a_row(kernel):
    both_schedules(kernel, *saturated_threshold_batch())


@pytest.mark.parametrize("kernel", GROUPS)
def test_next_decision_reads_the_word_being_written_whatever_the_bit(kernel):
    both_schedules(kernel, *word_in_flight_batch())


@pytest.mark.parametrize("kernel", GROUPS)
def test_long_run_on_one_context_saturates_and_reaches_the_special_state(kernel):
    both_schedules(kernel, *special_state_batch())


@pytest.mark.parametrize("kernel", GROUPS)
def test_segments_end_while_their_neighbours_go_on(kernel):
    nd = both_schedules(kernel, *uneven_segments_batch())
    assert len(nd) > 8 and max(nd) > 20 * min(nd)
