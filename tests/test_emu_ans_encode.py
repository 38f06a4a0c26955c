"""Coding rANS segment streams (container version 3) on the CPU warp emulator: kernel A with the rANS model and the rANS
pass (lep_encode.cu), held to the reference's fixtures and to the oracle's writer, at the pass's own edges."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (os.path.join(HERE, "emu"), os.path.join(os.path.dirname(HERE), "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

import emu  # noqa: E402
import emu_ans_encode as E  # noqa: E402
import oracle_ans  # noqa: E402
from ans_helpers import ans_cases, image_geometry, image_segments, load_ans_case  # noqa: E402
from helpers import coef_image_from_lep, random_coef_image  # noqa: E402

ANS, BOOL = E.CODER_ANS, E.CODER_BOOL
L55 = 1 << 55


def tok(p, bit):
    return np.uint16(p | (bit << 8))


def random_tokens(rng, n, lo=1, hi=256):
    return (rng.integers(lo, hi, n) | (rng.integers(0, 2, n) << 8)).astype(np.uint16)


def check_pass(streams, tok_caps=None):
    """The pass on token streams equals the oracle's writer, stays inside its slot and within ans_stream_bound."""
    res, bad = E.ans_pass(streams, tok_caps)
    assert bad == 0
    for t, (st, got) in zip(streams, res):
        rc, want = oracle_ans.ans_encode(t)
        assert (st, got) == (rc, want), (len(t), st, rc, len(got), len(want))
        assert len(got) <= E.stream_bound(len(t))
    return res


# ---------------------------------------------------------------------------------------------------- kernel A + pass
@pytest.mark.parametrize("name", ans_cases())
def test_reference_fixture_streams(name):
    """Every version-3 fixture: the planes and segments of its version-1 twin (the same input and flags), coded by kernel A
    with the rANS model and the pass, give the fixture's own segment streams and the oracle's, byte for byte."""
    lf, planes, _, want, _ = load_ans_case(name)
    img = coef_image_from_lep(lf, planes)
    res, _ = E.encode_images([img], [ANS])
    g = image_geometry(img)
    oracle = [oracle_ans.encode_segment(g, img.planes, *seg) for seg in image_segments(img)]
    assert [s for s, _, _ in res[0]] == [0] * img.nseg
    assert [d for _, d, _ in res[0]] == list(want)
    assert [d for _, d, _ in res[0]] == [s for _, s, _ in oracle]
    assert [n for _, _, n in res[0]] == [n for _, _, n in oracle]


@pytest.mark.parametrize("kernel", [0, 1, 2])
def test_mixed_batch_keeps_the_bool_streams(kernel):
    """Bool and rANS images interleaved in one batch: the bool streams are those of a bool-only run (every range coder
    form), the rANS streams the oracle's, and both come back in the caller's order."""
    rng = np.random.default_rng(31)
    imgs = [random_coef_image(rng, ncmp=3, mcuh=int(rng.integers(2, 6)), mcuv=int(rng.integers(2, 5)), nseg=int(rng.integers(1, 4)))
            for _ in range(6)]
    coders = [ANS, BOOL, BOOL, ANS, ANS, BOOL]
    bool_only = emu.encode_images(imgs, kernel=kernel)
    res, _ = E.encode_images(imgs, coders, kernel=kernel)
    for img, c, got, ref in zip(imgs, coders, res, bool_only):
        if c == BOOL:
            assert got == ref
        else:
            g = image_geometry(img)
            want = [oracle_ans.encode_segment(g, img.planes, *seg) for seg in image_segments(img)]
            assert got == [(rc, s, n) for rc, s, n in want]


def test_token_overflow_keeps_status_100():
    """A segment whose token bound is too small stops with 100 in kernel A, and the pass leaves it so."""
    rng = np.random.default_rng(5)
    img = random_coef_image(rng, ncmp=3, mcuh=4, mcuv=4, nseg=2, density=0.6)
    full, _ = E.encode_images([img], [ANS])
    nd = [n for _, _, n in full[0]]
    res, caps = E.encode_images([img], [ANS], token_bounds=[[8, nd[1]]])
    assert caps[0] < nd[0]
    assert res[0][0][:2] == (100, b"")
    assert res[0][1] == full[0][1]


# ---------------------------------------------------------------------------------------------------- the pass alone
@pytest.mark.parametrize("n", list(range(0, 41)) + [255, 256, 257, 511, 777])
def test_random_token_streams(n):
    rng = np.random.default_rng(100 + n)
    check_pass([random_tokens(rng, n), random_tokens(rng, n, 100, 160)])


@pytest.mark.parametrize("t", [tok(1, 0), tok(255, 1), tok(128, 0)], ids=["p1_bit0", "p255_bit1", "p128_bit0"])
@pytest.mark.parametrize("n", [1, 2, 7, 40, 333, 4096])
def test_uniform_streams(t, n):
    """(1, 0) and (255, 1): freq 1, 8 bits per decision, the largest output; (128, 0): one bit per decision."""
    (st, got), = check_pass([np.full(n, t, np.uint16)])
    if t != tok(128, 0) and n >= 40:
        assert len(got) >= n - 8            # close to the bound: the bound is not loose where it matters


def test_stream_above_2_20_tokens():
    rng = np.random.default_rng(9)
    n = (1 << 20) + 4097
    t = random_tokens(rng, n)
    t[: n // 3] = tok(1, 0)                 # a long stretch of 8-bit decisions, written right behind the reads
    check_pass([t])


def test_token_of_probability_0_asserts():
    t = np.array([tok(10, 1), tok(0, 1), tok(3, 0)], np.uint16)
    (st, got), = E.ans_pass([t])[0]
    assert (st, got) == (oracle_ans.ans_encode(t)[0], b"") and st == 1


@pytest.mark.parametrize("n", [3, 200, 4097, 100000])
def test_probability_0_streams_stay_in_their_slots(n):
    """Long streams of (0, 0) and (0, 1) tokens (a decision of freq 0 for the reference's writer, which asserts): status 1,
    and nothing written in front of the first slot, behind any slot or into the neighbouring segments."""
    rng = np.random.default_rng(n)
    zero0, zero1 = np.full(n, tok(0, 0), np.uint16), np.full(n, tok(0, 1), np.uint16)
    mixed = random_tokens(rng, n)
    mixed[::7] = tok(0, 0)
    good = random_tokens(rng, n + 5)
    res, bad = E.ans_pass([zero0, good, zero1, mixed, good])
    assert bad == 0
    assert [st for st, _ in res] == [1, 0, 1, 1, 0]
    assert res[1] == res[4] == oracle_ans.ans_encode(good)
    assert all(d == b"" for st, d in res if st)


def test_slot_too_small_gives_100():
    """A token slot that cannot hold the stream behind the unread tokens (never one of token_slot's) is refused with 100;
    nothing is written outside the slot."""
    n = 200
    t = np.full(n, tok(1, 0), np.uint16)
    assert not E.slot_fits(n, n) and E.slot_fits(n, (n + 64 + 63) // 64 * 64)
    res, bad = E.ans_pass([t, t], tok_caps=[n, 0])
    assert bad == 0
    assert res[0] == (100, b"")
    assert res[1] == oracle_ans.ans_encode(t)


def py_put(x, p, bit):
    start, f = (p, 256 - p) if bit else (0, p)
    word = None
    if x >= L55 * f:
        word, x = x & 0xffffffff, x >> 32
    return ((x // f) << 8) + x % f + start, word


def test_states_on_the_emission_threshold():
    """One decision at x = 2^55 freq - 1 (no word), 2^55 freq (a word) and 2^55 freq + 1, for every (p, bit)."""
    xs, toks = [], []
    for p in range(1, 256):
        for bit in (0, 1):
            f = 256 - p if bit else p
            for x in (L55 * f - 1, L55 * f, L55 * f + 1, (1 << 31), (1 << 63) - 1 if f == 256 else L55 * f - 2):
                if x < (1 << 63):
                    xs.append(x), toks.append(p | bit << 8)
    xo, w, e = E.ans_put(xs, toks)
    for x, t, a, b, c in zip(xs, toks, xo, w, e):
        want, word = py_put(x, t & 255, t >> 8)
        assert (int(a), bool(c)) == (want, word is not None), (x, t)
        if word is not None:
            assert int(b) == word


def threshold_hits(t):
    """States of the writer's two chains that sit exactly on the emission threshold 2^55 freq of their next decision."""
    n = len(t)
    seq = [(128, 0)] * 8 + ([(1, 1)] if n % 2 else []) + [(int(v) & 255, int(v) >> 8) for v in t[::-1]]
    x, hits = [1 << 31, 1 << 31], 0
    for i, (p, bit) in enumerate(seq):
        f = 256 - p if bit else p
        hits += x[i % 2] == L55 * f
        x[i % 2] = py_put(x[i % 2], p, bit)[0]
    return hits


def test_streams_through_the_threshold():
    """Token streams whose states reach 2^55 freq exactly (the first state at which a word leaves): after the trailing
    pairs both states are 2^35; (1, 0) multiplies a state by 256, (64, 0) by 4, (128, 0) by 2, so 2^(55 + k) meets a
    decision of freq 2^k (k < 8: freq 256 would need p = 0)."""
    for k in range(8):
        per_state = [tok(1, 0)] * 2 + [tok(64, 0)] * 2 + [tok(128, 0)] * k + [tok(2 ** k, 0)]
        t = np.array([v for v in per_state for _ in range(2)][::-1] * 3, np.uint16)       # both states, coded last to first
        assert threshold_hits(t) >= 2, k
        check_pass([t, t[1:]])


# ---------------------------------------------------------------------------------------------------- division and bound
def test_division_is_exact():
    xs, fs = [], []
    for f in range(1, 257):
        for k in (1, 2, 3, 255, 256, 1 << 23, (1 << 40) + 7, (1 << 63) // f - 1, (1 << 63) // f):
            for x in (k * f - 1, k * f):
                if 0 <= x < (1 << 63):
                    xs.append(x), fs.append(f)
        for x in (L55 * f - 1, L55 * f + 1, (1 << 63) - 1, 0, 1):
            if x < (1 << 63):
                xs.append(x), fs.append(f)
    q, r = E.ans_divide(xs, fs)
    for x, f, a, b in zip(xs, fs, q, r):
        assert (int(a), int(b)) == divmod(x, f), (x, f)


def test_stream_bound_and_slot():
    for n in (0, 1, 2, 39, 40, 1 << 20, (1 << 25) - 9, 1 << 25, 3 * 10 ** 9):
        assert E.stream_bound(n) == n + 29 + ((n + 9) >> 25)
    for n in (0, 1, 63, 64, 1000, (1 << 20) + 5, 2 * 10 ** 9):
        cap = (n + 64 + 63) // 64 * 64                      # token_slot
        assert E.slot_fits(n, cap)
    assert E.stream_bound(40) <= 40 + 40
