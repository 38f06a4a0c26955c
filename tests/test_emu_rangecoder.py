"""Kernel B (the range coder) alone, on token streams built to reach what its parallel form gets wrong first, against the
oracle's bool coder (oracle.bool_encode, the reference's vpx_write read as C).

The parallel form codes a segment in pieces of 1024 tokens: a range-only pass records a checkpoint per piece, one thread
per piece adds its splits into 16-bit digits (plain stores inside its own bit range, atomic adds on the digits it shares
with its neighbours), and one warp per segment resolves the carries 32 digits at a time and applies the stop rule.  The
streams below hit piece borders, carries that ripple over whole pieces and 32-digit steps, the extra zero byte of
vpx_stop_encode, and stream slots of len - 1 .. len + 2 bytes.  Every case runs under both schedules of the emulator: the
threads of a CTA in order and in reverse order, so a piece that plain-stores a digit its neighbour also adds to loses the
neighbour's part under one of them."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu  # noqa: E402
import oracle  # noqa: E402

# 0 = range-only pass + parallel pieces + carry pass (the default), 1 = one serial chain per segment, 2 = as 0 with the
# range pass's tokens fed through registers (LEPB200_RC_FEED=0)
KERNELS = [0, 1, 2]
SCHEDULES = [False, True]        # reverse


def tok(bit, prob):
    return (np.asarray(prob, dtype=np.uint16) & 0xff) | (np.asarray(bit, dtype=np.uint16) << 8)


def random_tokens(rng, n):
    """The whole token domain: prob 0..255 (0 is what a 'neverseen' branch codes with) with either bit."""
    return tok(rng.integers(0, 2, n), rng.integers(0, 256, n))


def carry_tokens(rng, runs, run_len):
    """Tokens that make carries ripple over long runs of 0xff bytes.  The coder's interval [low, low + range) is followed
    exactly (low as an unbounded integer, in units of the last bit shifted in).  A run picks the roundest point P inside
    the interval and then, for run_len tokens of random probability, the bit whose sub-interval still holds P: the code
    value stays just below P, so every byte that leaves is 0xff.  Large splits ((1, 255) until low passes P) close the run,
    and the carry walks back over all of those bytes."""
    low, rg, out = 0, 255, []

    def put(bit, prob):
        nonlocal low, rg
        split = 1 + (((rg - 1) * prob) >> 8)
        low, rg = (low + split, rg - split) if bit else (low, split)
        sh = 8 - rg.bit_length()
        low, rg = low << sh, rg << sh
        return sh

    put(0, 128)                                                        # the marker bit
    for _ in range(runs):
        hi = low + rg - 1
        b = hi.bit_length()
        while b > 0 and ((hi >> b) << b) <= low:
            b -= 1
        p = (hi >> b) << b                                             # roundest point in (low, low + rg)
        n = 0
        while n < run_len:
            prob = int(rng.integers(1, 256))
            split = 1 + (((rg - 1) * prob) >> 8)
            if low + split == p:
                continue
            bit = int(low + split < p)
            out.append((bit, prob))
            p <<= put(bit, prob)
            n += 1
        while low <= p:
            out.append((1, 255))
            p <<= put(1, 255)
        for _ in range(int(rng.integers(0, 40))):
            out.append((int(rng.integers(0, 2)), int(rng.integers(1, 256))))
            put(*out[-1])
    a = np.array(out, dtype=np.int64).reshape(-1, 2)
    return tok(a[:, 0], a[:, 1])


def check(kernel, reverse, streams, cap_delta=None, caps=None, run=None):
    """Codes `streams` in one launch; every stream must come back with status 0 and the oracle's bytes, no canary byte
    may change, and a stream lies in its slot exactly when the form can know it fits (serial: len < cap; parallel:
    L + 1 < cap, L = len without the stop-rule byte).  run(streams, caps) -> (per segment (status, bytes, moved), changed
    canary bytes) codes them instead of the emulator (the device tests pass the library's range coder).  -> the oracle's
    streams."""
    ref = []
    for s in streams:
        before = oracle.bool_counts()["stop_zero"]
        rc, b = oracle.bool_encode(s)
        assert rc == 0
        ref.append((b, oracle.bool_counts()["stop_zero"] > before))
    if caps is None:
        caps = [max(1, len(b) + cap_delta) for b, _ in ref]
    got, bad = run(streams, caps) if run else emu.range_code(kernel, streams, caps, reverse=reverse)
    assert bad == 0, "%d canary bytes changed" % bad
    for k, ((st, data, moved), (want, stop), cap) in enumerate(zip(got, ref, caps)):
        assert st == 0, (k, st, len(want), cap)
        assert data == want, (k, len(data), len(want), cap)
        need = len(want) if kernel == 1 else len(want) - stop + 1
        assert moved == (need >= cap), (k, moved, len(want), stop, cap)
    return [b for b, _ in ref]


# The cases: each codes its streams with `code(streams, cap_delta=..., caps=...)`, which is `check` bound to one kernel
# and schedule of the emulator or to the library's range coder on the device (test_gpu_kernel_edges.py).
def token_counts_around_pieces_and_loads(code):
    """0 tokens (marker and stop bits only), fewer than one 8-token load, 1024-token piece borders, 8 pieces."""
    rng = np.random.default_rng(11)
    counts = [0, 1, 7, 8, 9, 1023, 1024, 1025, 8 * 1024 - 1, 8 * 1024, 8 * 1024 + 1]
    code([random_tokens(rng, n) for n in counts], cap_delta=4096)


def full_token_domain(code):
    """Every (bit, prob) pair, prob 0 included, many times over, in random order and in long runs of each."""
    rng = np.random.default_rng(12)
    every = tok(np.arange(512) >> 8, np.arange(512) & 0xff)
    runs = np.repeat(every, 9)
    code([rng.permutation(np.tile(every, 20)), runs, runs[::-1].copy()], cap_delta=64)


def carries_across_pieces_and_digit_steps(code):
    """Carry walks of hundreds of bytes.  The longest walk runs back over a run of more than 3000 tokens (any 2048
    consecutive tokens hold a piece border), and walks of 64 bytes or more are longer than a 32-digit step of the carry
    pass."""
    rng = np.random.default_rng(13)
    oracle.bool_counts(reset=True)
    streams = [carry_tokens(rng, 3, 3000), carry_tokens(rng, 6, 1200), carry_tokens(rng, 20, 100)]
    code(streams, cap_delta=64)
    c = oracle.bool_counts()
    assert c["walk_max"] >= 200 and c["walks_64"] >= 6, c


def capacity_edges_and_stop_byte(code):
    """Slots of len - 1, len, len + 1 and len + 2 bytes for 60 streams, about an eighth of which end with the extra zero
    byte of the stop rule: the same bytes in every case, nothing written past a slot, the stream moved to the overflow
    arena exactly when it may not fit."""
    rng = np.random.default_rng(14)
    streams = [random_tokens(rng, int(n)) for n in rng.integers(0, 3000, 60)]
    oracle.bool_counts(reset=True)
    for d in (-1, 0, 1, 2):
        code(streams, cap_delta=d)
    assert oracle.bool_counts()["stop_zero"] >= 4 * 4


def batch_of_mixed_segments(code):
    """240 segments of mixed lengths and kinds in one launch (two CTAs of the range pass, 60 warps of the carry pass),
    slots from far too small to roomy."""
    rng = np.random.default_rng(15)
    streams = []
    for k in range(240):
        n = int(rng.choice([0, 5, 700, 1024, 2100, 5000]))
        streams.append(carry_tokens(rng, 2, 300) if k % 7 == 3 else random_tokens(rng, n))
    lens = [len(oracle.bool_encode(s)[1]) for s in streams]
    caps = [max(1, int(n * f)) for n, f in zip(lens, rng.choice([0.5, 0.99, 1.0, 1.01, 2.0], len(lens)))]
    code(streams, caps=caps)


def stream_of_more_than_a_million_tokens(code):
    """More than 1024 pieces in one segment: the piece threads of the grid (8 CTAs x 128) stride over them."""
    rng = np.random.default_rng(16)
    s = np.concatenate([random_tokens(rng, 600000), carry_tokens(rng, 4, 4000), random_tokens(rng, 450001)])
    assert len(s) > (1 << 20) and len(s) // 1024 > 8 * 128
    code([s], cap_delta=-1000)


CASES = [token_counts_around_pieces_and_loads, full_token_domain, carries_across_pieces_and_digit_steps,
         capacity_edges_and_stop_byte, batch_of_mixed_segments, stream_of_more_than_a_million_tokens]


def on_emulator(kernel, reverse):
    return lambda streams, **kw: check(kernel, reverse, streams, **kw)


@pytest.mark.parametrize("reverse", SCHEDULES)
@pytest.mark.parametrize("kernel", KERNELS)
def test_token_counts_around_pieces_and_loads(kernel, reverse):
    token_counts_around_pieces_and_loads(on_emulator(kernel, reverse))


@pytest.mark.parametrize("reverse", SCHEDULES)
@pytest.mark.parametrize("kernel", KERNELS)
def test_full_token_domain(kernel, reverse):
    full_token_domain(on_emulator(kernel, reverse))


@pytest.mark.parametrize("reverse", SCHEDULES)
@pytest.mark.parametrize("kernel", KERNELS)
def test_carries_across_pieces_and_digit_steps(kernel, reverse):
    carries_across_pieces_and_digit_steps(on_emulator(kernel, reverse))


@pytest.mark.parametrize("reverse", SCHEDULES)
@pytest.mark.parametrize("kernel", KERNELS)
def test_capacity_edges_and_stop_byte(kernel, reverse):
    capacity_edges_and_stop_byte(on_emulator(kernel, reverse))


@pytest.mark.parametrize("reverse", SCHEDULES)
@pytest.mark.parametrize("kernel", KERNELS)
def test_batch_of_mixed_segments(kernel, reverse):
    batch_of_mixed_segments(on_emulator(kernel, reverse))


@pytest.mark.slow
@pytest.mark.parametrize("kernel", KERNELS)
def test_stream_of_more_than_a_million_tokens(kernel):
    stream_of_more_than_a_million_tokens(on_emulator(kernel, kernel == 0))
