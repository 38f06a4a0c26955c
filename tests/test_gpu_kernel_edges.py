"""The range coder, gather and decode kernels on the device, at the inputs built to break them.

The emulator suite (tests/emu) runs these inputs with CTAs one after the other and plain memory.  Here they run through
the library's own launch code on the GPU, where what the emulator cannot show is real: the cp.async token ring of the
range pass and its prologue, the plain stores and atomic adds of piece CTAs that run at the same time, persistent work
queues shared by CTAs that run together, the group kernel's shared-memory front region at two CTAs per SM, and the
batch-size switches of the token feed and of the decode kernel.

Expected values come from the oracle (oracle.bool_encode, oracle.decode_segment, and oracle_ans for the rANS coder of
container version 3) or from the host writer's mux plan (lepb200_host_mux_plan); the inputs are the emulator tests' own
builders.
"""
import functools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu  # noqa: E402
import oracle  # noqa: E402
import test_emu_decode_lookahead as lookahead  # noqa: E402
import test_emu_model_interleave as interleave  # noqa: E402
import test_emu_rangecoder as rangecoder  # noqa: E402
from ans_helpers import judge, oracle_ans_streams, traces  # noqa: E402
from helpers import oracle_encode_image, random_coef_image  # noqa: E402
from test_emu_rangecoder import carry_tokens, random_tokens, tok  # noqa: E402

pytestmark = pytest.mark.gpu

# range coder forms: (environment, serial)
RC_FORMS = {
    "pieces-ring": ({"LEPB200_RC_MODE": "1", "LEPB200_RC_FEED": "1"}, False),
    "pieces-registers": ({"LEPB200_RC_MODE": "1", "LEPB200_RC_FEED": "0"}, False),
    "serial": ({"LEPB200_RC_MODE": "0"}, True),
}
# decode kernels: warp per segment, and the group kernel at every lane count the library ships; 32 segments per launch so
# that the groups of a launch share one queue and take second jobs
DEC_FORMS = {
    "warp": {"LEPB200_DEC_MODE": "1"},
    "group4": {"LEPB200_DEC_MODE": "2", "LEPB200_DEC_LANES": "4", "LEPB200_DEC_THREADS": "32"},
    "group8": {"LEPB200_DEC_MODE": "2", "LEPB200_DEC_LANES": "8", "LEPB200_DEC_THREADS": "32"},
    "group32": {"LEPB200_DEC_MODE": "2", "LEPB200_DEC_LANES": "32", "LEPB200_DEC_THREADS": "32"},
}
TUNING = ("LEPB200_RC_MODE", "LEPB200_RC_FEED", "LEPB200_DEC_MODE", "LEPB200_DEC_LANES", "LEPB200_DEC_THREADS",
          "LEPB200_DEC_GROUP_MIN")


def codec_with(monkeypatch, env):
    """A context created under `env` and nothing else of the library's tuning variables (it reads them when created)."""
    from lepton_b200 import LeptonB200Codec
    for k in TUNING:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    return LeptonB200Codec(0)


@pytest.fixture(params=list(RC_FORMS))
def range_coder(request, monkeypatch):
    """-> code(streams, cap_delta=, caps=): rangecoder.check on the library's range coder in one of its forms"""
    env, serial = RC_FORMS[request.param]
    c = codec_with(monkeypatch, env)
    yield lambda streams, **kw: rangecoder.check(1 if serial else 0, False, streams, run=c.range_code, **kw)
    c.close()


# ---------------------------------------------------------------------------------------------------- range coder
@pytest.mark.parametrize("case", rangecoder.CASES, ids=lambda f: f.__name__)
def test_range_coder_cases_of_the_emulator_suite(range_coder, case):
    case(range_coder)


def test_token_counts_around_loads_ring_and_piece_borders(range_coder):
    """The tail loop of 8-token loads, a cp.async ring whose prologue commits empty groups (fewer full loads than ring
    slots), and checkpoints that fall on piece borders; tight and roomy slots."""
    rng = np.random.default_rng(21)
    counts = [0, 1, 7, 8, 9, 255, 256, 257, 1023, 1024, 1025, 2048]
    streams = [random_tokens(rng, n) for n in counts]
    range_coder(streams, cap_delta=4096)
    range_coder(streams, cap_delta=0)


def test_segment_of_more_than_sixteen_million_tokens(range_coder):
    """2^24 + tokens in one segment with carry walks inside, in a slot too small: the stream moves to the overflow arena."""
    rng = np.random.default_rng(22)
    s = np.concatenate([random_tokens(rng, 9_000_000), carry_tokens(rng, 3, 3000), random_tokens(rng, 7_800_000)])
    assert len(s) > (1 << 24)
    range_coder([s], cap_delta=-1000)


def test_batch_past_the_feed_switch_takes_the_default_feed(monkeypatch):
    """More than 8192 segments with no feed override: the library's own switch picks the register feed.  Short random
    streams, every 97th a carry walk, slots from far too small to roomy."""
    c = codec_with(monkeypatch, {})
    rng = np.random.default_rng(23)
    streams = [carry_tokens(rng, 2, 1200) if k % 97 == 5 else random_tokens(rng, int(rng.integers(0, 400))) for k in range(8300)]
    oracle.bool_counts(reset=True)
    lens = [len(oracle.bool_encode(s)[1]) for s in streams]
    assert oracle.bool_counts()["walks_64"] > 0
    caps = [max(1, int(n * f)) for n, f in zip(lens, rng.choice([0.5, 1.0, 1.01, 2.0], len(lens)))]
    try:
        rangecoder.check(0, False, streams, caps=caps, run=c.range_code)
    finally:
        c.close()


# ---------------------------------------------------------------------------------------------------- gather
def exact_length_tokens(rng, n_bytes):
    """Tokens of probability 128 shift exactly one bit each, so their count sets the stream length: -> tokens whose
    oracle stream is n_bytes long (n_bytes >= 2: marker and stop bits alone make 2 bytes)."""
    n = max(0, 8 * (n_bytes - 2))
    while True:
        t = tok(rng.integers(0, 2, n), np.full(n, 128))
        got = len(oracle.bool_encode(t)[1])
        if got == n_bytes:
            return t
        n = max(0, n + 8 * (n_bytes - got) + (1 if got < n_bytes else -1))


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_gather_assembles_the_host_writers_files(monkeypatch, seed):
    """Stream lengths around every threshold of the writer (256 / 4096 / 8192 / 16384 / 32768 / 65536 / 131072 bytes and
    the 65537-byte lag that makes a stream urgent), the shortest stream the coder makes, 1 to 16 segments per file, and
    16 files whose header lengths take every residue mod 16 (every destination alignment), in one launch of the gather
    kernel through lepb200_encode_fetch_files: byte for byte the file the host writer's mux plan makes of the oracle's
    streams."""
    c = codec_with(monkeypatch, {})
    rng = np.random.default_rng(100 + seed)
    marks = [2, 3, 255, 256, 257, 4095, 4096, 4097, 8192, 8193, 16384, 32768, 32769, 65535, 65536, 65537, 131072, 131073]
    streams, per_file, headers, want_streams = [], [], [], []
    for f in range(16):
        nseg = int(rng.integers(1, 17))
        lens = [int(max(2, rng.choice(marks) + rng.integers(-3, 4))) for _ in range(nseg)]
        toks = [exact_length_tokens(rng, n) for n in lens]
        streams += toks
        per_file.append(nseg)
        want_streams.append([oracle.bool_encode(t)[1] for t in toks])
        hlen = 29 + (f * 7) % 16 + 16 * int(rng.integers(0, 50))
        headers.append(rng.integers(0, 256, size=hlen, dtype=np.uint8).tobytes())
    assert sorted(len(h) % 16 for h in headers) == list(range(16))
    caps = [len(oracle.bool_encode(t)[1]) + 64 for t in streams]
    try:
        files, moved, bad = c.range_code(streams, caps, files=per_file, headers=headers)
    finally:
        c.close()
    assert bad == 0 and not any(moved)
    for f, ((st, got), hdr, ss) in enumerate(zip(files, headers, want_streams)):
        plan, n = emu.mux_plan([len(s) for s in ss])
        want = bytearray(hdr)
        for k in range(n):
            p = plan[k]
            want += bytes(p.hdr[:p.nhdr]) + ss[p.id][p.src_off:p.src_off + p.len]
        want += (len(want) + 4).to_bytes(4, "little")
        assert st == 0, f
        assert got == bytes(want), f


# ---------------------------------------------------------------------------------------------------- decode
# Every decode batch below runs once with bool-coded streams (container versions 1, 2, 4) and once with rANS-coded ones
# (version 3): same grammar and batches, the other coder's kernels, judged against that coder's oracle.
BOOL, ANS = 0, 1
CODERS = {"bool": BOOL, "ans": ANS}


def device_run(codec):
    """ans_helpers.judge's run on a context: -> (status, decision count) of every segment"""
    def run(out, streams, coders):
        st = codec.decode_images(out, streams, coders)
        return st, codec.decode_decisions()
    return run


def decode_vs_oracle(codec, imgs, streams, coder=BOOL, refused=()):
    """Decodes `streams` for `imgs` in one batch of one coder (bool: the entry point without a coder argument): status,
    decision count and planes of every segment are the oracle's.  -> the oracle's statuses"""
    return judge(device_run(codec), imgs, streams, None if coder == BOOL else [coder] * len(imgs), refused)


def oracle_streams(imgs, coder=BOOL):
    if coder == ANS:
        return oracle_ans_streams(imgs)
    refs = [oracle_encode_image(img) for img in imgs]
    for r in refs:
        assert all(rc == 0 for rc, _, _ in r)
    return [[s for _, s, _ in r] for r in refs]


@pytest.fixture(params=list(DEC_FORMS))
def decoder(request, monkeypatch):
    c = codec_with(monkeypatch, DEC_FORMS[request.param])
    yield c
    c.close()


@pytest.fixture(params=list(CODERS))
def coder(request):
    return CODERS[request.param]


@pytest.mark.parametrize("batch", lookahead.HAZARD_BATCHES, ids=lambda f: f.__name__)
def test_read_ahead_hazard_batches(decoder, batch, coder):
    """With the rANS coder the special-state batch is the saturate-and-restart case: its all-ones sign branch counts
    up to c1 = 255, restarts at 129 and decides at probability 1 (the rANS model has no special state)."""
    imgs, _ = batch()
    streams = oracle_streams(imgs, coder)
    if coder == ANS and batch is lookahead.special_state_batch:
        t = traces(imgs, streams)
        assert np.any((t["c0"] == 1) & (t["c1"] == 255) & (t["bit"] == 1))
        assert np.any((t["c1"] == 129) & (t["prob"] < 128)) and np.any(t["prob"] == 1)
    decode_vs_oracle(decoder, imgs, streams, coder)


@pytest.mark.parametrize("spec", [interleave.PARTIAL_BLOCK, interleave.SECOND_CLAIMS], ids=["partial_block", "second_claims"])
def test_interleave_batches(decoder, spec, coder):
    sizes, seed, _ = spec
    imgs, streams, want = interleave.batch(sizes, seed)
    for img, (planes, _) in zip(imgs, want):
        img.planes = planes
    if coder == ANS:
        streams = oracle_ans_streams(imgs)
    decode_vs_oracle(decoder, imgs, streams, coder)


@functools.lru_cache(maxsize=None)
def small_segments(n, coder=BOOL, seed=31):
    """Images of 1..16 one-row segments, n segments in all, with their oracle streams."""
    rng = np.random.default_rng(seed + n)
    imgs, streams, left = [], [], n
    while left:
        nseg = min(left, int(rng.integers(1, 17)))
        img = random_coef_image(rng, ncmp=1, mcuh=int(rng.integers(1, 4)), mcuv=nseg, sf=((1, 1),), nseg=nseg, density=0.4)
        imgs.append(img)
        left -= nseg
    return imgs, oracle_streams(imgs, coder)


SEGMENT_COUNTS = list(range(1, 18)) + [23, 25, 63, 65, 255, 257, 1023, 1025, 6143, 6145, 6151, 6153]


@pytest.mark.parametrize("n", SEGMENT_COUNTS)
def test_segment_counts_of_every_residue_mod_8(monkeypatch, n, coder):
    """The batches below with the kernel the library picks itself: the warp kernel up to 6143 segments, the group kernel
    at 4 lanes from 6144 on (6145, 6151 and 6153: a partial last warp and interleave block in one launch).  A batch of
    one coder is one part, so the switch applies to the rANS part alone as it does to the bool one."""
    c = codec_with(monkeypatch, {})
    imgs, streams = small_segments(n, coder)
    try:
        decode_vs_oracle(c, imgs, streams, coder)
    finally:
        c.close()


# every kernel the library ships, each batch in ONE launch (no cap on the segments per launch)
ONE_LAUNCH_FORMS = {
    "warp": {"LEPB200_DEC_MODE": "1"},
    "group4": {"LEPB200_DEC_MODE": "2", "LEPB200_DEC_LANES": "4"},
    "group8": {"LEPB200_DEC_MODE": "2", "LEPB200_DEC_LANES": "8"},
    "group32": {"LEPB200_DEC_MODE": "2", "LEPB200_DEC_LANES": "32"},
}


@pytest.mark.parametrize("n", [n for n in SEGMENT_COUNTS if n < 6144])
@pytest.mark.parametrize("form", list(ONE_LAUNCH_FORMS))
def test_segment_counts_of_every_residue_mod_8_on_every_kernel(monkeypatch, form, n, coder):
    """Batches whose segment count takes every residue mod 8 forced onto each kernel: in the group kernel, a last warp
    with 1..7 of its groups busy (at 4 lanes; 1..3 at 8 lanes) and a partial last interleave block of 1..7 models, in a
    pool of exactly n models; at 32 lanes, one segment per warp."""
    c = codec_with(monkeypatch, ONE_LAUNCH_FORMS[form])
    imgs, streams = small_segments(n, coder)
    try:
        decode_vs_oracle(c, imgs, streams, coder)
    finally:
        c.close()


def test_damaged_streams_next_to_healthy_ones(decoder, coder):
    """48 one-segment images of one geometry (so the launch order is the batch order): every eighth segment from the
    third on is cut short and bit-flipped, so each warp of the group kernel and each interleave block of 8 models holds
    one damaged segment among healthy ones.  Statuses, decision counts and planes (those a failing segment wrote
    included) are the oracle's.  rANS streams are cut to every length residue mod 4 and damaged in the 16 state bytes
    as well as in the body, and one image with a zero quantiser is refused on the host (status 43) inside the batch."""
    rng = np.random.default_rng(41)
    imgs = [random_coef_image(rng, ncmp=3, mcuh=3, mcuv=2, sf=((2, 2), (1, 1), (1, 1)), nseg=1, density=0.6) for _ in range(48)]
    streams = oracle_streams(imgs, coder)
    for i, ss in enumerate(streams):
        if i % 8 == 3:
            b = bytearray(ss[0][:max(8, len(ss[0]) // (2 + i % 5))])
            if coder == ANS:
                b = b[:len(b) - (len(b) - i // 8) % 4]               # lengths of residue 0, 1, 2, 3, 0, 1 mod 4
            lo, hi = 4, len(b)
            if coder == ANS:
                lo, hi = (0, 16) if i // 8 % 2 else (16, len(b))    # the state bytes, or the body
            for _ in range(1 + i % 4):
                b[int(rng.integers(lo, min(hi, len(b))))] ^= int(rng.integers(1, 256))
            ss[0] = bytes(b)
    refused = ()
    if coder == ANS:
        assert sorted({len(ss[0]) % 4 for i, ss in enumerate(streams) if i % 8 == 3}) == [0, 1, 2, 3]
        imgs[21].qtables_zigzag = [[0] + list(q[1:]) for q in imgs[21].qtables_zigzag]
        refused = (21,)
    st = decode_vs_oracle(decoder, imgs, streams, coder, refused)
    assert sum(1 for s in st if s) >= 3 + len(refused)
