"""The oracle's rANS coder (container version 3) against the reference's -ans files (tests/golden/ans): its reader decodes
every fixture's streams to the planes of the same JPEG (the version-1 twin's planes) with the same number of decisions, and
its writer makes those streams again, byte for byte."""
import numpy as np
import pytest

import oracle
import oracle_ans
from ans_helpers import ans_cases, load_ans_case
from helpers import geometry_of, segments_of


@pytest.mark.parametrize("name", ans_cases())
def test_reader_decodes_the_reference_streams(name):
    lf, planes, bool_streams, streams, _ = load_ans_case(name)
    g, _, _ = geometry_of(lf)
    got = [np.zeros_like(p) for p in planes]          # blocks a truncated image does not code stay zero
    want = [np.zeros_like(p) for p in planes]
    for i, (y0, y1, last) in enumerate(segments_of(lf)):
        rc, nd = oracle_ans.decode_segment(g, got, y0, y1, last, streams[i])
        rc1, nd1 = oracle.decode_segment(g, want, y0, y1, last, bool_streams[i])
        assert rc == rc1 == 0 and nd == nd1, (name, i, rc, nd, nd1)
    for c in range(len(planes)):
        assert np.array_equal(got[c], planes[c]), (name, c)


@pytest.mark.parametrize("name", ans_cases())
def test_writer_makes_the_reference_streams(name):
    lf, planes, _, streams, _ = load_ans_case(name)
    g, _, _ = geometry_of(lf)
    for i, (y0, y1, last) in enumerate(segments_of(lf)):
        rc, data, _ = oracle_ans.encode_segment(g, planes, y0, y1, last)
        assert rc == 0 and data == streams[i], (name, i, rc, len(data), len(streams[i]))


def test_writer_round_trips_random_tokens():
    """Token streams of every length parity through the writer and back through the reader's decision rule."""
    rng = np.random.default_rng(5)
    for n in (0, 1, 2, 3, 17, 1000, 4097):
        probs = rng.integers(1, 256, n)
        bits = (rng.random(n) * 256 >= probs).astype(np.uint16)       # bit 1 with probability (256 - p) / 256
        rc, data = oracle_ans.ans_encode(probs.astype(np.uint16) | bits << 8)
        assert rc == 0 and len(data) % 4 == 0 and data[-4:] == b"\x00\x80\x00\x80"
        w = [int.from_bytes(data[k:k + 4], "little") for k in range(0, len(data), 4)] + [0] * 4
        x = [w[0] | w[1] << 32, w[2] | w[3] << 32]
        pos = 4
        for k in range(n):
            s = x[0]
            x[0] = x[1]
            p, cf = int(probs[k]), s & 255
            bit = int(cf >= p)
            assert bit == bits[k], (n, k)
            s = (256 - p if bit else p) * (s >> 8) + cf - (p if bit else 0)
            if s < 1 << 31:
                s = s << 32 | w[pos]
                pos += 1
            x[1] = s
    assert oracle_ans.ans_encode(np.array([0x100], np.uint16))[0] == 1       # probability 0 cannot be coded
