"""Device container assembly (SURVEY 8(f) row 3) without a GPU: the data-free MuxWriter plan of the product library
(lepb200_host_mux_plan) + lep_gather_kernel on the CPU warp emulator must reproduce reference-written .lep files byte for
byte from their own header and demuxed streams -- the same pieces lepb200_encode_fetch_files hands the kernel on the device."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu  # noqa: E402
import lepfmt
from helpers import GOLDEN, extreme_leps, golden_leps, read_golden


def split_lep(raw):
    """(everything in front of the mux packets, streams) of a .lep file"""
    lf = lepfmt.parse_container(raw)
    streams = lepfmt.demux(lf.payload)[:lf.nseg]
    return raw[:lf.payload_off], [bytes(s) for s in streams]


def test_golden_leps_reassembled_in_one_launch():
    raws = [open(os.path.join(GOLDEN, n), "rb").read() for n in golden_leps()]
    files = [split_lep(r) for r in raws]
    assert sum(len(ss) for _, ss in files) > len(files)            # multi-segment files among them
    got = emu.mux_files(files, grid=3)
    for n, g, r in zip(golden_leps(), got, raws):
        assert g == r, n


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_stream_lengths_match_the_host_writer(seed):
    """Stream lengths around every threshold of the writer (256 / 4096 / 8192 / 16384 / 32768 / 65536 / 131072 bytes and the
    65537-byte lag that makes a stream 'urgent'), 1 to 16 streams, odd header lengths (every source / destination
    alignment): the emulated device assembly equals the host writer's bytes (HostJpeg.write_lep's mux, itself pinned
    against the reference's files)."""
    from lepton_b200.codec import lib
    rng = np.random.default_rng(seed)
    marks = [0, 1, 255, 256, 257, 4095, 4096, 4097, 8192, 8193, 16384, 32768, 32769, 65535, 65536, 65537, 131072, 131073, 200000]
    files = []
    for f in range(6):
        nseg = int(rng.integers(1, 17))
        lens = [int(max(0, rng.choice(marks) + rng.integers(-3, 4))) if rng.random() < 0.7 else int(rng.integers(0, 300000)) for _ in range(nseg)]
        if f == 0:
            lens = [0] * nseg                                        # nothing but header and trailer
        streams = [rng.integers(0, 256, size=n, dtype=np.uint8).tobytes() for n in lens]
        hdr = rng.integers(0, 256, size=int(rng.integers(29, 900)), dtype=np.uint8).tobytes()
        files.append((hdr, streams))
    got = emu.mux_files(files, grid=5)
    for (hdr, streams), g in zip(files, got):
        plan, n = emu.mux_plan([len(s) for s in streams])
        want = bytearray(hdr)
        for k in range(n):
            p = plan[k]
            want += bytes(p.hdr[:p.nhdr]) + streams[p.id][p.src_off:p.src_off + p.len]
        want += (len(want) + 4).to_bytes(4, "little")
        assert g == bytes(want)
        # the plan covers every stream exactly once, in order
        seen = [0] * len(streams)
        for k in range(n):
            p = plan[k]
            assert p.src_off == seen[p.id]
            seen[p.id] += p.len
        assert seen == [len(s) for s in streams]


def test_extreme_corpus_leps_reassembled():
    """The reference's .lep files of the extreme corpus (one, four and eight segments) from their own pieces."""
    names = [n for n, _ in extreme_leps()]
    raws = [read_golden("extremes/" + n) for n in names]
    got = emu.mux_files([split_lep(r) for r in raws], grid=3)
    for n, g, r in zip(names, got, raws):
        assert g == r, n
