"""JPEGs embedded in larger files (-embedding=N) and -d on the host (CPU, no GPU): the JPEG front end plus the container
writer reproduce every .lep the unmodified reference CLI wrote (tests/golden/embedded.json, tests/golden/make_embedded.py)
when fed segment streams from the CPU oracle; the .lep reader takes the PGE section and still refuses PGR / SIZ."""
import hashlib
import json
import os
import struct
import sys
import zlib

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from helpers import GOLDEN, oracle_encode_image, read_golden  # noqa: E402
from make_embedded import LEP_FIXTURES, case_bytes, embedding_of, expected_status  # noqa: E402

EMB = json.load(open(os.path.join(GOLDEN, "embedded.json")))
CASES = sorted(EMB["cases"])
THREADS = {"skipverify": 1, "t4": 4, "t8": 8}


def md5(b):
    return hashlib.md5(b).hexdigest()


def host_lep(data, flags, min_threads):
    """(status, .lep) from the host front end, the CPU oracle's segment streams and the host container writer."""
    from lepton_b200 import HostJpeg
    off, discard = embedding_of(flags)
    hj = HostJpeg(data, min_threads=min_threads, embedding=off, discard_meta=discard)
    if hj.status:
        return hj.status, b""
    streams = [s for _, s, _ in oracle_encode_image(hj.coef_image())]
    return 0, hj.write_lep(streams)


@pytest.mark.parametrize("run", sorted(THREADS))
@pytest.mark.parametrize("case", CASES)
def test_front_end_and_container_match_reference(case, run):
    e = EMB["cases"][case]
    data = case_bytes(case)
    assert md5(data) == e["md5"], case
    r = e[run]
    st, lep = host_lep(data, e["flags"], THREADS[run])
    assert st == expected_status(r), (case, run, st, r)
    if st == 0:
        assert md5(lep) == r["lep_md5"], (case, run)


def test_offset_zero_gives_the_plain_lep():
    e = EMB["cases"]["android.jpg_e0"]
    assert e["skipverify"]["lep_md5"] == md5(read_golden("android.lep"))


def test_fixtures_are_the_recorded_files():
    for name in LEP_FIXTURES:
        assert md5(read_golden("embedded/%s.lep" % name)) == EMB["cases"][name]["skipverify"]["lep_md5"], name


def blob_sections(lep):
    """The inflated header blob of a version-1 .lep and its compressed length."""
    zlen = struct.unpack("<I", lep[24:28])[0]
    return zlib.decompress(lep[28:28 + zlen]), zlen


def with_blob(lep, blob):
    """The .lep with its header blob replaced by `blob`."""
    zlen = struct.unpack("<I", lep[24:28])[0]
    z = zlib.compress(blob, 9)
    return lep[:24] + struct.pack("<I", len(z)) + z + lep[28 + zlen:]


@pytest.mark.parametrize("name", LEP_FIXTURES)
def test_reader_takes_the_prefix_section(name):
    """PGE opens: geometry, splits and streams as the reference wrote them, the scan after SOI + header + prefix."""
    from lepton_b200 import HostLep
    lep = read_golden("embedded/%s.lep" % name)
    blob, _ = blob_sections(lep)
    assert b"PGE" in blob
    hl = HostLep(lep)
    assert hl.status == 0, hl.error
    off, n = hl.scan_layout()
    data = case_bytes(name)
    emb = embedding_of(EMB["cases"][name]["flags"])[0]
    if n:
        # the device re-encode's scan lies behind the prefix, the SOI and the header, and ends before the trailer
        assert data[emb:emb + 2] == b"\xff\xd8" and emb + 2 < off and off + n < len(data), (name, off, n)


@pytest.mark.parametrize("tag", [b"PGR", b"SIZ"])
def test_reader_refuses_slice_sections(tag):
    """The -startbyte slice sections stay outside this build: 200, never a wrong answer."""
    from lepton_b200 import HostLep
    lep = read_golden("embedded/trailingrst.jpg_p255_t1.lep")
    blob, _ = blob_sections(lep)
    i = blob.index(b"PGE")
    hl = HostLep(with_blob(lep, blob[:i] + tag + blob[i + 3:]))
    assert hl.status == 200, (hl.status, hl.error)


def test_prefix_comes_back_through_the_host_recoder():
    """The host baseline re-encoder writes prefix, SOI and header in front of the scan: every recorded baseline case with a
    prefix restores to its input from the reference's planes (host Huffman decode of the input)."""
    from lepton_b200 import HostJpeg, HostLep
    for name in ("trailingrst.jpg_p255_t1", "all22_tall.jpg_p70000_t1", "trunc_p1001"):
        e = EMB["cases"][name]
        lep = read_golden("embedded/%s.lep" % name)
        data = case_bytes(name)
        img = HostJpeg(data, embedding=embedding_of(e["flags"])[0]).coef_image()
        got = HostLep(lep).recode(img.planes)
        assert md5(got) == e["skipverify"]["restore"]["md5"] and got == data, name
