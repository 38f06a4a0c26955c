"""JPEGs embedded in larger files (-embedding=N) through the device kernels on the CPU warp emulator (tests/emu): the jobs
lep_plan.cuh builds for them are those of the plain JPEG -- the prefix never goes to the device -- and the kernels give the
reference's streams, planes, scan and container (tests/golden/embedded.json, tests/golden/make_embedded.py).  The host
then puts the prefix back in front of the SOI, and the zlib0 framing of the result is the reference's -zlib0 output."""
import hashlib
import json
import os
import struct
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import emu  # noqa: E402
import lepfmt  # noqa: E402
from helpers import GOLDEN, read_golden  # noqa: E402
from make_embedded import LEP_FIXTURES, case_bytes, embedding_of  # noqa: E402

EMB = json.load(open(os.path.join(GOLDEN, "embedded.json")))


def md5(b):
    return hashlib.md5(b).hexdigest()


def fixture(name):
    """(input bytes, offset, reference .lep, its segment streams, its bytes in front of the mux packets)."""
    lep = read_golden("embedded/%s.lep" % name)
    lf = lepfmt.parse_container(lep)
    zlen = struct.unpack("<I", lep[24:28])[0]
    return case_bytes(name), embedding_of(EMB["cases"][name]["flags"])[0], lep, lepfmt.demux(lf.payload)[:lf.nseg], lep[:28 + zlen + 3]


@pytest.mark.parametrize("name", LEP_FIXTURES)
def test_range_coder_and_gather_kernels(name):
    """Kernel A + B code the embedded file's planes to the reference's streams, and the gather kernel assembles the
    reference's .lep from them and the host-built header (PGE section included)."""
    from lepton_b200 import HostJpeg
    data, off, lep, streams, head = fixture(name)
    hj = HostJpeg(data, embedding=off, discard_meta="-d" in EMB["cases"][name]["flags"])
    assert hj.status == 0, hj.error
    got = emu.encode_images([hj.coef_image()])[0]
    assert [s for _, s, _ in got] == streams and all(st == 0 for st, _, _ in got), name
    assert emu.mux_files([(head, streams)])[0] == lep, name


@pytest.mark.parametrize("kernel", [emu.KERNEL_WARP, emu.KERNEL_G2(8)])
@pytest.mark.parametrize("name", LEP_FIXTURES)
def test_decode_kernels(name, kernel):
    """Both decode kernels take the reference's streams of an embedded file back to the planes of the JPEG alone."""
    from lepton_b200 import HostJpeg, HostLep
    data, off, lep, streams, _ = fixture(name)
    want = HostJpeg(data[off:]).coef_image()
    img = HostLep(lep).coef_image()
    st, _ = emu.decode_images(kernel, [img], [streams])
    assert st == [0] * len(streams), name
    for a, b in zip(img.planes, want.planes):
        assert np.array_equal(a, b), name


@pytest.mark.parametrize("mode", [emu.HUFF_SERIAL, emu.HUFF_SUBSEQ])
def test_huffman_decode_kernels_see_the_jpeg_alone(mode):
    """The device Huffman decoder's job holds de-stuffed scan bytes and tables only: for an embedded file it is the job of
    the JPEG without the prefix, and the host front end decodes both to the same planes."""
    from lepton_b200 import HostJpeg
    names = [n for n in LEP_FIXTURES if EMB["cases"][n]["flags"] == ["-embedding=%d" % embedding_of(EMB["cases"][n]["flags"])[0]]
             and not n.startswith("trunc")]
    jpegs = []
    for n in names:
        data, off, _, _, _ = fixture(n)
        a, b = HostJpeg(data, embedding=off).coef_image(), HostJpeg(data[off:]).coef_image()
        assert all(np.array_equal(x, y) for x, y in zip(a.planes, b.planes)) and a.luma_y_start == b.luma_y_start, n
        jpegs.append(data[off:])
    res, _ = emu.huffman_decode(mode, jpegs)
    for n, r in zip(names, res):
        assert r is not None and r["status"] == 0, n
        for p, h in zip(r["planes"], r["host_planes"]):
            assert np.array_equal(p, h), n


@pytest.mark.parametrize("name", LEP_FIXTURES)
def test_huffman_encode_kernel_and_restore(name):
    """The Huffman encode kernel writes the scan as it lies in the input, behind prefix, SOI and header; the host puts the
    pieces together to the input (the reference's restore), and frames it as the reference's -zlib0 output."""
    from lepton_b200 import HostJpeg, HostLep
    from lepton_b200.codec import zlib0_frame
    data, off, lep, _, _ = fixture(name)
    rec = EMB["cases"][name]["skipverify"]
    hl = HostLep(lep)
    soff, n = hl.scan_layout()
    if n == 0:                              # truncated: a file for the host re-encoder (test_host_embedded.py)
        assert name.startswith("trunc"), name
        return
    job = emu.henc_job(hl)
    scan, segs = emu.huffman_encode(job, HostJpeg(data, embedding=off).coef_image())
    if "-d" in EMB["cases"][name]["flags"]:
        # -d: the container keeps the size of the file with its metadata, so the promised scan length is too long: the
        # kernel reports the short last segment and the host re-encoder takes the file
        assert any(st for st, _ in segs), name
        return
    assert all(st == 0 for st, _ in segs) and scan == data[soff:soff + n], name
    back = hl.assemble(scan)
    assert back == data and md5(back) == rec["restore"]["md5"], name
    assert md5(zlib0_frame(back)) == rec["restore_zlib0"]["md5"], name

