"""Streams of concatenated .lep files through the device kernels on the CPU warp emulator (tests/emu): every member of every
case of tests/golden/concat.json that the reference restores goes through a decode kernel and, where the device takes its
scan, the Huffman encode kernel; the host re-encoder takes the rest.  The members' JPEGs joined give the reference's
output, and framed as one zlib stream whose Adler-32 is combined from the encode kernel's segment sums, its -zlib0 output."""
import hashlib
import json
import os
import sys
import zlib

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import emu  # noqa: E402
from helpers import GOLDEN  # noqa: E402
from make_concat import case_bytes, expected  # noqa: E402

CON = json.load(open(os.path.join(GOLDEN, "concat.json")))
RESTORED = sorted(n for n, e in CON["cases"].items() if expected(n, e, "plain")[0] == 0)


def md5(b):
    return hashlib.md5(b).hexdigest()


def adler32_combine(a, b, len_b):
    m = 65521
    rem = len_b % m
    s1 = ((a & 0xFFFF) + (b & 0xFFFF) + m - 1) % m
    s2 = (rem * (a & 0xFFFF) + (a >> 16) + (b >> 16) + m - rem) % m
    return (s2 << 16) | s1


def zlib0(data, adler):
    """One zlib stream of stored 65535-byte blocks over `data` (the last one BFINAL) ending in `adler`."""
    out = bytearray(b"\x78\x01")
    for p in range(0, len(data), 65535):
        b = data[p:p + 65535]
        out += bytes([1 if p + len(b) == len(data) else 0]) + len(b).to_bytes(2, "little") + (len(b) ^ 0xFFFF).to_bytes(2, "little") + b
    return bytes(out) + adler.to_bytes(4, "big")


@pytest.fixture(scope="module", autouse=True)
def brotli():
    from lepton_b200 import lib
    if not lib().lepb200_host_brotli_available():
        pytest.skip("libbrotlidec (libbrotlidec.so.1) not found: the version-2 members of concat.json cannot be read")


def restore_member(data, k, kernel):
    """(JPEG, its Adler-32, whether the device encoded the scan) of member k: decode kernel, then the Huffman encode kernel
    (the scan's Adler-32 from its segment sums, the host's of the bytes around it) or the host re-encoder."""
    from lepton_b200 import HostLep
    hl = HostLep(data, member=k)
    assert hl.status == 0, (k, hl.error)
    img = hl.coef_image()
    streams = hl.streams(img.nseg)
    st, _ = emu.decode_images(kernel, [img], [streams])
    assert st == [0] * img.nseg, k
    off, n = hl.scan_layout()
    if n == 0:
        jpeg = hl.recode(img.planes)
        return jpeg, zlib.adler32(jpeg), False
    scan, segs = emu.huffman_encode_segments(emu.henc_job(hl), img)
    assert all(s[0] == 0 for s in segs), (k, segs)
    jpeg = hl.assemble(scan)
    assert jpeg[off:off + n] == scan
    a = zlib.adler32(jpeg[:off])
    for _, _, produced, ad in segs:
        a = adler32_combine(a, ad, produced)
    return jpeg, adler32_combine(a, zlib.adler32(jpeg[off + n:]), len(jpeg) - off - n), True


@pytest.mark.parametrize("kernel", [emu.KERNEL_WARP, emu.KERNEL_G2(8)], ids=["warp", "g2"])
@pytest.mark.parametrize("name", RESTORED)
def test_members_through_the_kernels(name, kernel):
    from lepton_b200 import lep_members
    e = CON["cases"][name]
    data = case_bytes(e["parts"])
    ms = lep_members(data)
    parts = [restore_member(data, k, kernel) for k in range(len(ms))]
    joined = b"".join(j for j, _, _ in parts)
    if name != "zeta_first":                                     # a CE B6 stream is zlib output without the flag
        assert md5(joined) == e["plain"]["md5"], name
    adler = 1
    for j, a, _ in parts:
        assert a == zlib.adler32(j)
        adler = adler32_combine(adler, a, len(j))
    z = zlib0(joined, adler)
    zkey = "plain" if name == "zeta_first" else "zlib0"
    assert md5(z) == e[zkey]["md5"] and len(z) == e[zkey]["len"], name


def test_cases_reach_the_encode_kernel():
    """Most members' scans are re-encoded by the kernel; the progressive and truncated ones by the host."""
    from lepton_b200 import HostLep, lep_members
    dev = host = 0
    for n in RESTORED:
        data = case_bytes(CON["cases"][n]["parts"])
        for k in range(len(lep_members(data))):
            if HostLep(data, member=k).scan_layout()[1]:
                dev += 1
            else:
                host += 1
    assert dev >= 40 and host >= 20, (dev, host)
