"""zlib0 output without a GPU: the Adler-32 the baseline Huffman-encode kernel (lep_huffenc.cu) takes over the bytes each
thread-segment writes, on the CPU warp emulator (tests/emu); the stored-block framing of the host against the reference's
-zlib0 output (tests/golden/zlib0.json, tests/golden/make_zlib0.py); and zeta-headed containers (magic CE B6) in the
host .lep reader."""
import hashlib
import os
import sys
import zlib

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import emu  # noqa: E402
from helpers import (DENSE, EXTREMES, GEOMETRY, GOLDEN, MANIFEST, dense_leps, extreme_leps, geometry_leps,  # noqa: E402
                     read_golden)
from make_zlib0 import sweep_jpeg, zeta  # noqa: E402

ZLIB0 = __import__("json").load(open(os.path.join(GOLDEN, "zlib0.json")))


def adler32_combine(a, b, len_b):
    """zlib's adler32_combine: the Adler-32 of X + Y from those of X and Y and the length of Y."""
    m = 65521
    rem = len_b % m
    s1 = ((a & 0xFFFF) + (b & 0xFFFF) + m - 1) % m
    s2 = (rem * (a & 0xFFFF) + (a >> 16) + (b >> 16) + m - rem) % m
    return (s2 << 16) | s1


def device_recode_gate(e):
    """Files the device Huffman encoder takes (see test_emu_geometry.py): colour, or one 1x1 component without padding."""
    return len(e["sampling"]) == 3 or (e["sampling"] == [[1, 1]] and e["nch"] == e["bch"] and e["ncv"] == e["bcv"])


def henc_cases():
    """(name, JPEG, .lep) of every job the emulator tests of the encode kernel build."""
    out = []
    for n in ["android.jpg", "androidcrop.jpg", "androidcropoptions.jpg", "androidtrail.jpg", "grayscale.jpg", "iphonecrop2.jpg",
              "trailingrst.jpg", "trailingrst2.jpg"]:
        out.append((n, read_golden(n), read_golden(n[:-4] + ".lep")))
    for n in ["androidcrop_t2.lep", "android_t4.lep", "iphonecrop2_t8.lep"]:
        out.append((n, read_golden(MANIFEST[n]["source"]), read_golden(n)))
    for name, source in extreme_leps():
        out.append(("extremes/" + name, read_golden(EXTREMES[source]["path"]), read_golden("extremes/" + name)))
    for name, source in dense_leps():
        out.append(("dense/" + name, read_golden(DENSE[source]["path"]), read_golden("dense/" + name)))
    for name, source in geometry_leps():
        if device_recode_gate(GEOMETRY[source]):
            out.append(("geometry/" + name, read_golden(GEOMETRY[source]["path"]), read_golden("geometry/" + name)))
    return out


CASES = henc_cases()


@pytest.mark.parametrize("reverse", [False, True])
@pytest.mark.parametrize("case", range(len(CASES)), ids=[c[0] for c in CASES])
def test_segment_adler32_of_the_encode_kernel(case, reverse):
    """Every thread-segment's checksum is zlib.adler32 of exactly the bytes it wrote (stuffed zeros and restart markers
    included), the segments lie back to back, their checksums combine to the scan's, and the scan bytes are the original
    file's -- with the emulator's CTAs and threads run in order and in reverse."""
    from lepton_b200 import HostJpeg, HostLep
    name, jpg, lep = CASES[case]
    hl = HostLep(lep)
    assert hl.status == 0, hl.error
    off, n = hl.scan_layout()
    job = emu.henc_job(hl)
    assert n > 0 and job.scan_bytes == n, name
    scan, segs = emu.huffman_encode_segments(job, HostJpeg(jpg).coef_image(), reverse)
    assert scan == jpg[off:off + n], name
    assert [s[0] for s in segs] == [0] * job.nseg, (name, segs)
    pos, whole = 0, zlib.adler32(b"")
    for st, first, produced, ad in segs:
        assert first == pos, (name, segs)
        assert ad == zlib.adler32(scan[first:first + produced]), (name, first, produced)
        whole = adler32_combine(whole, ad, produced)
        pos += produced
    assert pos == n and whole == zlib.adler32(scan), name


def test_cases_cover_the_encode_kernel_jobs():
    assert len(CASES) >= 40
    assert sum(emu.henc_job(__import__("lepton_b200").HostLep(lep)).nseg > 1 for _, _, lep in CASES) >= 20


def blocks(z):
    """Stored-block lengths and BFINAL flags of a zlib0 stream; checks the headers and the trailer on the way."""
    assert z[:2] == b"\x78\x01"
    p, out = 2, []
    while True:
        final, ln, nln = z[p], int.from_bytes(z[p + 1:p + 3], "little"), int.from_bytes(z[p + 3:p + 5], "little")
        assert final in (0, 1) and ln ^ nln == 0xFFFF
        out.append(ln)
        p += 5 + ln
        if final:
            break
    assert p + 4 == len(z)
    return out


@pytest.mark.parametrize("rec", ZLIB0["sweep"], ids=lambda r: str(r["total"]))
def test_host_framing_matches_the_reference(rec):
    """The framing hook gives the reference's -zlib0 output byte for byte over the length sweep (one block, one byte short
    of, exactly at and one past one and two blocks, three full blocks), and zlib takes it back to the JPEG."""
    from lepton_b200.codec import zlib0_frame
    jpg = sweep_jpeg(rec["total"])
    assert hashlib.md5(jpg).hexdigest() == rec["jpg_md5"]
    z = zlib0_frame(jpg)
    assert len(z) == rec["zlib0_size"] == 2 + len(jpg) + 5 * -(-len(jpg) // 65535) + 4
    assert hashlib.md5(z).hexdigest() == rec["zlib0_md5"]
    assert zlib.decompress(z) == jpg
    b = blocks(z)
    assert b[:-1] == [65535] * (len(b) - 1) and 0 < b[-1] <= 65535


def test_host_framing_small_and_empty():
    from lepton_b200.codec import zlib0_frame
    for n in (0, 1, 2, 65534, 65535, 65536):
        data = bytes((7 * i) & 0xFF for i in range(n))
        z = zlib0_frame(data)
        assert zlib.decompress(z) == data and int.from_bytes(z[-4:], "big") == zlib.adler32(data)


@pytest.mark.parametrize("rel", sorted(ZLIB0["leps"]))
def test_host_lep_opens_zeta_copies(rel):
    """A zeta copy opens with the status, geometry, splits and segment streams of the tau file, and says it is zeta."""
    from lepton_b200 import HostLep
    lep = read_golden(rel)
    a, b = HostLep(lep), HostLep(zeta(lep))
    assert (a.status, a.error) == (b.status, b.error), rel
    assert not a.zlib0 and b.zlib0
    if a.status:
        return
    ia, ib = a.coef_image(), b.coef_image()
    for f in ("ncmp", "mcuv", "bch", "bcv", "qtables_zigzag", "luma_y_start", "trunc_bcv", "trunc_bc"):
        assert getattr(ia, f) == getattr(ib, f), (rel, f)
    nseg = len(ia.luma_y_start)
    assert a.streams(nseg) == b.streams(nseg), rel
    assert a.scan_layout() == b.scan_layout(), rel
