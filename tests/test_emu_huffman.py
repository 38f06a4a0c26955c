"""The baseline Huffman decode kernels on the CPU warp emulator (tests/emu): lep_huffdecode_kernel (one warp per image)
and the sub-sequence kernels of lep_huffpar.cu (one thread per sub-sequence of the scan, self-synchronising) must both
reproduce the host decoder's coefficient planes -- which tests/test_host_frontend.py pins to the reference's -ujg dumps --
and must agree with each other on every output the host reads back: status, pad bit, end position and the per-MCU-row
states the thread handoffs are made of."""
import io
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu  # noqa: E402
from helpers import GOLDEN

GOLDEN_JPEGS = ["android.jpg", "androidcrop.jpg", "androidcropoptions.jpg", "androidtrail.jpg", "colorswap.jpg", "grayscale.jpg",
                "iphonecrop2.jpg", "trailingrst.jpg", "trailingrst2.jpg"]


def pil_jpeg(seed, w, h, q=85, sub=2):
    from PIL import Image
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    img = np.stack([128 + 70 * np.sin(xx / (9.0 + c) + yy / (17.0 - c) + seed) for c in range(3)], -1)
    img += rng.normal(0, 18, (h, w, 3))
    b = io.BytesIO()
    Image.fromarray(np.clip(img, 0, 255).astype(np.uint8), "RGB").save(b, "JPEG", quality=q, subsampling=sub)
    return b.getvalue()


def check_equal(a, b, name):
    assert a["status"] == b["status"], name
    assert (a["padbit"], a["end_bitpos"], a["nrows"]) == (b["padbit"], b["end_bitpos"], b["nrows"]), name
    assert a["rows"] == b["rows"], name
    for pa, pb in zip(a["planes"], b["planes"]):
        assert np.array_equal(pa, pb), name


@pytest.mark.parametrize("sub_bits", [256, 1024, 4096])
def test_golden_jpegs_both_kernels_match_the_host_decoder(sub_bits):
    """Both kernels, with the CTAs and threads of every launch in order and in reverse order."""
    jpegs = [open(os.path.join(GOLDEN, n), "rb").read() for n in GOLDEN_JPEGS]
    for reverse in (False, True):
        ser, _ = emu.huffman_decode(emu.HUFF_SERIAL, jpegs, reverse=reverse)
        par, (iters, redo) = emu.huffman_decode(emu.HUFF_SUBSEQ, jpegs, sub_bits=sub_bits, reverse=reverse)
        taken = 0
        for n, s, p in zip(GOLDEN_JPEGS, ser, par):
            assert (s is None) == (p is None), n
            if s is None:
                continue
            taken += 1
            assert s["status"] == 0, n
            for got, want in zip(s["planes"], s["host_planes"]):
                assert np.array_equal(got, want), n
            check_equal(p, s, n)
        assert taken >= 6 and iters >= 2 and redo == 0


@pytest.mark.parametrize("w,h,q,sub", [(640, 480, 85, 2), (333, 211, 95, 0), (1024, 96, 60, 1), (64, 64, 85, 2), (1920, 1080, 85, 2)])
def test_synthetic_jpegs_subsequence_kernels(w, h, q, sub):
    jpegs = [pil_jpeg(7 * k + w, w, h, q, sub) for k in range(3)]
    ser, _ = emu.huffman_decode(emu.HUFF_SERIAL, jpegs)
    for bits in (512, 4096):
        par, (iters, redo) = emu.huffman_decode(emu.HUFF_SUBSEQ, jpegs, sub_bits=bits)
        for k, (s, p) in enumerate(zip(ser, par)):
            assert s is not None and s["status"] == 0
            for got, want in zip(s["planes"], s["host_planes"]):
                assert np.array_equal(got, want)
            check_equal(p, s, "image %d, %d-bit sub-sequences" % (k, bits))
        assert redo == 0


def test_damaged_scans_fall_back_to_the_serial_walk():
    """Bit flips, a cut-off tail and appended junk: whatever the sub-sequence kernels meet, the outcome (status and, for
    status 0, every output) is the serial kernel's, under both schedules.  The short-scan corpus rides along untouched
    (complete files whose scan is short, damaged or oddly padded, tests/golden/make_shortscan.py): the serial kernel's
    status is the host decoder's, or "not handled" (200) where the data ends inside a block or a zero run passes the end
    of one -- the file API gives those to the host decoder."""
    from helpers import SHORTSCAN, shortscan_jpegs
    short = [n for n in shortscan_jpegs() if SHORTSCAN[n]["path"].startswith("shortscan/")]
    jpegs = [pil_jpeg(100 + k, 320, 240) for k in range(6)] + [open(os.path.join(GOLDEN, SHORTSCAN[n]["path"]), "rb").read() for n in short]

    def mutate(i, buf):
        if i == 1:
            buf[len(buf) // 2] ^= 0x5a
        elif i == 2:
            del buf[len(buf) * 2 // 3:]
        elif i == 3:
            buf.extend(b"\x12\x34\x56\x78" * 40)
        elif i == 4:
            for k in range(50, len(buf), 97):
                buf[k] ^= 1 << (k % 8)
        elif i == 5:
            buf[-1] ^= 0x01
    ser, _ = emu.huffman_decode(emu.HUFF_SERIAL, jpegs, mutate=mutate)
    assert ser[0]["status"] == 0
    assert any(s["status"] != 0 for s in ser[1:6])
    for n, s in zip(short, ser[6:]):
        assert s["status"] in (s["host_status"], 200), (n, s["status"], s["host_status"])
    assert {s["status"] for s in ser[6:]} == {0, 42, 200}
    for reverse in (False, True):
        par, (iters, redo) = emu.huffman_decode(emu.HUFF_SUBSEQ, jpegs, sub_bits=1024, mutate=mutate, reverse=reverse)
        for k, (s, p) in enumerate(zip(ser, par)):
            assert p["status"] == s["status"], (k, reverse)
            if s["status"] == 0:
                check_equal(p, s, "image %d, reverse %s" % (k, reverse))
        assert redo >= 1


def test_no_convergence_within_the_budget_is_handed_to_the_serial_kernel():
    jpegs = [pil_jpeg(5, 640, 480)]
    ser, _ = emu.huffman_decode(emu.HUFF_SERIAL, jpegs)
    for reverse in (False, True):
        par, (iters, redo) = emu.huffman_decode(emu.HUFF_SUBSEQ, jpegs, sub_bits=256, iter_cap=1, reverse=reverse)
        assert redo == 1
        check_equal(par[0], ser[0], "iteration budget 1, reverse %s" % reverse)


# ---- the way back: lep_huffencode_kernel (one warp per thread-segment) on the emulator
HENC_FILES = ["android.jpg", "androidcrop.jpg", "androidcropoptions.jpg", "androidtrail.jpg", "grayscale.jpg", "iphonecrop2.jpg",
              "trailingrst.jpg", "trailingrst2.jpg"]


@pytest.mark.parametrize("name", HENC_FILES)
def test_huffman_encode_kernel_recreates_the_original_scan(name):
    """Planes of the JPEG (host Huffman decoder, pinned against the reference's -ujg dump) + the job the product builds from the
    reference-written .lep (tables, per-segment MCU rows, DC predictors, pending bits, byte counts of the ThreadHandoffs)
    -> lep_huffencode_kernel on the emulator -> exactly the entropy-coded bytes of the original file's scan, every segment
    reporting the byte count its handoff promises (recode_row_range, src/lepton/recoder.cc:472-545; restart markers and
    0xFF stuffing included)."""
    from lepton_b200 import HostJpeg, HostLep
    jpg = open(os.path.join(GOLDEN, name), "rb").read()
    hl = HostLep(open(os.path.join(GOLDEN, name[:-4] + ".lep"), "rb").read())
    assert hl.status == 0, hl.error
    off, n = hl.scan_layout()
    assert n > 0
    job = emu.henc_job(hl)
    assert job.scan_bytes == n
    img = HostJpeg(jpg).coef_image()
    scan, segs = emu.huffman_encode(job, img)
    assert [st for st, _ in segs] == [0] * job.nseg, segs
    assert scan == jpg[off:off + n]
    assert hl.assemble(scan) == jpg


def test_huffman_encode_kernel_multi_segment_reference_files():
    """Reference-written .lep files with 2 / 4 / 8 thread-segments (-minencodethreads): every segment starts from its own
    handoff (bits pending in its first byte, DC predictors) and the pieces meet byte for byte."""
    from helpers import MANIFEST
    from lepton_b200 import HostJpeg, HostLep
    for lep_name in ["androidcrop_t2.lep", "android_t4.lep", "iphonecrop2_t8.lep"]:
        jpg = open(os.path.join(GOLDEN, MANIFEST[lep_name]["source"]), "rb").read()
        hl = HostLep(open(os.path.join(GOLDEN, lep_name), "rb").read())
        assert hl.status == 0, hl.error
        off, n = hl.scan_layout()
        job = emu.henc_job(hl)
        assert n > 0 and job.nseg == int(lep_name.split("_t")[1].split(".")[0])
        scan, segs = emu.huffman_encode(job, HostJpeg(jpg).coef_image())
        assert [st for st, _ in segs] == [0] * job.nseg, (lep_name, segs)
        assert scan == jpg[off:off + n], lep_name


# ---- the extreme corpus: Huffman codes up to 16 bits, category-11 magnitudes, runs of stuffed 0xFF bytes
@pytest.mark.parametrize("sub_bits", [256, 1024, 4096])
def test_extreme_jpegs_both_kernels_match_the_host_decoder(sub_bits):
    """Serial and sub-sequence kernels give the host decoder's planes (pinned to the reference's -ujg dumps) and agree on
    every row state.  The colour files are large enough that the sub-sequence kernels take them."""
    from helpers import EXTREMES, extreme_jpegs, read_golden
    names = extreme_jpegs()
    jpegs = [read_golden(EXTREMES[n]["path"]) for n in names]
    ser, _ = emu.huffman_decode(emu.HUFF_SERIAL, jpegs)
    par, (iters, redo) = emu.huffman_decode(emu.HUFF_SUBSEQ, jpegs, sub_bits=sub_bits)
    for n, s, p in zip(names, ser, par):
        assert (s is None) == (p is None), n
        if s is None:
            assert not n.startswith("color"), n
            continue
        assert s["status"] == 0, n
        for got, want in zip(s["planes"], s["host_planes"]):
            assert np.array_equal(got, want), n
        check_equal(p, s, n)
    assert all(ser[names.index(n)] is not None for n in ("color420_long.jpg", "color444_long.jpg", "odd_rst.jpg"))
    assert iters > 0
    # with 256-bit sub-sequences, 16-bit codes resynchronise too slowly for some of these files: the serial kernel redoes
    # them (same outputs, checked above)
    assert redo == 0 or sub_bits == 256


def test_huffman_encode_kernel_recreates_the_extreme_scans():
    """lep_huffencode_kernel re-creates the scan of every extreme file byte for byte from the reference's .lep records:
    16-bit codes, 0xFF stuffing, restart markers, and 4 and 8 segments whose handoffs carry extreme DC predictors."""
    from helpers import EXTREMES, extreme_leps, read_golden
    from lepton_b200 import HostJpeg, HostLep
    multi = 0
    for name, source in extreme_leps():
        jpg = read_golden(EXTREMES[source]["path"])
        hl = HostLep(read_golden("extremes/" + name))
        assert hl.status == 0, hl.error
        off, n = hl.scan_layout()
        job = emu.henc_job(hl)
        assert n > 0 and job.scan_bytes == n
        img = HostJpeg(jpg).coef_image()
        scan, segs = emu.huffman_encode(job, img)
        assert [st for st, _ in segs] == [0] * job.nseg, (name, segs)
        assert scan == jpg[off:off + n], name
        assert hl.assemble(scan) == jpg, name
        multi += job.nseg > 1
    assert multi >= 5
