"""The JPEG-side kernels on the device, at the inputs built to break them: lep_huffdecode_kernel (lep_huff.cu), the
sub-sequence kernels of lep_huffpar.cu and lep_huffencode_kernel (lep_huffenc.cu).

The emulator suite (tests/test_emu_huffman.py) runs these kernels with one CTA after the other.  Here they run through
the library's own launch code on the GPU: the host-driven synchronisation iterations of the sub-sequence kernels and
their hand-off to the serial kernel, the in-place and pre-uploaded staging of the scans (and the 16 zero bytes the
decoder reads past each one), several images per CTA with placeholder scans between them, and the re-encode in parts
with its per-part Adler-32.

Expected values never come from the kernels:
  status, planes      the host decoder (HostJpeg, pinned to the reference's -ujg dumps) and the reference's fixtures
  pad bit, end and    walk_scan() below, a plain Huffman walker over the de-stuffed bytes lepb200_host_jpeg_scan hands
  row states          out (the reader twin of jpegwriter.BitWriter)
  decision counts     the oracle (oracle_encode_image)
  scan bytes          the original file (HostLep.scan_layout) and zlib.adler32
The device plane arena has no read-back, so the decoded planes are checked the way the product uses them: uploaded for
the encoder with lepb200_encode_upload_resident, token bounds set from the returned rows as lep_file.cc does, and coded;
the streams and decision counts must be the oracle's for the host planes.
"""
import ctypes
import functools
import hashlib
import os
import sys
import zlib

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu  # noqa: E402
from emu import _HEncImage, _HuffRow, _Scan  # noqa: E402
from helpers import (DENSE, EXTREMES, SHORTSCAN, SHORTSCAN_REFUSED, dense_leps, extreme_jpegs, extreme_leps,  # noqa: E402
                     oracle_encode_image, random_coef_image, read_golden, shortscan_jpegs, shortscan_lep, shortscan_status)
from jpegwriter import write_baseline  # noqa: E402

pytestmark = pytest.mark.gpu

TUNING = ("LEPB200_HUFF_PAR", "LEPB200_HUFF_SUBSEQ_BITS", "LEPB200_HUFF_WARPS")
ST_OUT_OVERFLOW = 100
NOT_HANDLED = 200


def md5(b):
    return hashlib.md5(b).hexdigest()


@functools.lru_cache(None)
def L():
    import lepton_b200
    lib = lepton_b200.lib()
    vp, i = ctypes.c_void_p, ctypes.c_int
    sig = {"lepb200_huffman_decode_to_device": ([vp, ctypes.POINTER(_Scan), i], i),
           "lepb200_huffman_stage_reserve": ([vp, ctypes.c_size_t], ctypes.POINTER(ctypes.c_uint8)),
           "lepb200_huffman_stage_upload": ([vp, ctypes.c_size_t, ctypes.c_size_t], i),
           "lepb200_encode_upload_resident": ([vp, vp, i], i),
           "lepb200_last_huffman_iterations": ([vp], i), "lepb200_last_huffman_redone": ([vp], i),
           "lepb200_host_jpeg_scan": ([vp, ctypes.POINTER(_Scan)], i),
           "lepb200_huffman_encode_resident": ([vp, ctypes.POINTER(_HEncImage), i], i),
           "lepb200_huffman_encode_resident_parts": ([vp, ctypes.POINTER(_HEncImage), i, i], i),
           "lepb200_huffman_encode_parts": ([vp], i),
           "lepb200_huffman_encode_wait_part": ([vp, ctypes.POINTER(_HEncImage), i, i, ctypes.POINTER(i), ctypes.POINTER(i)], i),
           "lepb200_huffman_encode_fetch": ([vp, ctypes.POINTER(_HEncImage), i], i),
           "lepb200_huffman_encode_adler32": ([vp, i, i, ctypes.POINTER(ctypes.c_uint32)], i)}
    for name, (args, res) in sig.items():
        f = getattr(lib, name)
        f.argtypes, f.restype = args, res
    return lib


def codec_with(monkeypatch, env):
    """A context created under `env` and no other Huffman tuning variable (the library reads them at creation)."""
    from lepton_b200 import LeptonB200Codec
    for k in TUNING:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, str(v))
    return LeptonB200Codec(0)


# ------------------------------------------------------------------------------------------ plain Huffman walker
def _decode_map(t):
    """_HuffTable -> {(length, code): symbol}"""
    out, code, k = {}, 0, 0
    for ln in range(1, 17):
        for _ in range(t.bits[ln]):
            out[(ln, code)] = t.vals[k]
            k += 1
            code += 1
        code <<= 1
    return out


def walk_scan(sc, data):
    """The baseline scan decode the kernels implement, one bit at a time over the de-stuffed bytes (zeros past the end):
    -> dict(status, padbit, end_bitpos, rows [(bitpos, lastdc, mcu_y)]).  status 0, 42 (bad code, EOB after a zero,
    inconsistent padding, data left over) or 200 (a zero run past the end of a block, data that ends inside a block)."""
    bits = "".join("{:08b}".format(b) for b in data)
    total = len(bits)
    pos = 0

    def bit(p):
        return 1 if p < total and bits[p] == "1" else 0

    def read(n):
        nonlocal pos
        v = 0
        for _ in range(n):
            v = (v << 1) | bit(pos)
            pos += 1
        return v

    def symbol(m):
        code = 0
        for ln in range(1, 17):
            code = (code << 1) | read(1)
            if (ln, code) in m:
                return m[(ln, code)]
        return None

    ncmp, mcuh, mcuv, rsti = sc.ncmp, sc.mcuh, sc.mcuv, sc.rsti
    dcm = [_decode_map(sc.dc[c]) for c in range(ncmp)]
    acm = [_decode_map(sc.ac[c]) for c in range(ncmp)]
    H, V = list(sc.H), list(sc.V)
    if ncmp > 1:
        order = [(c, my) for my in range(mcuv) for mx in range(mcuh) for c in range(ncmp) for _ in range(H[c] * V[c])]
        per_unit = sum(H[c] * V[c] for c in range(ncmp))
        rows_at = {u * per_unit for u in range(0, mcuv * mcuh, mcuh)}
    else:
        nch, ncv = sc.nch[0], sc.ncv[0]
        bch = mcuh * H[0]
        order = []
        for by in range(ncv):
            for bx in range(nch):
                order.append((0, (by * bch + bx) // (H[0] * V[0]) // mcuh))
        per_unit = 1
        rows_at = {k for k in range(len(order)) if ((k // nch) * bch + k % nch) % (H[0] * V[0]) == 0
                   and (((k // nch) * bch + k % nch) // (H[0] * V[0])) % mcuh == 0}
    rows, dc, padbit, final_y = [], [0, 0, 0], -1, mcuv

    def res(status):
        return dict(status=status, padbit=padbit, end_bitpos=pos, rows=rows)
    rows.append((0, (0, 0, 0), 0))
    nunits_blocks = len(order)
    unit_blocks = per_unit if ncmp > 1 else 1
    for k, (c, my) in enumerate(order):
        s = symbol(dcm[c])
        if s is None or s > 16:
            return res(42)
        v = read(s)
        dc[c] = (dc[c] + (v if s == 0 or v >= 1 << (s - 1) else v + 1 - (1 << s)) + 32768) % 65536 - 32768
        bpos, last_nz = 1, True
        while bpos < 64:
            s = symbol(acm[c])
            if s is None:
                return res(42)
            if s == 0:
                if bpos > 1 and not last_nz:
                    return res(42)
                break
            r, z = s >> 4, s & 15
            if r + bpos >= 64:
                return res(NOT_HANDLED)
            read(z)
            bpos += r + 1
            last_nz = z != 0
        if pos > total:
            return res(NOT_HANDLED)
        sta = 0
        if k + 1 == nunits_blocks:
            sta = 2
        elif rsti and (k + 1) % (unit_blocks * rsti) == 0:
            sta = 1
        if pos >= total:
            sta = 2
        if sta:
            fb = padbit
            if pos % 8 and pos < total:
                last = bit(pos)
                pos += 1
                fb, off = last, 1
                while pos % 8:
                    last = bit(pos)
                    pos += 1
                    fb |= last << off
                    off += 1
                while off < 7:
                    fb |= last << off
                    off += 1
            if padbit != -1 and padbit != fb:
                return res(42)
            padbit = fb
            if sta == 2:
                final_y = order[k + 1][1] if k + 1 < nunits_blocks else mcuv       # the data may end before the last row
                break
            dc = [0, 0, 0]
        if k + 1 in rows_at:
            rows.append((pos, tuple(dc), order[k + 1][1]))
    rows.append((pos, tuple(dc), final_y))
    return res(0 if pos >= total else 42)


# ------------------------------------------------------------------------------------------ device decode + check
class Scans:
    """Host scans of JPEG files (lepb200_host_jpeg_scan), with their de-stuffed bytes held here so that they can be cut,
    extended or moved into the staging buffer.  edit(i, bytes) -> the bytes file i is decoded from."""

    def __init__(self, jpegs, edit=None):
        from lepton_b200 import HostJpeg
        self.hjs, self.scans, self.data = [], [], []
        for i, jpg in enumerate(jpegs):
            hj = HostJpeg(jpg)
            sc = _Scan()
            assert L().lepb200_host_jpeg_scan(hj._h, ctypes.byref(sc)) == 0, i
            d = ctypes.string_at(sc.entropy, sc.nbytes)
            if edit is not None:
                d = edit(i, d)
            self.hjs.append(hj)
            self.scans.append(sc)
            self.data.append(d)


def device_decode(codec, scans, placeholders=(), stage="gather"):
    """lepb200_huffman_decode_to_device over a Scans batch -> (per image dict(status, padbit, end_bitpos, nrows, rows) or None
    for a placeholder, iterations, images redone).  stage: gather (scans in the caller's buffers), inplace (inside the
    pinned staging buffer, 16-byte aligned, 16 zero bytes behind each) or upload (the same, pushed by stage_upload)."""
    n = len(scans.scans)
    arr = (_Scan * n)()
    keep = []
    offs, tot = [], 0
    for k, d in enumerate(scans.data):
        offs.append(tot)
        tot += (len(d) + 32 + 15) & ~15
    base = L().lepb200_huffman_stage_reserve(codec._ctx, tot) if stage != "gather" else None
    for k, (sc, d) in enumerate(zip(scans.scans, scans.data)):
        ctypes.memmove(ctypes.byref(arr[k]), ctypes.byref(sc), ctypes.sizeof(_Scan))
        rows = (_HuffRow * (sc.mcuv + 1))()
        keep.append(rows)
        arr[k].rows = ctypes.cast(rows, ctypes.POINTER(_HuffRow))
        if k in placeholders:
            arr[k].entropy, arr[k].nbytes = None, 0
            continue
        if base is None:
            buf = ctypes.create_string_buffer(d, max(1, len(d)))
            keep.append(buf)
            arr[k].entropy = ctypes.addressof(buf)
        else:
            addr = ctypes.addressof(base.contents) + offs[k]
            ctypes.memset(addr, 0x5A, (len(d) + 32 + 15) & ~15)       # whatever lies behind a scan must not be read as data
            ctypes.memmove(addr, d, len(d))
            ctypes.memset(addr + len(d), 0, 16)
            arr[k].entropy = addr
        arr[k].nbytes = len(d)
    if stage == "upload":
        assert L().lepb200_huffman_stage_upload(codec._ctx, 0, tot) == 0
    codec._check(L().lepb200_huffman_decode_to_device(codec._ctx, arr, n), "huffman_decode_to_device")
    out = []
    for k in range(n):
        a = arr[k]
        if k in placeholders:
            out.append(None)
            continue
        rows = [(a.rows[r].bitpos, tuple(a.rows[r].lastdc), a.rows[r].mcu_y, a.rows[r].tokens) for r in range(max(0, min(a.nrows, a.mcuv + 1)))]
        out.append(dict(status=a.status, padbit=a.padbit, end_bitpos=a.end_bitpos, nrows=a.nrows, rows=rows))
    return out, L().lepb200_last_huffman_iterations(codec._ctx), L().lepb200_last_huffman_redone(codec._ctx)


def row_split(img, rows=None):
    """One segment per MCU row the scan reached (the last one takes the rest when there are more than 16 rows)."""
    mul = img.bcv[0] // img.mcuv
    n = img.mcuv if rows is None else max(1, min(img.mcuv, rows[-1][2]))
    return [r * mul for r in range(min(n, 16))]


def token_bounds(rows, starts, mul, mcuv):
    """seg_token_bound of each segment from the row tokens, as lep_file.cc select_segments sets it: none (0, the library
    counts) when the scan ended before its last MCU row, since the rows do not count the blocks past that point."""
    if rows[-1][2] < mcuv:
        return [0] * len(starts)
    r, st = 0, []
    for y in starts:
        while r + 1 < len(rows) and mul * rows[r][2] < y:
            r += 1
        st.append(rows[r][3])
    st.append(rows[-1][3])
    return [max(1, st[t + 1] - st[t]) for t in range(len(starts))]


def encode_resident_and_check(codec, scans, res, placeholders=()):
    """Uploads the batch the last device_decode left resident -- placeholders and images the device did not decode with
    their host planes -- with one segment per MCU row and the token bounds of the returned rows (lep_file.cc), codes it,
    and holds every image with device status 0 and every placeholder to the oracle run over the host planes."""
    from lepton_b200.codec import _Image
    n = len(scans.scans)
    imgs, carr = [], (_Image * n)()
    for k, hj in enumerate(scans.hjs):
        img = hj.coef_image() if hj.status == 0 else None
        if img is None:                                   # planes the host refused: a zero placeholder keeps the layout
            sc = scans.scans[k]
            from lepton_b200 import CoefImage
            bch = [sc.mcuh * sc.H[c] for c in range(sc.ncmp)]
            bcv = [sc.mcuv * sc.V[c] for c in range(sc.ncmp)]
            img = CoefImage(ncmp=sc.ncmp, mcuv=sc.mcuv, bch=bch, bcv=bcv, qtables_zigzag=[[1] * 64] * sc.ncmp,
                            planes=[np.zeros((bch[c] * bcv[c], 64), np.int16) for c in range(sc.ncmp)])
        r = res[k]
        dev = r is not None and r["status"] == 0
        img.luma_y_start = row_split(img, r["rows"] if dev else None)
        img.trunc_bcv = img.trunc_bc = None
        imgs.append(img)
        carr[k] = img.to_c()
        if dev:
            for c in range(img.ncmp):
                carr[k].planes[c] = None                  # resident: the device-decoded planes
            for t, b in enumerate(token_bounds(r["rows"], img.luma_y_start, img.bcv[0] // img.mcuv, img.mcuv)):
                carr[k].seg_token_bound[t] = b
    codec._check(L().lepb200_encode_upload_resident(codec._ctx, carr, n), "encode_upload_resident")
    codec._enc_imgs = imgs
    codec.encode_launch()
    got = codec.encode_fetch()
    checked = 0
    for k, img in enumerate(imgs):
        r = res[k]
        if not (k in placeholders or (r is not None and r["status"] == 0)) or scans.hjs[k].status != 0:
            continue
        want = oracle_encode_image(img)
        assert [g.status for g in got[k]] == [w[0] for w in want], (k, [g.status for g in got[k]])
        assert all(g.status != ST_OUT_OVERFLOW for g in got[k]), k
        assert [g.data for g in got[k]] == [w[1] for w in want], "image %d: streams differ from the oracle's for the host planes" % k
        assert [g.ndecisions for g in got[k]] == [w[2] for w in want], k
        if r is not None:
            for t, b in enumerate(token_bounds(r["rows"], img.luma_y_start, img.bcv[0] // img.mcuv, img.mcuv)):
                assert b == 0 or b >= want[t][2], ("token bound below the oracle's decision count", k, t, b, want[t][2])
        checked += 1
    return checked


def check_rows_against_walker(scans, res):
    for k, r in enumerate(res):
        if r is None or r["status"] != 0:
            continue
        w = walk_scan(scans.scans[k], scans.data[k])
        assert w["status"] == 0, k
        assert (r["padbit"], r["end_bitpos"]) == (w["padbit"], w["end_bitpos"]), k
        assert [row[:3] for row in r["rows"]] == w["rows"], k
        assert r["nrows"] == len(w["rows"]), k


def same_outputs(a, b, what):
    for k, (x, y) in enumerate(zip(a, b)):
        if x is None or y is None:
            assert x is y, (what, k)
            continue
        assert x["status"] == y["status"], (what, k, x["status"], y["status"])
        if x["status"] == 0:
            assert x == y, (what, k)


def device_takes(jpg):
    """Whether the file API hands this file to the device Huffman decoder (one baseline scan in frame order)."""
    from lepton_b200 import HostJpeg
    hj = HostJpeg(jpg)
    return L().lepb200_host_jpeg_scan(hj._h, ctypes.byref(_Scan())) == 0


# zig-zag index -> AlignedBlock index (lep_huff.cu c_zigzag_to_aligned)
ZZ_TO_ALIGNED = [49, 50, 57, 58, 0, 51, 52, 1, 2, 59, 60, 3, 4, 5, 53, 54, 6, 7, 8, 9, 61, 62, 10, 11, 12, 13, 14, 55, 56, 15,
                 16, 17, 18, 19, 20, 63, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32, 33, 34, 35, 36, 37, 38, 39, 40, 41,
                 42, 43, 44, 45, 46, 47, 48]


def jpeg_of(img):
    """A baseline JPEG (tests/jpegwriter.py) whose scan codes exactly the planes of a helpers.random_coef_image image."""
    if img.ncmp == 1:
        sampling, mcuh = [(1, 1)], img.bch[0]
    else:
        mcuh = img.bch[1]                                # chroma is 1x1 in every geometry used here
        sampling = [(img.bch[c] // mcuh, img.bcv[c] // img.mcuv) for c in range(img.ncmp)]
    hmax, vmax = max(h for h, _ in sampling), max(v for _, v in sampling)
    planes = []
    for c in range(img.ncmp):
        p = np.asarray(img.planes[c], np.int64)[:, ZZ_TO_ALIGNED]
        p[:, 1:] = np.clip(p[:, 1:], -1023, 1023)
        planes.append(p.reshape(img.bcv[c], img.bch[c], 64))
    q = [list(img.qtables_zigzag[c]) for c in range(img.ncmp)]
    qbits = 16 if max(max(t) for t in q) > 255 else 8
    return write_baseline(planes, mcuh * 8 * hmax, img.mcuv * 8 * vmax, sampling, q, qbits=qbits)


def scan_bytes(jpg):
    """Length of the de-stuffed scan the device decoder gets for this file."""
    from lepton_b200 import HostJpeg
    hj, sc = HostJpeg(jpg), _Scan()
    assert L().lepb200_host_jpeg_scan(hj._h, ctypes.byref(sc)) == 0
    return sc.nbytes


def shortscan_device():
    """(names, files) of the short-scan corpus the device Huffman decoder takes."""
    names = [n for n in shortscan_jpegs() if device_takes(read_golden(SHORTSCAN[n]["path"]))]
    return names, [read_golden(SHORTSCAN[n]["path"]) for n in names]


# ---------------------------------------------------------------------------------------------------- decode kernels
@pytest.mark.timeout(600, method="thread")
@pytest.mark.parametrize("par", [0, 1])
def test_short_and_damaged_scans_decode_like_the_host(monkeypatch, par):
    """The short-scan corpus: the device's status is the host decoder's, or "not handled" (200) where the host goes on past
    the end of the data or refuses a zero run past the end of a block; rows match the walker and planes the host's."""
    names, files = shortscan_device()
    scans = Scans(files)
    codec = codec_with(monkeypatch, {"LEPB200_HUFF_PAR": par, "LEPB200_HUFF_SUBSEQ_BITS": 256})
    res, _, _ = device_decode(codec, scans)
    ok = 0
    for n, hj, r in zip(names, scans.hjs, res):
        assert r["status"] in (hj.status, NOT_HANDLED), (n, r["status"], hj.status)
        if r["status"] == NOT_HANDLED:
            assert walk_scan(scans.scans[names.index(n)], scans.data[names.index(n)])["status"] == NOT_HANDLED, n
        ok += r["status"] == 0
    assert ok >= 10 and any(r["status"] == NOT_HANDLED for r in res)
    check_rows_against_walker(scans, res)
    assert encode_resident_and_check(codec, scans, res) >= ok
    codec.close()


@pytest.mark.timeout(600, method="thread")
def test_token_bounds_hold_one_mcu_row_per_segment(monkeypatch):
    """Every MCU row its own segment (up to 16): the difference of consecutive row tokens must cover the oracle's
    decision count of that row, on the extreme and dense corpora (16-bit codes, category-11 magnitudes, noise) and on
    random planes in the coder tests' geometries (helpers.random_coef_image, written by tests/jpegwriter.py)."""
    names = [n for n in extreme_jpegs() if EXTREMES[n]["status_want"] == 0] + [s for _, s in dense_leps()]
    names = sorted(set(names), key=names.index)
    files = [read_golden(EXTREMES[n]["path"] if n in EXTREMES else DENSE[n]["path"]) for n in names]
    keep = [f for f in files if device_takes(f)]
    # and random planes in the coder tests' geometries, up to 20 MCU rows
    rng = np.random.default_rng(90)
    for sf, mcuh, mcuv in [(((2, 2), (1, 1), (1, 1)), 5, 4), (((2, 1), (1, 1), (1, 1)), 3, 9), (((1, 1),) * 3, 4, 17),
                           (((1, 2), (1, 1), (1, 1)), 2, 6), (((1, 1),), 7, 20), (((2, 2), (1, 1), (1, 1)), 1, 16)]:
        keep.append(jpeg_of(random_coef_image(rng, ncmp=len(sf), mcuh=mcuh, mcuv=mcuv, sf=sf, density=0.4)))
    scans = Scans(keep)
    codec = codec_with(monkeypatch, {})
    res, _, _ = device_decode(codec, scans)
    assert all(r["status"] == 0 for r in res)
    check_rows_against_walker(scans, res)
    assert encode_resident_and_check(codec, scans, res) == len(keep) >= 12
    codec.close()


def _cut_to(d, n):
    return d[:n] if len(d) >= n else d + bytes(n - len(d))


@pytest.mark.timeout(600, method="thread")
@pytest.mark.parametrize("bits", [256, 512, 2048, 4096, 16384])
def test_subsequence_kernels_match_the_serial_kernel(monkeypatch, bits):
    """LEPB200_HUFF_PAR=1 against =0: scans shorter than one sub-sequence, scans cut or zero-extended to exactly k
    sub-sequences and one byte either side, the 16-bit-code extreme files, and colour files with restart intervals (which
    the serial kernel takes).  Every output must be the serial run's, and the walker's where the status is 0."""
    ej = extreme_jpegs
    sub = bits // 8
    long_names = [n for n in ej() if "long" in n and EXTREMES[n]["status_want"] == 0]
    base = [read_golden(EXTREMES[n]["path"]) for n in long_names]
    big = max(base, key=len)
    jpegs, edits = [], []
    for j in shortscan_device()[1][:12]:
        jpegs.append(j)
        edits.append(None)
    for k in (1, 2, 3):
        for dlt in (-1, 0, 1):
            jpegs.append(big)
            edits.append(k * sub + dlt)
    jpegs += base
    edits += [None] * len(base)
    rst = [read_golden(EXTREMES[n]["path"]) for n in ej() if "rst" in n and EXTREMES[n]["status_want"] == 0]
    jpegs += rst
    edits += [None] * len(rst)
    scans = Scans(jpegs, edit=lambda i, d: d if edits[i] is None else _cut_to(d, edits[i]))
    ser_c = codec_with(monkeypatch, {"LEPB200_HUFF_PAR": 0})
    ser, it0, _ = device_decode(ser_c, scans)
    assert it0 == 0
    ser_c.close()
    par_c = codec_with(monkeypatch, {"LEPB200_HUFF_PAR": 1, "LEPB200_HUFF_SUBSEQ_BITS": bits})
    par, iters, redone = device_decode(par_c, scans)
    same_outputs(par, ser, "%d-bit sub-sequences" % bits)
    check_rows_against_walker(scans, par)
    assert [r["status"] for r in par] == [walk_scan(sc, d)["status"] for sc, d in zip(scans.scans, scans.data)]
    assert iters >= 3
    if bits == 256:
        assert redone >= 1
    encode_resident_and_check(par_c, scans, par)
    par_c.close()


@pytest.mark.timeout(600, method="thread")
@pytest.mark.parametrize("warps", [1, 3, 8])
def test_launch_shapes_with_placeholders(monkeypatch, warps):
    """LEPB200_HUFF_WARPS images per CTA, batches of every size residue, placeholder scans (plane slot only) between real
    ones: the placeholders' slots hold exactly the host planes given to encode_upload_resident, the neighbours their own."""
    files = [read_golden(SHORTSCAN[n]["path"]) for n in shortscan_jpegs() if SHORTSCAN[n]["status_want"] == 0 and n.endswith("_full.jpg")]
    for n in range(warps, 2 * warps + 1):
        jpegs = [files[k % len(files)] for k in range(n)]
        scans = Scans(jpegs)
        ph = set(range(1, n, 3))
        codec = codec_with(monkeypatch, {"LEPB200_HUFF_WARPS": warps, "LEPB200_HUFF_PAR": 0})
        res, _, _ = device_decode(codec, scans, placeholders=ph)
        assert all(r["status"] == 0 for r in res if r is not None)
        check_rows_against_walker(scans, res)
        assert encode_resident_and_check(codec, scans, res, placeholders=ph) == n
        codec.close()


@pytest.mark.timeout(600, method="thread")
def test_staging_gather_inplace_and_upload_agree(monkeypatch):
    """The same batch with its scans in the caller's buffers, inside the pinned staging buffer, and pushed by
    stage_upload, at de-stuffed lengths of every residue mod 16: identical outputs (every image decodes with status 0,
    so rows, pad bit and end position are compared too), and the oracle's planes."""
    rng, by_res = np.random.default_rng(16), {}
    while len(by_res) < 16:
        sf = [((2, 2), (1, 1), (1, 1)), ((1, 1),)][len(by_res) % 2]
        img = random_coef_image(rng, ncmp=len(sf), mcuh=int(rng.integers(1, 4)), mcuv=int(rng.integers(1, 4)), sf=sf)
        j = jpeg_of(img)
        by_res.setdefault(scan_bytes(j) % 16, j)
    scans = Scans([by_res[r] for r in range(16)])
    outs = []
    for stage in ("gather", "inplace", "upload"):
        codec = codec_with(monkeypatch, {})
        res, _, _ = device_decode(codec, scans, stage=stage)
        outs.append(res)
        check_rows_against_walker(scans, res)
        encode_resident_and_check(codec, scans, res)
        codec.close()
    assert all(r["status"] == 0 for res in outs for r in res)
    assert outs[1] == outs[0] and outs[2] == outs[0]


# ---------------------------------------------------------------------------------------------------- re-encode kernel
MULTI = ["androidcrop_t2.lep", "android_t4.lep", "iphonecrop2_t8.lep", "trailingrst2.lep"]


def reencode_batch():
    """(lep bytes, source JPEG bytes) of the multi-segment reference files, with None between them (skipped images)."""
    from helpers import MANIFEST
    out = []
    for n in MULTI:
        src = MANIFEST[n]["source"] if n in MANIFEST else n[:-4] + ".jpg"
        out.append((read_golden(n), read_golden(src)))
    for name, source in extreme_leps():
        if "_t" in name or "odd_rst_t4" in name:
            out.append((read_golden("extremes/" + name), read_golden(EXTREMES[source]["path"])))
    for name, source in dense_leps():
        if "_t" in name:
            out.append((read_golden("dense/" + name), read_golden(DENSE[source]["path"])))
    from lepton_b200 import HostLep
    out = [item for item in out if HostLep(item[0]).scan_layout()[1] > 0]     # the device re-encodes these
    batch = []
    for k, item in enumerate(out):
        batch.append(item)
        if k % 3 == 1:
            batch.append(None)
    return batch


def device_reencode_setup(codec, batch):
    """decode_upload + decode_launch of the reference streams, and the re-encode jobs (a skipped image has scan_bytes 0
    and the planes of the image next to it)."""
    from lepton_b200 import HostLep
    imgs, streams, jobs, want = [], [], (_HEncImage * len(batch))(), []
    for k, item in enumerate(batch):
        lep, jpg = item if item is not None else batch[k - 1]
        hl = HostLep(lep)
        assert hl.status == 0, hl.error
        img = hl.coef_image()
        imgs.append(img)
        streams.append(hl.streams(img.nseg))
        if item is None:
            jobs[k].scan_bytes = 0
            want.append(None)
            continue
        jobs[k] = emu.henc_job(hl)
        off, n = hl.scan_layout()
        assert n > 0 and jobs[k].scan_bytes == n
        want.append(jpg[off:off + n])
    codec.decode_upload(imgs, streams)
    codec.decode_launch()
    return jobs, want


def scans_of(jobs, k):
    return ctypes.string_at(jobs[k].data, jobs[k].scan_bytes) if jobs[k].scan_bytes else None


@pytest.mark.timeout(600, method="thread")
def test_reencode_batch_scan_bytes_status_and_adler32(monkeypatch):
    batch = reencode_batch()
    assert sum(b is None for b in batch) >= 3 and len(batch) >= 10
    codec = codec_with(monkeypatch, {})
    jobs, want = device_reencode_setup(codec, batch)
    n = len(batch)
    codec._check(L().lepb200_huffman_encode_resident(codec._ctx, jobs, n), "huffman_encode_resident")
    codec._check(L().lepb200_huffman_encode_fetch(codec._ctx, jobs, n), "huffman_encode_fetch")
    ad = (ctypes.c_uint32 * n)()
    assert L().lepb200_huffman_encode_adler32(codec._ctx, 0, n, ad) == 0
    for k in range(n):
        if want[k] is None:
            assert ad[k] == 1, k
            continue
        assert jobs[k].status == 0, k
        assert scans_of(jobs, k) == want[k], k
        assert ad[k] == zlib.adler32(want[k]), k
    codec.close()


@pytest.mark.timeout(600, method="thread")
def test_reencode_in_parts(monkeypatch):
    batch = reencode_batch()
    n = len(batch)
    codec = codec_with(monkeypatch, {})
    for nparts in sorted({1, 2, 3, 7, n, n + 3}):
        jobs, want = device_reencode_setup(codec, batch)
        codec._check(L().lepb200_huffman_encode_resident_parts(codec._ctx, jobs, n, nparts), "huffman_encode_resident_parts")
        np_ = L().lepb200_huffman_encode_parts(codec._ctx)
        assert 1 <= np_ <= min(nparts, 16)
        cover, ad = 0, (ctypes.c_uint32 * n)()
        for p in range(np_):
            a, b = ctypes.c_int(), ctypes.c_int()
            assert L().lepb200_huffman_encode_wait_part(codec._ctx, jobs, n, p, ctypes.byref(a), ctypes.byref(b)) == 0
            assert a.value == cover and b.value >= a.value, (nparts, p)
            cover = b.value
            assert L().lepb200_huffman_encode_adler32(codec._ctx, a.value, b.value, ad) == 0
        assert cover == n, nparts
        parts = [scans_of(jobs, k) for k in range(n)]
        for k in range(n):
            if want[k] is None:
                assert ad[k] == 1
                continue
            assert jobs[k].status == 0 and parts[k] == want[k], (nparts, k)
            assert ad[k] == zlib.adler32(want[k]), (nparts, k)
        # the same batch fetched whole gives the same bytes
        jobs2, _ = device_reencode_setup(codec, batch)
        codec._check(L().lepb200_huffman_encode_resident(codec._ctx, jobs2, n), "huffman_encode_resident")
        codec._check(L().lepb200_huffman_encode_fetch(codec._ctx, jobs2, n), "huffman_encode_fetch")
        assert [scans_of(jobs2, k) for k in range(n)] == parts, nparts
    codec.close()


@pytest.mark.timeout(600, method="thread")
@pytest.mark.parametrize("what", ["bytes+1", "bytes-1", "overhang"])
def test_reencode_bad_handoff_fails_its_image_alone(monkeypatch, what):
    """One segment's handoff wrong -- its expected byte count one off, or its count of pending bits changed so that the
    segment's bits end in another byte -- fails that image alone with status 1; its neighbours are exact."""
    batch = reencode_batch()
    n = len(batch)
    codec = codec_with(monkeypatch, {})
    jobs, want = device_reencode_setup(codec, batch)
    if what != "overhang":
        victim = next(k for k in range(n) if want[k] is not None and jobs[k].nseg >= 4)
        jobs[victim].seg[1].expect_bytes += 1 if what == "bytes+1" else -1
    else:
        # bits of segment t: overhang(t) + coded = 8 * bytes(t) + overhang(t + 1); moving overhang(t) so that the sum
        # crosses a byte border changes the bytes segment t writes
        victim, t = next((k, t) for k in range(n) if want[k] is not None for t in range(jobs[k].nseg - 1)
                         if jobs[k].seg[t].overhang_bits != jobs[k].seg[t + 1].overhang_bits)
        o, o1 = jobs[victim].seg[t].overhang_bits, jobs[victim].seg[t + 1].overhang_bits
        jobs[victim].seg[t].overhang_bits = o + 8 - o1 if o < o1 else o - o1 - 1
    codec._check(L().lepb200_huffman_encode_resident(codec._ctx, jobs, n), "huffman_encode_resident")
    codec._check(L().lepb200_huffman_encode_fetch(codec._ctx, jobs, n), "huffman_encode_fetch")
    for k in range(n):
        if want[k] is None:
            continue
        if k == victim:
            assert jobs[k].status == 1, what
        else:
            assert jobs[k].status == 0 and scans_of(jobs, k) == want[k], (what, k)
    codec.close()


# ---------------------------------------------------------------------------------------------------- file API
@pytest.mark.timeout(600, method="thread")
@pytest.mark.parametrize("gpu_huffman", [True, False])
def test_file_api_short_scans_end_like_the_reference(gpu_huffman):
    """Compress with the device Huffman decoder on and off: the reference's status and .lep for every file of the
    short-scan corpus (the device's "not handled" files go through the host decoder); decompress restores each one."""
    from lepton_b200 import LeptonB200FileCodec
    names = shortscan_jpegs()
    files = [read_golden(SHORTSCAN[n]["path"]) for n in names]
    c = LeptonB200FileCodec(0, gpu_huffman=gpu_huffman)
    got = c.compress(files)
    for n, (st, lep) in zip(names, got):
        assert st == shortscan_status(n), (n, st, shortscan_status(n))
        if st == 0:
            assert md5(lep) == SHORTSCAN[n]["lep_md5"] and lep == shortscan_lep(n), n
    for n in SHORTSCAN_REFUSED:
        assert SHORTSCAN[n]["rc_verify"] == 41 and SHORTSCAN[n]["back_md5"] != SHORTSCAN[n]["jpg_md5"], n
    ok = [(n, lep) for n, (st, lep) in zip(names, got) if st == 0]
    back = c.decompress([lep for _, lep in ok])
    for (n, _), (st, jpg) in zip(ok, back):
        assert st == 0 and md5(jpg) == SHORTSCAN[n]["back_md5"], n
    c.close()


@pytest.mark.timeout(600, method="thread")
def test_file_api_scan_ending_early_among_device_decoded_files(monkeypatch):
    """A complete file whose data ends at a restart border before its last MCU row, batched only with files the device
    decodes: no file of the batch goes to the host decoder, so the encoder runs on the bounds of the Huffman rows, which
    do not count the blocks past the end of the data.  It must still give the reference's .lep."""
    from lepton_b200 import LeptonB200FileCodec
    names = ["c420_rst2_cut_rst.jpg"] + [n for n in shortscan_jpegs() if n.endswith("_full.jpg")]
    files = [read_golden(SHORTSCAN[n]["path"]) for n in names]
    scans = Scans(files)
    codec = codec_with(monkeypatch, {})
    res, _, _ = device_decode(codec, scans)
    codec.close()
    assert all(r["status"] == 0 for r in res) and res[0]["rows"][-1][2] < scans.scans[0].mcuv
    c = LeptonB200FileCodec(0, gpu_huffman=True)
    got = c.compress(files)
    c.close()
    for n, (st, lep) in zip(names, got):
        assert st == 0 and md5(lep) == SHORTSCAN[n]["lep_md5"], (n, st)
