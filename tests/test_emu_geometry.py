"""The geometry corpus (tests/golden/geometry/, tests/golden/make_geometry.py: every class of sampling factors in {1, 2}
for one and three components, at whole, partial, one-column and odd-width sizes, with restart intervals and 4 / 8
thread-segments) through the host front end, the container and every emulated kernel, against the reference CLI's
.lep files, planes and scans; and random planes over the same geometries against the oracle.

The oracle restates row_spec_from_index and the rest of the geometry with the same reading as the kernels, so a
misreading they shared would not show against it.  The reference's files pin the oracle first
(test_oracle_decodes_the_reference_streams), then everything else is held to them."""
import hashlib
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu  # noqa: E402
import lepfmt  # noqa: E402
from helpers import (GEOMETRY, coef_image_from_lep, geometry_jpegs, geometry_leps, load_geometry_lep,  # noqa: E402
                     oracle_decode_image, oracle_decode_planes, oracle_encode_image, plane_hashes, random_coef_image,
                     read_golden)

KERNELS = [0, 1, 2]          # range coder: parallel, serial, parallel with the register token feed
DECODERS = [emu.KERNEL_WARP] + [emu.KERNEL_G2(g) for g in (1, 2, 4, 8, 16, 32)]
CLASSES = ["alike", "cb_ne_cr", "chroma_heavy", "grey", "luma"]


def md5(b):
    return hashlib.md5(b).hexdigest()


def mult(e):
    return [bv // e["mcuv"] for bv in e["bcv"]]


def device_recode_gate(e):
    """Which files the device Huffman encoder takes (gpu_recode_setup in lep_recode.cc, then the geometry check of
    henc_launch in lep_capi.cu): every colour file, and one-component files whose scan walks the whole plane (1x1
    sampling, no padding blocks).  The others go to the host re-encoder."""
    if len(e["sampling"]) == 3:
        return True
    return e["sampling"] == [[1, 1]] and e["nch"] == e["bch"] and e["ncv"] == e["bcv"]


def source_of(lep_name):
    return lep_name if lep_name in GEOMETRY else lep_name[:-4] + ".jpg"


def test_corpus_covers_the_geometries():
    """The committed files are the ones geometry.json describes, and they hold the cases the tests lean on: every class
    with an accepted file, chroma with more rows per MCU row than luma, Cb and Cr of different widths and heights,
    partial MCUs in some components only, restart intervals, and 4- and 8-segment records of chroma-heavy files."""
    jp = geometry_jpegs()
    for n in jp:
        assert md5(read_golden(GEOMETRY[n]["path"])) == GEOMETRY[n]["jpg_md5"], n
    for name, source in geometry_leps():
        e = GEOMETRY[name] if name in GEOMETRY else GEOMETRY[source]
        assert md5(read_golden("geometry/" + name)) == e["lep_md5"], name
    acc = [GEOMETRY[n] for n in jp if GEOMETRY[n]["status_want"] == 0]
    assert sorted({e["cls"] for e in acc}) == CLASSES
    colour = [e for e in acc if len(e["sampling"]) == 3]
    assert sum(mult(e)[1] > mult(e)[0] for e in colour) >= 8
    assert sum(e["bch"][1] != e["bch"][2] for e in colour) >= 8
    assert sum(e["bcv"][1] != e["bcv"][2] for e in colour) >= 8
    mixed = [e for e in colour if len({e["nch"][c] < e["bch"][c] or e["ncv"][c] < e["bcv"][c] for c in range(3)}) == 2]
    assert len(mixed) >= 8
    assert sum(e["restart"] == 1 for e in colour) >= 6 and sum(e["restart"] == 3 and e["mcuh"] % 3 for e in colour) >= 6
    assert sum(not device_recode_gate(e) for e in acc) >= 8
    for t in (4, 8):
        recs = [e for n, e in GEOMETRY.items() if n.endswith("_t%d.lep" % t)]
        assert len(recs) >= 8 and all(e["nseg"] == t for e in recs)
        assert sum(len(GEOMETRY[e["source"]]["sampling"]) == 3 and mult(GEOMETRY[e["source"]])[1] >
                   mult(GEOMETRY[e["source"]])[0] for e in recs) >= 2


@pytest.mark.parametrize("cls", CLASSES)
def test_front_end_and_container_match_reference(cls):
    """Every file of a class: the front end's planes are the reference's -ujg dump, its splits are the reference's
    (plain and with -minencodethreads), and the container written around the reference's streams is the reference's
    .lep byte for byte."""
    from lepton_b200 import HostJpeg
    n = 0
    for name, source in geometry_leps():
        e = GEOMETRY[source]
        if e["cls"] != cls:
            continue
        rec = GEOMETRY.get(name, {})
        threads = int(rec["flags"][0].split("=")[1]) if rec else 1
        ref = read_golden("geometry/" + name)
        hj = HostJpeg(read_golden(e["path"]), min_threads=threads)
        assert hj.status == 0, (name, hj.error)
        img = hj.coef_image()
        assert plane_hashes(img.planes) == e["plane_sha256"], name
        assert (list(img.bch), list(img.bcv), img.mcuv) == (e["bch"], e["bcv"], e["mcuv"]), name
        lf = lepfmt.parse_container(ref)
        assert list(img.luma_y_start) == [h.luma_y_start for h in lf.handoffs], name
        assert hj.write_lep(lepfmt.demux(lf.payload, lf.version)[:lf.nseg]) == ref, name
        n += 1
    assert n >= 12


def test_oracle_decodes_the_reference_streams():
    """The oracle decodes every reference .lep of the corpus to the reference's planes: it is pinned for these
    geometries before the random sweep compares kernels with it."""
    for name, source in geometry_leps():
        planes, _ = oracle_decode_planes(load_geometry_lep(name))
        assert plane_hashes(planes) == GEOMETRY[source]["plane_sha256"], name


def corpus_batch():
    """Every .lep record as the encoder gets it -> (images, reference streams per image, names)."""
    imgs, want, names = [], [], []
    for name, source in geometry_leps():
        lf = load_geometry_lep(name)
        planes, streams = oracle_decode_planes(lf)
        imgs.append(coef_image_from_lep(lf, planes))
        want.append(list(streams[:lf.nseg]))
        names.append((name, source))
    return imgs, want, names


@pytest.mark.parametrize("kernel", KERNELS)
def test_corpus_encodes_to_the_reference_streams(kernel):
    """Kernel A + B over the whole corpus in one batch over three persistent CTAs: the reference's streams."""
    imgs, want, names = corpus_batch()
    got = emu.encode_images(imgs, grid_cap=3, kernel=kernel)
    for (name, _), g, w in zip(names, got, want):
        assert [x[0] for x in g] == [0] * len(w), name
        assert [x[1] for x in g] == w, name


@pytest.mark.parametrize("kernel", DECODERS)
def test_corpus_decodes_to_the_reference_planes(kernel):
    """The warp kernel and the group kernel at every group size, the whole corpus in one launch into sentinel planes:
    the reference's -ujg planes from the reference's streams."""
    imgs, want, names = corpus_batch()
    out = [coef_image_from_lep(load_geometry_lep(n), [np.full_like(p, 77) for p in img.planes]) for img, (n, _) in zip(imgs, names)]
    st, _ = emu.decode_images(kernel, out, want, grid_cap=3)
    assert all(s == 0 for s in st), st
    for (name, source), img in zip(names, out):
        assert plane_hashes(img.planes) == GEOMETRY[source]["plane_sha256"], name


def check_equal(a, b, name):
    assert a["status"] == b["status"], name
    assert (a["padbit"], a["end_bitpos"], a["nrows"]) == (b["padbit"], b["end_bitpos"], b["nrows"]), name
    assert a["rows"] == b["rows"], name
    for pa, pb in zip(a["planes"], b["planes"]):
        assert np.array_equal(pa, pb), name


@pytest.mark.parametrize("sub_bits", [256, 1024, 4096])
def test_both_huffman_kernels_match_the_host_decoder(sub_bits):
    """lep_huffdecode_kernel and the sub-sequence kernels on every JPEG of the corpus: the host decoder's planes (pinned
    to the -ujg dumps above), and the same status, pad bit, end position and row states.  Every colour file without
    restarts long enough for the sub-sequence kernels (4 sub-sequences) is decoded by them, with no file handed back to
    the serial kernel at 1024 and 4096 bits."""
    names = geometry_jpegs()
    jpegs = [read_golden(GEOMETRY[n]["path"]) for n in names]
    ser, _ = emu.huffman_decode(emu.HUFF_SERIAL, jpegs)
    par, (iters, redo) = emu.huffman_decode(emu.HUFF_SUBSEQ, jpegs, sub_bits=sub_bits)
    eligible = 0
    for n, s, p in zip(names, ser, par):
        assert s is not None and p is not None, n
        assert s["status"] == 0, n
        for got, want in zip(s["planes"], s["host_planes"]):
            assert np.array_equal(got, want), n
        check_equal(p, s, n)
        eligible += s["ncmp"] == 3 and s["rsti"] == 0 and s["nbytes"] * 8 >= 4 * sub_bits
    colour_plain = sum(len(GEOMETRY[n]["sampling"]) == 3 and not GEOMETRY[n]["restart"] for n in names)
    # all of them at 256 bits; at 1024 all but the smallest (one MCU column); at 4096 the larger ones
    assert eligible >= {256: colour_plain, 1024: colour_plain - 4, 4096: 10}[sub_bits], (eligible, colour_plain)
    assert iters > 0
    # with 256-bit sub-sequences one file does not synchronise within the iteration budget; the serial kernel redoes it
    # (same outputs, checked above)
    assert redo == 0 or sub_bits == 256, redo


def test_huffman_encode_kernel_recreates_the_scans():
    """Every .lep record, multi-segment ones included: where the device re-encode takes the file, lep_huffencode_kernel
    re-creates the original scan byte for byte from the job built from the reference's .lep; where it does not (one
    component with sampling other than 1x1), the file is handed to the host re-encoder (no scan layout, an empty job),
    never mis-coded.  The host re-encoder restores every file."""
    from lepton_b200 import HostJpeg, HostLep
    taken = handed = 0
    for name, source in geometry_leps():
        e = GEOMETRY[source]
        jpg = read_golden(e["path"])
        hl = HostLep(read_golden("geometry/" + name))
        assert hl.status == 0, (name, hl.error)
        img = HostJpeg(jpg).coef_image()
        off, n = hl.scan_layout()
        job = emu.henc_job(hl)
        if device_recode_gate(e):
            assert n > 0 and job.scan_bytes == n, name
            scan, segs = emu.huffman_encode(job, img)
            assert [st for st, _ in segs] == [0] * job.nseg, (name, segs)
            assert scan == jpg[off:off + n], name
            assert hl.assemble(scan) == jpg, name
            taken += job.nseg > 1
        else:
            assert (off, n) == (0, 0) and job.scan_bytes == 0, name
            handed += 1
        assert hl.recode(img.planes) == jpg, name
    assert taken >= 14 and handed >= 8, (taken, handed)


def test_corpus_leps_reassembled_by_the_gather_kernel():
    from test_emu_mux import split_lep
    names = [n for n, _ in geometry_leps()]
    raws = [read_golden("geometry/" + n) for n in names]
    got = emu.mux_files([split_lep(r) for r in raws], grid=3)
    for n, g, r in zip(names, got, raws):
        assert g == r, n


# ---- random planes over every geometry of the corpus, against the oracle
SWEEP = sorted({tuple(tuple(s) for s in GEOMETRY[n]["sampling"]) for n in geometry_jpegs()})


def sweep_images(seed, trunc):
    """Two random images per geometry, 1 to 8 segments, MCU grids from one column to 7 x 10."""
    rng = np.random.default_rng(seed)
    imgs = []
    for sf in SWEEP:
        for _ in range(2):
            mcuv = int(rng.integers(2, 11))
            imgs.append(random_coef_image(rng, ncmp=len(sf), mcuh=int(rng.integers(1, 8)), mcuv=mcuv, sf=sf,
                                          nseg=int(rng.integers(1, 9)), trunc=trunc))
    return imgs


@pytest.mark.parametrize("trunc", [False, True, "any"])
def test_random_geometry_sweep_encode_vs_oracle(trunc):
    """Kernel A + B on random planes of every geometry, untruncated and with random truncation bounds (non-zero data
    past every bound), in one batch over three CTAs: statuses, streams and decision counts of the oracle."""
    imgs = sweep_images(31, trunc)
    assert len(imgs) == 2 * len(SWEEP) >= 38
    got = emu.encode_images(imgs, grid_cap=3, kernel=0)
    for k, (img, g) in enumerate(zip(imgs, got)):
        ref = oracle_encode_image(img)
        assert [(x[0], x[1], x[2]) for x in g] == [tuple(r) for r in ref], (k, img.bch, img.bcv, img.trunc_bcv, img.trunc_bc)


@pytest.mark.parametrize("kernel", [emu.KERNEL_WARP] + [emu.KERNEL_G2(g) for g in (4, 8, 32)])
@pytest.mark.parametrize("trunc", [False, True, "any"])
def test_random_geometry_sweep_decode_vs_oracle(kernel, trunc):
    """The oracle's streams of those images decoded into sentinel planes by the warp kernel and the group kernel:
    statuses, decision counts and the oracle's planes."""
    from lepton_b200 import CoefImage
    imgs = sweep_images(32, trunc)
    refs = [oracle_encode_image(img) for img in imgs]
    assert all(rc == 0 for r in refs for rc, _, _ in r)
    out = [CoefImage(ncmp=i.ncmp, mcuv=i.mcuv, bch=i.bch, bcv=i.bcv, qtables_zigzag=i.qtables_zigzag,
                     planes=[np.full_like(p, -5) for p in i.planes], luma_y_start=i.luma_y_start, trunc_bcv=i.trunc_bcv,
                     trunc_bc=i.trunc_bc) for i in imgs]
    st, nd = emu.decode_images(kernel, out, [[s for _, s, _ in r] for r in refs], grid_cap=3)
    assert all(s == 0 for s in st), st
    assert nd == [n for r in refs for _, _, n in r]
    for k, (img, o, r) in enumerate(zip(imgs, out, refs)):
        want = oracle_decode_image(img, [s for _, s, _ in r])
        if not trunc:
            want = img.planes
        for c in range(img.ncmp):
            assert np.array_equal(o.planes[c], want[c]), (k, c, img.bch, img.bcv, img.trunc_bcv, img.trunc_bc)
