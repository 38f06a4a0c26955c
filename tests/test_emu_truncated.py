"""Truncated JPEGs (tests/golden/truncated/, tests/golden/make_truncated.py): small baseline files cut at every byte of
their scan, held to what the reference CLI made of every cut -- host front end, container, the coder's truncation
bounds in kernel A, the row walk, the decode kernels and the JPEG re-creation -- and random truncation bounds against
the oracle.

What the reference does that the library deliberately does not (DESIGN.md section 6):
  * A cut whose last block holds a coefficient the coder cannot code (a DC code cut short reads zeros for its magnitude
    bits) is refused with COEFFICIENT_OUT_OF_RANGE (6).  With -minencodethreads the reference's other threads then
    print THREAD_PROTOCOL_ERROR (5) as well and the process may leave a partial file; the library has no thread
    protocol and reports 6 for the file, whatever its segment count.
  * Most multi-segment records of a cut are .lep files the reference's own decoder refuses (it asserts on the
    overhang bits of a handoff).  The library restores the cut from every one of them."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu  # noqa: E402
import lepfmt  # noqa: E402
from helpers import (TRUNC_STATUS, TRUNC_THREADS, TRUNCATED, coef_image_from_lep, lep_chain, load_truncated_lep,  # noqa: E402
                     oracle_decode_image, oracle_decode_planes, oracle_encode_image, random_coef_image, read_golden,
                     truncated_cut_of, truncated_cuts, truncated_leps, truncated_source, truncated_sources)

KERNELS = [0, 1, 2]          # range coder: parallel, serial, parallel with the register token feed
DECODERS = [emu.KERNEL_WARP] + [emu.KERNEL_G2(g) for g in (1, 2, 4, 8, 16, 32)]


def library_status(hj, streams_of):
    """The status the library gives a file: the front end's, else the first failing segment's (the coder reports per
    segment; a file with one failing segment fails)."""
    if hj.status:
        return hj.status
    return next((rc for rc, _, _ in streams_of if rc), 0)


def test_corpus_covers_the_cut_classes():
    """Every class the generator selects for is in the committed subset, and the records hold the cases the tests lean
    on: refused cuts, cuts the reference's multi-thread run refuses with THREAD_PROTOCOL_ERROR, .lep files the reference
    cannot decode itself, and segments that start past the last coded row."""
    import hashlib
    for k in ["first_mcu_row", "mcu_row_boundary", "chroma_inside_mcu", "row_past_bound", "eof_fixup", "inside_ff00",
              "inside_rst", "no_eoi", "complete"] + ["%s_%s" % (k, f) for k in ("segment_past_rows", "reference_cannot_decode",
                                                                               "multi_segment") for f in ("t4", "t8")]:
        assert TRUNCATED["classes"].get(k), k
    codes = {f: "".join(TRUNCATED["runs"][n][f]["codes"] for n in truncated_sources()) for f in TRUNC_THREADS}
    assert set("".join(codes.values())) <= set(TRUNC_STATUS)
    assert "u" in codes["t1"] and "c" in codes["t1"] and "t" not in codes["t1"]
    assert "t" in codes["t4"] and "t" in codes["t8"]
    assert codes["t4"].count("n") > 100
    for n in truncated_sources():
        assert hashlib.md5(truncated_source(n)).hexdigest() == TRUNCATED["sources"][n]["jpg_md5"], n
    for name in truncated_leps():
        assert hashlib.md5(read_golden("truncated/" + name)).hexdigest() == TRUNCATED["leps"][name]["lep_md5"], name


@pytest.mark.parametrize("flag", sorted(TRUNC_THREADS))
@pytest.mark.parametrize("name", sorted(TRUNCATED["sources"]))
def test_every_cut_front_end_and_container_match_reference(name, flag):
    """Every cut, plain and with -minencodethreads=4 / 8: the library's status is the reference's (6 where the
    reference's threads reported THREAD_PROTOCOL_ERROR over a 6), and the containers built around the oracle's streams
    are the reference's files (lep_chain: all of them, in cut order).  Each container holds the truncation bounds and
    the splits, and HostJpeg.coef_image() carries the same ones."""
    from lepton_b200 import HostJpeg
    src = truncated_source(name)
    leps = []
    for cut, code in truncated_cuts(name, flag):
        hj = HostJpeg(src[:cut], min_threads=TRUNC_THREADS[flag])
        img = hj.coef_image() if hj.status == 0 else None
        ref = oracle_encode_image(img) if img is not None else []
        assert library_status(hj, ref) == TRUNC_STATUS[code], (name, flag, cut, hj.status, hj.error, code)
        if TRUNC_STATUS[code]:
            continue
        lep = hj.write_lep([s for _, s, _ in ref])
        lf = lepfmt.parse_container(lep)
        assert (list(img.trunc_bcv), list(img.trunc_bc)) == tuple(lepfmt.truncation(lf)), (name, flag, cut)
        assert list(img.luma_y_start) == [h.luma_y_start for h in lf.handoffs], (name, flag, cut)
        leps.append(lep)
    assert lep_chain(leps) == TRUNCATED["runs"][name][flag]["lep_chain"], (name, flag)


def test_coef_image_carries_the_truncation_bounds():
    """HostJpeg(cut).coef_image() and HostLep(lep).coef_image() carry trunc_bcv / trunc_bc, the bounds the reference
    wrote into the .lep, so that encode_images / decode_images code exactly the blocks the reference codes."""
    from lepton_b200 import HostJpeg, HostLep
    cut = 0
    for lep in truncated_leps():
        e = TRUNCATED["leps"][lep]
        assert (e["trunc_bcv"], e["trunc_bc"]) == tuple(lepfmt.truncation(load_truncated_lep(lep))), lep
        img = HostJpeg(truncated_cut_of(lep), min_threads=TRUNC_THREADS[e["flag"]]).coef_image()
        assert (list(img.trunc_bcv), list(img.trunc_bc), list(img.luma_y_start)) == (e["trunc_bcv"], e["trunc_bc"], e["splits"]), lep
        img = HostLep(read_golden("truncated/" + lep)).coef_image()
        assert (list(img.trunc_bcv), list(img.trunc_bc)) == (e["trunc_bcv"], e["trunc_bc"]), lep
        cut += e["trunc_bc"] != [img.bch[c] * img.bcv[c] for c in range(img.ncmp)]
    assert cut >= 20


def coded_blocks(img, c):
    """Mask of the blocks of component c the coder reads: those before trunc_bc, and the first block of every row before
    trunc_bcv (vp8_encoder.cc codes it whatever the bound; it is zero in a truncated file)."""
    n = img.bch[c] * img.bcv[c]
    m = np.arange(n) < img.trunc_bc[c]
    m[np.arange(n) % img.bch[c] == 0] |= np.arange(n)[np.arange(n) % img.bch[c] == 0] < img.trunc_bcv[c] * img.bch[c]
    return m


def committed_batch():
    """Every committed .lep of a cut as the encoder gets it -> (images, reference streams, oracle planes, names)."""
    imgs, want, planes_all = [], [], []
    for name in truncated_leps():
        lf = load_truncated_lep(name)
        planes, streams = oracle_decode_planes(lf)
        imgs.append(coef_image_from_lep(lf, planes))
        want.append(list(streams[:lf.nseg]))
        planes_all.append(planes)
    return imgs, want, planes_all, truncated_leps()


def test_oracle_reproduces_the_committed_streams():
    imgs, want, _, names = committed_batch()
    for img, w, name in zip(imgs, want, names):
        assert [(rc, s) for rc, s, _ in oracle_encode_image(img)] == [(0, s) for s in w], name


def test_front_end_planes_are_the_oracle_planes():
    """The coefficient planes the front end reads from a cut, within the truncation bounds, are the ones the oracle
    decodes from the reference's .lep (eof fix-up included); past the bounds the decoded planes are zero."""
    from lepton_b200 import HostJpeg
    _, _, planes_all, names = committed_batch()
    for name, planes in zip(names, planes_all):
        e = TRUNCATED["leps"][name]
        img = HostJpeg(truncated_cut_of(name), min_threads=TRUNC_THREADS[e["flag"]]).coef_image()
        for c in range(img.ncmp):
            n = img.trunc_bc[c]
            assert np.array_equal(np.asarray(img.planes[c])[:n], planes[c][:n]), (name, c)
            assert not planes[c][n:].any(), (name, c)


@pytest.mark.parametrize("kernel", KERNELS)
def test_committed_cuts_encode_to_the_reference_streams(kernel):
    """Kernel A + B on every committed cut (t4 / t8 records included) in one batch over three persistent CTAs, the
    planes carrying non-zero data past the bounds: the reference's streams."""
    imgs, want, planes_all, names = committed_batch()
    for img in imgs:
        for c in range(img.ncmp):
            skipped = ~coded_blocks(img, c)
            assert not img.planes[c][img.trunc_bc[c]:].any()
            img.planes[c][skipped] = 3
    got = emu.encode_images(imgs, grid_cap=3, kernel=kernel)
    for name, g, w in zip(names, got, want):
        assert [x[0] for x in g] == [0] * len(w), name
        assert [x[1] for x in g] == w, name


@pytest.mark.parametrize("kernel", DECODERS)
def test_committed_cuts_decode_to_the_oracle_planes(kernel):
    """Both decode kernels on the reference's streams, into planes pre-filled with a sentinel: the oracle's planes,
    so every block past the bound comes back as 0."""
    imgs, want, planes_all, names = committed_batch()
    out = [coef_image_from_lep(load_truncated_lep(n), [np.full_like(p, 77) for p in img.planes]) for img, n in zip(imgs, names)]
    st, _ = emu.decode_images(kernel, out, want, grid_cap=3)
    assert all(s == 0 for s in st), st
    for name, img, planes in zip(names, out, planes_all):
        for c in range(img.ncmp):
            assert np.array_equal(img.planes[c], planes[c]), (name, c)


def test_committed_leps_restore_the_cut():
    """HostLep re-creates every cut from the oracle's planes, t4 / t8 records included -- also the ones the reference's
    own decoder refuses (a deliberate difference, DESIGN.md section 6)."""
    from lepton_b200 import HostLep
    _, _, planes_all, names = committed_batch()
    refused = 0
    for name, planes in zip(names, planes_all):
        e = TRUNCATED["leps"][name]
        hl = HostLep(read_golden("truncated/" + name))
        assert hl.status == 0, (name, hl.error)
        assert hl.recode(planes) == truncated_cut_of(name), name
        refused += dict(truncated_cuts(e["source"], e["flag"]))[e["cut"]] == "n"
    assert refused >= 4


def test_thread_protocol_error_cuts_fail_with_the_coefficient_status():
    """Where the reference's multi-thread run printed THREAD_PROTOCOL_ERROR, the plain run failed with
    COEFFICIENT_OUT_OF_RANGE: the library reports 6 for those cuts at every segment count, from the segment that
    holds the coefficient."""
    from lepton_b200 import HostJpeg
    n = 0
    for name in truncated_sources():
        src = truncated_source(name)
        plain = dict(truncated_cuts(name))
        for flag in ("t4", "t8"):
            for cut, code in truncated_cuts(name, flag):
                if code != "t":
                    continue
                assert plain[cut] == "c", (name, flag, cut)
                hj = HostJpeg(src[:cut], min_threads=TRUNC_THREADS[flag])
                st = [rc for rc, _, _ in oracle_encode_image(hj.coef_image())]
                assert hj.status == 0 and 6 in st, (name, flag, cut, st)
                got = emu.encode_images([hj.coef_image()], kernel=0)[0]
                assert [g[0] for g in got] == st, (name, flag, cut)
                n += 1
    assert n >= 20


# the random geometries of test_emu_encode.py / test_emu_decode.py, up to 8 segments
RANDOM_CFGS = [
    dict(ncmp=3, mcuh=5, mcuv=4, sf=((2, 2), (1, 1), (1, 1)), nseg=1),
    dict(ncmp=3, mcuh=7, mcuv=6, sf=((2, 2), (1, 1), (1, 1)), nseg=3),
    dict(ncmp=3, mcuh=9, mcuv=5, sf=((1, 1), (1, 1), (1, 1)), nseg=2),
    dict(ncmp=3, mcuh=6, mcuv=4, sf=((2, 1), (1, 1), (1, 1)), nseg=2),
    dict(ncmp=1, mcuh=11, mcuv=7, sf=((1, 1),), nseg=4),
    dict(ncmp=1, mcuh=1, mcuv=9, sf=((1, 1),), nseg=2),
    dict(ncmp=3, mcuh=1, mcuv=3, sf=((2, 2), (1, 1), (1, 1)), nseg=1),
    dict(ncmp=3, mcuh=12, mcuv=8, sf=((2, 2), (1, 1), (1, 1)), nseg=8, density=0.9, amp=100, qscale=0.3),
    dict(ncmp=3, mcuh=6, mcuv=8, sf=((2, 1), (1, 1), (1, 1)), nseg=8),
    dict(ncmp=1, mcuh=5, mcuv=8, sf=((1, 1),), nseg=8),
]


def random_truncated(cfg, seed, trunc, count=12):
    rng = np.random.default_rng(seed)
    imgs = [random_coef_image(rng, trunc=trunc, **cfg) for _ in range(count)]
    cut = [any(img.trunc_bc[c] < img.bch[c] * img.bcv[c] for c in range(img.ncmp)) for img in imgs]
    assert sum(cut) >= count // 2, cut
    return imgs


@pytest.mark.parametrize("trunc", [True, "any"])
@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("cfg", RANDOM_CFGS)
def test_random_truncation_bounds_encode_vs_oracle(kernel, cfg, trunc):
    """Random truncation bounds over the random geometries (non-zero data past every bound), twelve images in one
    batch over three CTAs: statuses, streams and decision counts of the oracle.  trunc="any": every component ends on
    its own, so chroma rows can outlast the luma rows and the row walk must not stop at the last luma row."""
    imgs = random_truncated(cfg, 777, trunc)
    got = emu.encode_images(imgs, grid_cap=3, kernel=kernel)
    for k, (img, g) in enumerate(zip(imgs, got)):
        ref = oracle_encode_image(img)
        assert [(x[0], x[1], x[2]) for x in g] == [tuple(r) for r in ref], (k, img.trunc_bcv, img.trunc_bc)


@pytest.mark.parametrize("trunc", [True, "any"])
@pytest.mark.parametrize("kernel", DECODERS)
@pytest.mark.parametrize("cfg", RANDOM_CFGS)
def test_random_truncation_bounds_decode_vs_oracle(kernel, cfg, trunc):
    """The oracle's streams of those images decoded into sentinel planes: the oracle's planes (zero past the bounds but
    for the first block of a row the rounded-up trunc_bcv adds), one get per put."""
    imgs = random_truncated(cfg, 778, trunc)
    refs = [oracle_encode_image(img) for img in imgs]
    from lepton_b200 import CoefImage
    out = [CoefImage(ncmp=i.ncmp, mcuv=i.mcuv, bch=i.bch, bcv=i.bcv, qtables_zigzag=i.qtables_zigzag,
                     planes=[np.full_like(p, -5) for p in i.planes], luma_y_start=i.luma_y_start, trunc_bcv=i.trunc_bcv,
                     trunc_bc=i.trunc_bc) for i in imgs]
    st, nd = emu.decode_images(kernel, out, [[s for _, s, _ in r] for r in refs], grid_cap=3)
    assert all(s == 0 for s in st), st
    assert nd == [n for r in refs for _, _, n in r]
    for k, (img, o, r) in enumerate(zip(imgs, out, refs)):
        want = oracle_decode_image(img, [s for _, s, _ in r])
        for c in range(img.ncmp):
            assert np.array_equal(o.planes[c], want[c]), (k, c, img.trunc_bcv, img.trunc_bc)
