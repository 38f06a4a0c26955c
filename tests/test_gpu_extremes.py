"""GPU parity at the coder's numeric limits: the extreme corpus of tests/golden/extremes/ (tests/golden/make_extremes.py --
16-bit quantisers, magnitudes of category 11 at every position, DC values that wrap, Huffman codes 16 bits long, runs of
stuffed 0xFF bytes, restart markers, partial MCUs, files split into 4 and 8 thread-segments, files the reference refuses)
and random planes in the same regimes, through the sm_90a kernels on every kernel path the library can take.  Expected
values are what the reference CLI wrote (tests/golden/extremes.json) or, for random planes, the pinned oracle."""
import hashlib
import os
import subprocess

import numpy as np
import pytest

from helpers import (EXTREMES, GOLDEN, coef_image_from_lep, extreme_jpegs, extreme_leps, load_extreme_lep, oracle_decode_planes,
                     oracle_encode_image, plane_hashes, random_coef_image, read_golden)

pytestmark = pytest.mark.gpu

COLOUR = ("color420_long", "color444_long", "odd_rst")


def md5(b):
    return hashlib.md5(b).hexdigest()


def extreme_batch():
    """(images, per image [(status, stream or None)] per segment): the .lep records with the reference's streams, and the
    refused JPEGs (front end's planes) with the oracle's statuses."""
    from lepton_b200 import HostJpeg
    imgs, want = [], []
    for name, _ in extreme_leps():
        lf = load_extreme_lep(name)
        planes, streams = oracle_decode_planes(lf)
        imgs.append(coef_image_from_lep(lf, planes))
        want.append([(0, s) for s in streams[:lf.nseg]])
    for n in extreme_jpegs():
        if EXTREMES[n]["status_want"]:
            img = HostJpeg(read_golden(EXTREMES[n]["path"])).coef_image()
            imgs.append(img)
            want.append([(rc, s if rc == 0 else None) for rc, s, _ in oracle_encode_image(img)])
    return imgs, want


@pytest.mark.parametrize("env", [{}, {"LEPB200_RC_MODE": "0"}, {"LEPB200_RC_FEED": "0"}])
def test_extreme_batch_encode_matches_reference_streams(monkeypatch, env):
    """The whole corpus in ONE batch: the reference's streams, status 6 exactly where the reference refuses; with the
    default parallel range coder, the serial one, and the register-fed range pass."""
    from lepton_b200 import LeptonB200Codec
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    imgs, want = extreme_batch()
    c = LeptonB200Codec(0)
    try:
        got = c.encode_images(imgs)
    finally:
        c.close()
    assert sum(len(w) for w in want) > 30
    for k, (g, w) in enumerate(zip(got, want)):
        assert [s.status for s in g] == [st for st, _ in w], k
        for i, (seg, (st, ref)) in enumerate(zip(g, w)):
            if st == 0:
                assert seg.data == ref, "image %d segment %d differs from the reference stream" % (k, i)


@pytest.mark.parametrize("mode,lanes", [("1", None), ("2", "4"), ("2", "8"), ("2", "32")])
def test_extreme_batch_decode_matches_reference_planes(monkeypatch, mode, lanes):
    """Every .lep record in one batch decodes to the reference's -ujg planes: warp kernel (LEPB200_DEC_MODE=1) and the
    group kernel at every group size the library ships."""
    from lepton_b200 import LeptonB200Codec
    monkeypatch.setenv("LEPB200_DEC_MODE", mode)
    if lanes:
        monkeypatch.setenv("LEPB200_DEC_LANES", lanes)
    imgs, streams_all, names = [], [], []
    for name, source in extreme_leps():
        lf = load_extreme_lep(name)
        planes, streams = oracle_decode_planes(lf)
        imgs.append(coef_image_from_lep(lf, [np.full_like(p, 77) for p in planes]))
        streams_all.append(streams[:lf.nseg])
        names.append((name, source))
    c = LeptonB200Codec(0)
    try:
        st = c.decode_images(imgs, streams_all)
    finally:
        c.close()
    assert all(s == 0 for s in st), st
    for (name, source), img in zip(names, imgs):
        assert plane_hashes(img.planes) == EXTREMES[source]["plane_sha256"], name


@pytest.mark.parametrize("cfg", [
    dict(gpu_huffman=True),
    dict(gpu_huffman=False),
    dict(gpu_huffman=True, env={"LEPB200_HUFF_PAR": "0"}),
    dict(gpu_huffman=True, env={"LEPB200_HUFF_PAR": "1", "LEPB200_HUFF_SUBSEQ_BITS": "512"}),
    dict(gpu_huffman=True, env={"LEPB200_DEVICE_MUX": "0"}),
    dict(gpu_huffman=True, env={"LEPB200_DEVICE_MUX": "1"}),
    # 256-bit sub-sequences: the 16-bit codes of some files do not resynchronise within the 62 iterations, so the serial
    # kernel redoes them on the device
    dict(gpu_huffman=True, env={"LEPB200_HUFF_SUBSEQ_BITS": "256", "LEPB200_TRACE": "1"}, serial_redo=True),
])
def test_extreme_files_compress_to_the_reference_lep_and_back(monkeypatch, capfd, cfg):
    """File API: compress gives the reference CLI's .lep byte for byte (status 6 and no output for the refused files);
    decompress restores every input, the colour files through the device Huffman encoder when it is on."""
    from lepton_b200 import LeptonB200FileCodec
    for k, v in cfg.get("env", {}).items():
        monkeypatch.setenv(k, v)
    names = extreme_jpegs()
    jpegs = [read_golden(EXTREMES[n]["path"]) for n in names]
    fc = LeptonB200FileCodec(0, host_threads=4, gpu_huffman=cfg["gpu_huffman"])
    try:
        res = fc.compress(jpegs)
        leps = []
        for n, j, (st, lep) in zip(names, jpegs, res):
            e = EXTREMES[n]
            assert md5(j) == e["jpg_md5"], n
            assert st == e["status_want"], (n, st)
            if st == 0:
                assert md5(lep) == e["lep_md5"], "%s: .lep differs from the reference CLI's" % n
                leps.append((n, j, lep))
            else:
                assert lep == b"", n
        back = fc.decompress([lep for _, _, lep in leps])
        recoded = fc.last_gpu_recoded
    finally:
        fc.close()
    for (n, j, _), (st, out) in zip(leps, back):
        assert st == 0 and out == j, n
        assert md5(out) == EXTREMES[n]["back_md5"], n
    if cfg["gpu_huffman"]:
        assert recoded >= len(COLOUR), recoded
    if cfg.get("serial_redo"):
        import re
        redone = [int(n) for n in re.findall(r"(\d+) images redone by the serial kernel", capfd.readouterr().err)]
        assert redone and max(redone) > 0, redone        # files the sub-sequence kernels gave up on, decoded again serially


@pytest.mark.parametrize("threads", [4, 8])
def test_extreme_files_multi_segment_records(threads):
    """-minencodethreads=N: the reference's 4- and 8-segment files, whose thread handoffs carry extreme DC predictors,
    compressed and restored."""
    from lepton_b200 import LeptonB200FileCodec
    recs = sorted(n for n, e in EXTREMES.items() if n.endswith("_t%d.lep" % threads))
    assert recs
    jpegs = [read_golden(EXTREMES[EXTREMES[n]["source"]]["path"]) for n in recs]
    fc = LeptonB200FileCodec(0, host_threads=4, min_encode_threads=threads)
    try:
        res = fc.compress(jpegs)
        back = fc.decompress([lep for _, lep in res])
    finally:
        fc.close()
    for n, j, (st, lep), (st2, out) in zip(recs, jpegs, res, back):
        assert st == 0 and md5(lep) == EXTREMES[n]["lep_md5"], n
        assert st2 == 0 and out == j, n


def test_cli_extreme_file(tmp_path):
    """The command line on a 4:2:0 file with 16-bit Huffman codes and category-11 magnitudes, and on a refused file."""
    exe = os.path.join(os.path.dirname(GOLDEN), "..", "lepton_b200", "bin", "lepton-b200")
    assert os.path.exists(exe), "build() did not produce the CLI"
    e = EXTREMES["color420_long.jpg"]
    src = os.path.join(GOLDEN, e["path"])
    lep, back = str(tmp_path / "o.lep"), str(tmp_path / "o.jpg")
    r = subprocess.run([exe, "-skipverify", src, lep], capture_output=True)
    assert r.returncode == 0, r.stderr
    assert md5(open(lep, "rb").read()) == e["lep_md5"]
    r = subprocess.run([exe, lep, back], capture_output=True)
    assert r.returncode == 0, r.stderr
    assert open(back, "rb").read() == open(src, "rb").read()
    r = subprocess.run([exe, "-skipverify", os.path.join(GOLDEN, EXTREMES["cat12.jpg"]["path"]), str(tmp_path / "x.lep")],
                       capture_output=True)
    assert r.returncode == 6, (r.returncode, r.stderr)


@pytest.mark.parametrize("cfg", [
    dict(ncmp=3, mcuh=6, mcuv=4, sf=((2, 2), (1, 1), (1, 1)), nseg=3, q16=True, max_cat=11),
    dict(ncmp=1, mcuh=8, mcuv=8, sf=((1, 1),), nseg=4, q16=True, max_cat=11, density=0.9),
    dict(ncmp=3, mcuh=6, mcuv=4, sf=((2, 1), (1, 1), (1, 1)), nseg=3, max_cat=11),
    dict(ncmp=1, mcuh=8, mcuv=8, sf=((1, 1),), nseg=8, max_cat=11, density=0.9),
    dict(ncmp=3, mcuh=5, mcuv=4, sf=((1, 1), (1, 1), (1, 1)), nseg=2, q16=True, max_cat=11, dc_max=2047),
    dict(ncmp=1, mcuh=6, mcuv=8, sf=((1, 1),), nseg=8, dc_max=2047),
])
def test_random_extreme_planes_vs_oracle(monkeypatch, cfg):
    """Random planes in the extreme regimes: encode status per segment, stream and decision count as the oracle; every
    segment the oracle codes decodes back (warp and group kernel) to the input planes."""
    from lepton_b200 import CoefImage, LeptonB200Codec
    rng = np.random.default_rng(4321)
    img = random_coef_image(rng, **cfg)
    ref = oracle_encode_image(img)
    c = LeptonB200Codec(0)
    try:
        got = c.encode_images([img])[0]
        assert [g.status for g in got] == [r[0] for r in ref]
        for g, r in zip(got, ref):
            if r[0] == 0:
                assert (g.data, g.ndecisions) == (r[1], r[2])
    finally:
        c.close()
    if any(r[0] for r in ref):
        return
    for mode in ("1", "2"):
        monkeypatch.setenv("LEPB200_DEC_MODE", mode)
        c = LeptonB200Codec(0)
        out = CoefImage(ncmp=img.ncmp, mcuv=img.mcuv, bch=img.bch, bcv=img.bcv, qtables_zigzag=img.qtables_zigzag,
                        planes=[np.full_like(p, -5) for p in img.planes], luma_y_start=img.luma_y_start)
        try:
            st = c.decode_images([out], [[r[1] for r in ref]])
        finally:
            c.close()
        assert st == [0] * len(ref), (mode, st)
        for a, b in zip(out.planes, img.planes):
            assert np.array_equal(a, b), mode
