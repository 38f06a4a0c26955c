"""GPU parity on the geometry corpus (tests/golden/geometry/, tests/golden/make_geometry.py: every class of sampling
factors in {1, 2} for one and three components, partial MCUs, one-column files, restart intervals, 4 and 8
thread-segments) through the sm_90a kernels on every path the library can take, and random planes over the same
geometries against the oracle.  Expected values are what the reference CLI wrote (tests/golden/geometry.json)."""
import hashlib
import os
import subprocess

import numpy as np
import pytest

from helpers import (GEOMETRY, GOLDEN, coef_image_from_lep, geometry_jpegs, geometry_leps, load_geometry_lep,
                     oracle_decode_image, oracle_decode_planes, oracle_encode_image, plane_hashes, read_golden)
from test_emu_geometry import device_recode_gate, sweep_images

pytestmark = pytest.mark.gpu

EXE = os.path.join(os.path.dirname(GOLDEN), "..", "lepton_b200", "bin", "lepton-b200")


def md5(b):
    return hashlib.md5(b).hexdigest()


@pytest.mark.parametrize("cfg", [
    dict(gpu_huffman=True),
    dict(gpu_huffman=False),
    dict(gpu_huffman=True, env={"LEPB200_HUFF_PAR": "0"}),
    dict(gpu_huffman=True, env={"LEPB200_HUFF_PAR": "1", "LEPB200_HUFF_SUBSEQ_BITS": "512"}),
    dict(gpu_huffman=False, env={"LEPB200_RC_MODE": "0"}),
])
def test_geometry_files_compress_to_the_reference_lep_and_back(monkeypatch, cfg):
    """File API over the whole corpus in one call (GPU or host Huffman decode, both range-coder forms): the reference
    CLI's .lep byte for byte, or its exit status; decompress restores every input, through the device Huffman encoder
    where it takes the file and the host re-encoder where it does not."""
    from lepton_b200 import LeptonB200FileCodec
    for k, v in cfg.get("env", {}).items():
        monkeypatch.setenv(k, v)
    names = geometry_jpegs()
    jpegs = [read_golden(GEOMETRY[n]["path"]) for n in names]
    fc = LeptonB200FileCodec(0, host_threads=4, gpu_huffman=cfg["gpu_huffman"])
    try:
        res = fc.compress(jpegs)
        leps = []
        for n, j, (st, lep) in zip(names, jpegs, res):
            e = GEOMETRY[n]
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
        assert md5(out) == GEOMETRY[n]["back_md5"], n
    if cfg["gpu_huffman"]:
        assert recoded == sum(device_recode_gate(GEOMETRY[n]) for n, _, _ in leps), recoded


@pytest.mark.parametrize("threads", [4, 8])
def test_geometry_multi_segment_records(threads):
    """-minencodethreads=N: the reference's 4- and 8-segment files, chroma-heavy geometries among them, compressed in
    one call and restored."""
    from lepton_b200 import LeptonB200FileCodec
    recs = sorted(n for n, e in GEOMETRY.items() if n.endswith("_t%d.lep" % threads))
    assert len(recs) >= 8
    jpegs = [read_golden(GEOMETRY[GEOMETRY[n]["source"]]["path"]) for n in recs]
    fc = LeptonB200FileCodec(0, host_threads=4, min_encode_threads=threads)
    try:
        res = fc.compress(jpegs)
        back = fc.decompress([lep for _, lep in res])
    finally:
        fc.close()
    for n, j, (st, lep), (st2, out) in zip(recs, jpegs, res, back):
        assert st == 0 and md5(lep) == GEOMETRY[n]["lep_md5"], n
        assert st2 == 0 and out == j, n


@pytest.mark.parametrize("mode,lanes", [("1", None), ("2", "4"), ("2", "8"), ("2", "32")])
def test_geometry_leps_decode_in_one_batch(monkeypatch, mode, lanes):
    """Every .lep record of the corpus in one batch into sentinel planes, warp kernel and group kernel forced: the
    reference's -ujg planes."""
    from lepton_b200 import LeptonB200Codec
    monkeypatch.setenv("LEPB200_DEC_MODE", mode)
    if lanes:
        monkeypatch.setenv("LEPB200_DEC_LANES", lanes)
    imgs, streams_all, names = [], [], []
    for name, source in geometry_leps():
        lf = load_geometry_lep(name)
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
        assert plane_hashes(img.planes) == GEOMETRY[source]["plane_sha256"], name


def test_cli_geometry_files(tmp_path):
    """The command line, one file at a time and in batch mode, on files of every class: chroma with more rows than luma,
    Cb and Cr unlike, a one-column file with restart markers, and grey files the host re-encoder restores."""
    assert os.path.exists(EXE), "build() did not produce the CLI"
    picks = ["y11_c22_plus1.jpg", "y22_cb12_cr11_odd.jpg", "y21_c12_rst3.jpg", "all12_col.jpg", "g22_plus1.jpg",
             "g11_odd.jpg", "y12_c21_tall.jpg"]
    for n in picks[:3]:
        e = GEOMETRY[n]
        src = os.path.join(GOLDEN, e["path"])
        lep, back = str(tmp_path / "o.lep"), str(tmp_path / "o.jpg")
        r = subprocess.run([EXE, "-skipverify", src, lep], capture_output=True)
        assert r.returncode == 0, (n, r.returncode, r.stderr)
        assert md5(open(lep, "rb").read()) == e["lep_md5"], n
        r = subprocess.run([EXE, lep, back], capture_output=True)
        assert r.returncode == 0, (n, r.stderr)
        assert open(back, "rb").read() == open(src, "rb").read(), n
    leps_dir, back_dir = tmp_path / "leps", tmp_path / "back"
    leps_dir.mkdir()
    back_dir.mkdir()
    r = subprocess.run([EXE, "-skipverify", "-outdir=%s" % leps_dir] + [os.path.join(GOLDEN, GEOMETRY[n]["path"]) for n in picks],
                       capture_output=True)
    assert r.returncode == 0, (r.returncode, r.stderr)
    for n in picks:
        assert md5((leps_dir / (n[:-4] + ".lep")).read_bytes()) == GEOMETRY[n]["lep_md5"], n
    r = subprocess.run([EXE, "-outdir=%s" % back_dir] + [str(leps_dir / (n[:-4] + ".lep")) for n in picks], capture_output=True)
    assert r.returncode == 0, (r.returncode, r.stderr)
    for n in picks:
        assert (back_dir / n).read_bytes() == read_golden(GEOMETRY[n]["path"]), n


@pytest.mark.parametrize("trunc", [False, True, "any"])
def test_random_geometry_sweep_vs_oracle(monkeypatch, trunc):
    """Random planes of every geometry of the corpus, 1 to 8 segments, untruncated and with random truncation bounds,
    through LeptonB200Codec: the oracle's statuses, streams and decision counts; decoded back by the warp kernel and the
    group kernel at G = 4, 8 and 32 into sentinel planes, the oracle's planes."""
    from lepton_b200 import CoefImage, LeptonB200Codec
    imgs = sweep_images(32, trunc)
    refs = [oracle_encode_image(img) for img in imgs]
    assert all(rc == 0 for r in refs for rc, _, _ in r)
    c = LeptonB200Codec(0)
    try:
        got = c.encode_images(imgs)
    finally:
        c.close()
    for k, (g, r) in enumerate(zip(got, refs)):
        assert [(s.status, s.data, s.ndecisions) for s in g] == [tuple(x) for x in r], k
    want = [oracle_decode_image(img, [s for _, s, _ in r]) for img, r in zip(imgs, refs)]
    for mode, lanes in (("1", None), ("2", "4"), ("2", "8"), ("2", "32")):
        monkeypatch.setenv("LEPB200_DEC_MODE", mode)
        if lanes:
            monkeypatch.setenv("LEPB200_DEC_LANES", lanes)
        out = [CoefImage(ncmp=i.ncmp, mcuv=i.mcuv, bch=i.bch, bcv=i.bcv, qtables_zigzag=i.qtables_zigzag,
                         planes=[np.full_like(p, -5) for p in i.planes], luma_y_start=i.luma_y_start, trunc_bcv=i.trunc_bcv,
                         trunc_bc=i.trunc_bc) for i in imgs]
        c = LeptonB200Codec(0)
        try:
            st = c.decode_images(out, [[s for _, s, _ in r] for r in refs])
        finally:
            c.close()
        assert all(s == 0 for s in st), (mode, lanes, st)
        for k, (o, w) in enumerate(zip(out, want)):
            for ch in range(o.ncmp):
                assert np.array_equal(o.planes[ch], w[ch]), (mode, lanes, k, ch)
