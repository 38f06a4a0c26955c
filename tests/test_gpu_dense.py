"""GPU parity on the dense corpus (tests/golden/dense/, tests/golden/make_dense.py): white-noise JPEGs every thread-segment
of which needs more range-coder stream than the slot it starts with, so every stream moves to the overflow arena --
through the codec with both range-coder forms, the file API with every Huffman and mux option, and the CLI.  Expected
values are what the reference CLI wrote (tests/golden/dense.json)."""
import hashlib
import os
import subprocess

import numpy as np
import pytest

from helpers import (DENSE, GOLDEN, coef_image_from_lep, dense_jpegs, dense_leps, golden_leps, load_dense_lep, load_lep,
                     oracle_decode_planes, plane_hashes, read_golden)

pytestmark = pytest.mark.gpu

# Kernel launches of one LeptonB200Codec.encode_images call on a batch of photos, whose streams all fit their slots:
# count pre-pass + token offsets (2), kernel A (1), range pass + digit offsets + pieces + carries (4), compaction (1).
# The overflow arena adds no launch there; the count is the same as before streams could grow.
PHOTO_ENCODE_LAUNCHES = 8


def md5(b):
    return hashlib.md5(b).hexdigest()


def dense_batch():
    imgs, want, names = [], [], []
    for name, source in dense_leps():
        lf = load_dense_lep(name)
        planes, streams = oracle_decode_planes(lf)
        imgs.append(coef_image_from_lep(lf, planes))
        want.append(list(streams[:lf.nseg]))
        names.append((name, source))
    return imgs, want, names


@pytest.mark.parametrize("env", [{}, {"LEPB200_RC_MODE": "0"}, {"LEPB200_RC_FEED": "0"}])
def test_dense_batch_encode_matches_reference_streams(monkeypatch, env):
    from lepton_b200 import LeptonB200Codec
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    imgs, want, names = dense_batch()
    c = LeptonB200Codec(0)
    try:
        got = c.encode_images(imgs)
    finally:
        c.close()
    for (name, _), g, w in zip(names, got, want):
        assert [s.status for s in g] == [0] * len(w), name
        assert [s.data for s in g] == w, name


@pytest.mark.parametrize("mode,lanes", [("1", None), ("2", "4"), ("2", "8"), ("2", "32")])
def test_dense_batch_decode_matches_reference_planes(monkeypatch, mode, lanes):
    from lepton_b200 import LeptonB200Codec
    monkeypatch.setenv("LEPB200_DEC_MODE", mode)
    if lanes:
        monkeypatch.setenv("LEPB200_DEC_LANES", lanes)
    imgs, want, names = dense_batch()
    out = [coef_image_from_lep(load_dense_lep(n), [np.full_like(p, 77) for p in img.planes]) for img, (n, _) in zip(imgs, names)]
    c = LeptonB200Codec(0)
    try:
        st = c.decode_images(out, want)
    finally:
        c.close()
    assert all(s == 0 for s in st), st
    for (name, source), img in zip(names, out):
        assert plane_hashes(img.planes) == DENSE[source]["plane_sha256"], name


@pytest.mark.parametrize("cfg", [
    dict(gpu_huffman=True),
    dict(gpu_huffman=False),
    dict(gpu_huffman=True, env={"LEPB200_HUFF_PAR": "0"}),
    dict(gpu_huffman=True, env={"LEPB200_DEVICE_MUX": "0"}),
    dict(gpu_huffman=True, env={"LEPB200_DEVICE_MUX": "1"}),
    dict(gpu_huffman=True, env={"LEPB200_RC_MODE": "0"}),
    dict(gpu_huffman=False, env={"LEPB200_RC_MODE": "0", "LEPB200_DEVICE_MUX": "0"}),
    # 256-bit sub-sequences: the 16-bit codes of some files do not resynchronise within the 62 iterations, so the serial
    # kernel redoes them on the device
    dict(gpu_huffman=True, env={"LEPB200_HUFF_SUBSEQ_BITS": "256", "LEPB200_TRACE": "1"}, serial_redo=True),
])
def test_dense_files_compress_to_the_reference_lep_and_back(monkeypatch, capfd, cfg):
    """File API (resident upload after the GPU Huffman decoder, or host planes; device or host container assembly;
    both range-coder forms): the reference CLI's .lep byte for byte, and decompress restores every input."""
    from lepton_b200 import LeptonB200FileCodec
    for k, v in cfg.get("env", {}).items():
        monkeypatch.setenv(k, v)
    names = dense_jpegs()
    jpegs = [read_golden(DENSE[n]["path"]) for n in names]
    fc = LeptonB200FileCodec(0, host_threads=4, gpu_huffman=cfg["gpu_huffman"])
    try:
        res = fc.compress(jpegs)
        for n, j, (st, lep) in zip(names, jpegs, res):
            assert md5(j) == DENSE[n]["jpg_md5"], n
            assert st == 0, (n, st)
            assert md5(lep) == DENSE[n]["lep_md5"], "%s: .lep differs from the reference CLI's" % n
        back = fc.decompress([lep for _, lep in res])
    finally:
        fc.close()
    for n, j, (st, out) in zip(names, jpegs, back):
        assert st == 0 and out == j, n
        assert md5(out) == DENSE[n]["back_md5"], n
    if cfg.get("serial_redo"):
        import re
        redone = [int(n) for n in re.findall(r"(\d+) images redone by the serial kernel", capfd.readouterr().err)]
        assert redone and max(redone) > 0, redone        # files the sub-sequence kernels gave up on, decoded again serially


def test_dense_files_among_photos_in_one_compress():
    """Dense files between the golden photos in one call: only their segments take the overflow arena, so the device
    gather reads streams from two arenas in one launch."""
    from lepton_b200 import LeptonB200FileCodec
    from helpers import MANIFEST
    photos = [n for n in sorted(MANIFEST) if n.endswith(".jpg") and MANIFEST[n].get("encode_rc") == 0 and MANIFEST[n].get("lep_md5")
              and not MANIFEST[n].get("progressive")]
    assert len(photos) >= 4
    items = []
    for k, n in enumerate(dense_jpegs()):
        items.append((read_golden(DENSE[n]["path"]), DENSE[n]["lep_md5"]))
        if k < len(photos):
            items.append((read_golden(photos[k]), MANIFEST[photos[k]]["lep_md5"]))
    fc = LeptonB200FileCodec(0, host_threads=4)
    try:
        res = fc.compress([j for j, _ in items])
        back = fc.decompress([lep for _, lep in res])
    finally:
        fc.close()
    for k, ((j, want), (st, lep), (st2, out)) in enumerate(zip(items, res, back)):
        assert st == 0 and md5(lep) == want, k
        assert st2 == 0 and out == j, k


def test_dense_multi_segment_record():
    from lepton_b200 import LeptonB200FileCodec
    recs = sorted(n for n, e in DENSE.items() if n.endswith(".lep"))
    assert recs
    for n in recs:
        e = DENSE[n]
        threads = int(e["flags"][0].split("=")[1])
        j = read_golden(DENSE[e["source"]]["path"])
        fc = LeptonB200FileCodec(0, host_threads=4, min_encode_threads=threads)
        try:
            (st, lep), = fc.compress([j])
            (st2, out), = fc.decompress([lep])
        finally:
            fc.close()
        assert st == 0 and md5(lep) == e["lep_md5"], n
        assert st2 == 0 and out == j, n


def test_photo_encode_launch_count_unchanged():
    """Photos, whose streams fit their slots, take no extra launch for the overflow arena."""
    from lepton_b200 import LeptonB200Codec
    imgs = []
    for name in golden_leps():
        lf = load_lep(name)
        planes, _ = oracle_decode_planes(lf)
        imgs.append(coef_image_from_lep(lf, planes))
    c = LeptonB200Codec(0)
    try:
        before = c.kernel_launches
        got = c.encode_images(imgs)
        assert all(s.status == 0 for g in got for s in g)
        assert c.kernel_launches - before == PHOTO_ENCODE_LAUNCHES
    finally:
        c.close()


def test_cli_dense_file(tmp_path):
    """The command line on the Pillow noise file: exit code 0 (not 100), the reference's bytes, and the round trip."""
    exe = os.path.join(os.path.dirname(GOLDEN), "..", "lepton_b200", "bin", "lepton-b200")
    assert os.path.exists(exe), "build() did not produce the CLI"
    e = DENSE["pillow_noise_q100.jpg"]
    src = os.path.join(GOLDEN, e["path"])
    lep, back = str(tmp_path / "o.lep"), str(tmp_path / "o.jpg")
    r = subprocess.run([exe, "-skipverify", src, lep], capture_output=True)
    assert r.returncode == 0, (r.returncode, r.stderr)
    assert md5(open(lep, "rb").read()) == e["lep_md5"]
    r = subprocess.run([exe, lep, back], capture_output=True)
    assert r.returncode == 0, r.stderr
    assert open(back, "rb").read() == open(src, "rb").read()
