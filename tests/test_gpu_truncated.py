"""GPU parity on the truncated corpus (tests/golden/truncated/, tests/golden/make_truncated.py): small baseline JPEGs cut
at every byte of their scan, through the file API with every Huffman, mux and range-coder option, the codec (encode on
the front end's CoefImage, decode at every group size), the CLI with -minencodethreads, and one decode batch large
enough for the library to pick the group kernel itself.  Expected values are what the reference CLI wrote
(tests/golden/truncated.json); where the library deliberately differs from the reference (DESIGN.md section 6) the
tests pin the library's outcome."""
import hashlib
import os
import subprocess

import numpy as np
import pytest

from helpers import (GOLDEN, MANIFEST, TRUNC_STATUS, TRUNC_THREADS, TRUNCATED, coef_image_from_lep, lep_chain,
                     load_truncated_lep, oracle_decode_planes, read_golden, truncated_cut_of, truncated_cuts,
                     truncated_leps, truncated_source, truncated_sources)

pytestmark = pytest.mark.gpu

DEC_GROUP_MIN = 6144          # segments from which the library decodes with lep_decode_g2_kernel (lep_capi.cu)


def all_cuts(flag="t1"):
    """(source, bytes, code) of every cut of the corpus."""
    out = []
    for name in truncated_sources():
        src = truncated_source(name)
        out += [(name, src[:cut], code) for cut, code in truncated_cuts(name, flag)]
    return out


def check_chains(cuts, leps, flag):
    """The .lep files of the clean cuts of every source, in cut order, against truncated.json's lep_chain."""
    for name in truncated_sources():
        got = [lep for (n, _, code), lep in zip(cuts, leps) if n == name and TRUNC_STATUS[code] == 0]
        assert lep_chain(got) == TRUNCATED["runs"][name][flag]["lep_chain"], (name, flag)


def photos():
    names = [n for n in sorted(MANIFEST) if n.endswith(".jpg") and MANIFEST[n].get("encode_rc") == 0 and MANIFEST[n].get("lep_md5")
             and not MANIFEST[n].get("progressive")]
    assert len(names) >= 3
    return [(read_golden(n), MANIFEST[n]["lep_md5"]) for n in names[:3]]


@pytest.mark.parametrize("cfg", [
    dict(gpu_huffman=True),
    dict(gpu_huffman=False),
    dict(gpu_huffman=True, env={"LEPB200_RC_MODE": "0"}),
])
def test_every_cut_compresses_to_the_reference_lep_and_back(monkeypatch, cfg):
    """All cuts in one compress call, a few complete photos between them: the truncated files take the host Huffman
    path, the photos the device Huffman decoder and, on the way back, the device re-encode -- both live in one batch.
    Every status is the reference's, every .lep is the reference's, and decompress restores every input."""
    from lepton_b200 import LeptonB200FileCodec
    for k, v in cfg.get("env", {}).items():
        monkeypatch.setenv(k, v)
    cuts = all_cuts()
    ph = photos()
    items = [(j, TRUNC_STATUS[code]) for _, j, code in cuts]
    step = len(items) // len(ph)
    for k, (j, m) in enumerate(ph):
        items.insert(k * step + k, (j, 0))
    fc = LeptonB200FileCodec(0, host_threads=8, gpu_huffman=cfg["gpu_huffman"])
    try:
        res = fc.compress([j for j, _ in items])
        ok = [(j, lep) for (j, rc), (st, lep) in zip(items, res) if rc == 0]
        back = fc.decompress([lep for _, lep in ok])
    finally:
        fc.close()
    for k, ((j, rc), (st, _)) in enumerate(zip(items, res)):
        assert st == rc, (k, len(j), st, rc)
    for k, (j, m) in enumerate(ph):
        assert items[k * step + k][0] == j and hashlib.md5(res[k * step + k][1]).hexdigest() == m, k
    cut_res = [r for i, r in enumerate(res) if i not in {k * step + k for k in range(len(ph))}]
    check_chains(cuts, [lep for _, lep in cut_res], "t1")
    assert len(ok) > 4000
    for k, ((j, _), (st, out)) in enumerate(zip(ok, back)):
        assert st == 0 and out == j, (k, len(j), st)


@pytest.mark.parametrize("env", [{}, {"LEPB200_RC_MODE": "0"}])
def test_codec_encodes_the_front_end_image_like_the_reference(monkeypatch, env):
    """encode_images on HostJpeg(cut).coef_image() for every cut the reference codes, plain and with
    -minencodethreads=4 / 8: the container around the GPU streams is the reference's .lep.  The image carries the
    truncation bounds, so the blocks past them are not coded."""
    from lepton_b200 import HostJpeg, LeptonB200Codec
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    for flag in sorted(TRUNC_THREADS):
        cuts = all_cuts(flag)
        hjs = [HostJpeg(j, min_threads=TRUNC_THREADS[flag]) for _, j, _ in cuts]
        todo = [k for k, hj in enumerate(hjs) if hj.status == 0]
        assert all(hjs[k].status == TRUNC_STATUS[cuts[k][2]] for k in range(len(cuts)) if k not in set(todo))
        c = LeptonB200Codec(0)
        try:
            got = c.encode_images([hjs[k].coef_image() for k in todo])
        finally:
            c.close()
        leps = [b""] * len(cuts)
        for k, g in zip(todo, got):
            st = next((s.status for s in g if s.status), 0)
            assert st == TRUNC_STATUS[cuts[k][2]], (flag, k, [s.status for s in g])
            if st == 0:
                leps[k] = hjs[k].write_lep([s.data for s in g])
        check_chains(cuts, leps, flag)


@pytest.mark.parametrize("mode,lanes", [("1", None), ("2", "4"), ("2", "8"), ("2", "32")])
def test_codec_decodes_the_committed_cuts_to_the_oracle_planes(monkeypatch, mode, lanes):
    """decode_images on every committed reference .lep (t4 / t8 records included) into sentinel planes, warp kernel and
    the group kernel at every group size the library ships: the oracle's planes, zero past the bounds."""
    from lepton_b200 import HostLep, LeptonB200Codec
    monkeypatch.setenv("LEPB200_DEC_MODE", mode)
    if lanes:
        monkeypatch.setenv("LEPB200_DEC_LANES", lanes)
    imgs, streams, want = [], [], []
    for name in truncated_leps():
        lf = load_truncated_lep(name)
        planes, s = oracle_decode_planes(lf)
        img = HostLep(read_golden("truncated/" + name)).coef_image()
        img.planes = [np.full_like(p, 77) for p in img.planes]
        imgs.append(img)
        streams.append(list(s[:lf.nseg]))
        want.append(planes)
    c = LeptonB200Codec(0)
    try:
        st = c.decode_images(imgs, streams)
    finally:
        c.close()
    assert all(s == 0 for s in st), st
    for name, img, planes in zip(truncated_leps(), imgs, want):
        for k in range(img.ncmp):
            assert np.array_equal(img.planes[k], planes[k]), (name, k)


def test_large_decode_batch_takes_the_group_kernel_by_itself(monkeypatch):
    """The t8 records repeated into one batch of at least DEC_GROUP_MIN segments, no decode-mode override: the library
    chooses lep_decode_g2_kernel by batch size, and every segment decodes to the oracle's planes."""
    from lepton_b200 import LeptonB200Codec
    monkeypatch.delenv("LEPB200_DEC_MODE", raising=False)
    monkeypatch.delenv("LEPB200_DEC_LANES", raising=False)
    recs = [n for n in truncated_leps() if TRUNCATED["leps"][n]["flag"] == "t8" and load_truncated_lep(n).nseg > 1]
    assert recs
    base = []
    for name in recs:
        lf = load_truncated_lep(name)
        planes, s = oracle_decode_planes(lf)
        base.append((lf, planes, list(s[:lf.nseg])))
    imgs, streams, want = [], [], []
    k = 0
    while sum(im.nseg for im in imgs) < DEC_GROUP_MIN:
        lf, planes, s = base[k % len(base)]
        imgs.append(coef_image_from_lep(lf, [np.full_like(p, -9) for p in planes]))
        streams.append(s)
        want.append(planes)
        k += 1
    c = LeptonB200Codec(0)
    try:
        st = c.decode_images(imgs, streams)
    finally:
        c.close()
    assert len(st) >= DEC_GROUP_MIN and all(s == 0 for s in st)
    for i, (img, planes) in enumerate(zip(imgs, want)):
        for p, q in zip(img.planes, planes):
            assert np.array_equal(p, q), i


def test_cli_minencodethreads_on_cuts(tmp_path):
    """The command line with -minencodethreads=4 / 8 on a sample of cuts: the reference's .lep where it wrote one and
    the round trip; 6 (COEFFICIENT_OUT_OF_RANGE) where the reference's threads reported THREAD_PROTOCOL_ERROR."""
    exe = os.path.join(os.path.dirname(GOLDEN), "..", "lepton_b200", "bin", "lepton-b200")
    assert os.path.exists(exe), "build() did not produce the CLI"
    def run(args):
        return subprocess.run([exe] + args, capture_output=True)

    jpg, lep, back = str(tmp_path / "c.jpg"), str(tmp_path / "c.lep"), str(tmp_path / "b.jpg")
    sample = [(e["source"], e["cut"], e["flag"], n) for n, e in TRUNCATED["leps"].items() if e["flag"] != "t1"]
    for name in truncated_sources():
        for flag in ("t4", "t8"):
            cuts = truncated_cuts(name, flag)
            sample += [(name, cut, flag, None) for cut, code in cuts[::37] + [x for x in cuts if x[1] == "t"][:2]]
    assert sum(1 for _, _, _, n in sample if n) >= 8
    for name, cut, flag, ref in sample:
        code = dict(truncated_cuts(name, flag))[cut]
        for p in (lep, back):
            if os.path.exists(p):
                os.unlink(p)
        with open(jpg, "wb") as f:
            f.write(truncated_source(name)[:cut])
        p = run(["-skipverify", "-minencodethreads=%d" % TRUNC_THREADS[flag], jpg, lep])
        assert p.returncode == TRUNC_STATUS[code], (name, flag, cut, p.returncode, code, p.stderr)
        if TRUNC_STATUS[code]:
            continue
        if ref:
            assert open(lep, "rb").read() == read_golden("truncated/" + ref), ref
        p = run([lep, back])
        assert p.returncode == 0 and open(back, "rb").read() == truncated_source(name)[:cut], (name, flag, cut, p.stderr)


def test_committed_leps_decompress_to_the_cut():
    """Every committed reference .lep of a cut restores the cut through the file API -- the multi-segment records
    the reference's own decoder refuses included."""
    from lepton_b200 import LeptonB200FileCodec
    names = truncated_leps()
    fc = LeptonB200FileCodec(0, host_threads=4)
    try:
        back = fc.decompress([read_golden("truncated/" + n) for n in names])
    finally:
        fc.close()
    for n, (st, out) in zip(names, back):
        assert st == 0 and out == truncated_cut_of(n), n
