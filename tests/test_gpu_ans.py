"""Container version 3 (the reference's -ans files: rANS-coded streams) on the GPU: the decode kernels through the C ABI,
and the file API and the CLI against what the reference restored from every fixture of tests/golden/ans.json
(tests/golden/make_ans.py)."""
import hashlib
import os
import subprocess
import zlib

import numpy as np
import pytest

from ans_helpers import ANS, ANS_DIR, ans_cases, load_ans_case
from helpers import GOLDEN, coef_image_from_lep, read_golden

pytestmark = pytest.mark.gpu

EXE = os.path.join(os.path.dirname(GOLDEN), "..", "lepton_b200", "bin", "lepton-b200")
SMALL = [n for n in ans_cases() if n.startswith("geo_") or n in ("colorswap", "all22_tall_t8", "cut_iphonecrop2_9001")]


def md5(b):
    return hashlib.md5(b).hexdigest()


def brotli_available():
    from lepton_b200 import lib
    return bool(lib().lepb200_host_brotli_available())


def ans_lep(name):
    return open(os.path.join(ANS_DIR, name + ".lep"), "rb").read()


def restore_want(name, key):
    e = ANS[name]["restore_zlib0" if key == "zlib0" else "restore"]
    return e["rc"], e["md5"]


def batch(replicas):
    """Every fixture once and the small ones `replicas` times more: (images, streams, the oracle's planes)."""
    imgs, streams, want = [], [], []
    for name in ans_cases() + SMALL * replicas:
        lf, planes, _, st, _ = load_ans_case(name)
        imgs.append(coef_image_from_lep(lf, [np.full_like(p, 77) for p in planes]))
        streams.append(st)
        want.append(planes)
    return imgs, streams, want


@pytest.mark.parametrize("mode", ["warp", "group-by-size"])
def test_c_abi_batch_decodes_to_the_reference_planes(mode, monkeypatch):
    """One batch through lepb200_decode_upload_coded: the warp kernel (mode 1), and a batch of more than 6144 segments
    that takes the group kernel by the library's own rule."""
    from lepton_b200 import CODER_ANS, LeptonB200Codec
    if mode == "warp":
        monkeypatch.setenv("LEPB200_DEC_MODE", "1")
    imgs, streams, want = batch(0 if mode == "warp" else 300)
    nseg = sum(im.nseg for im in imgs)
    assert mode == "warp" or nseg >= 6144
    codec = LeptonB200Codec(0)
    try:
        st = codec.decode_images(imgs, streams, coders=[CODER_ANS] * len(imgs))
    finally:
        codec.close()
    assert st == [0] * nseg
    for k, (img, planes) in enumerate(zip(imgs, want)):
        for c in range(img.ncmp):
            assert np.array_equal(img.planes[c], planes[c]), (k, c)


@pytest.mark.parametrize("lanes", ["4", "8", "32"])
def test_group_kernel_every_shape(lanes, monkeypatch):
    from lepton_b200 import CODER_ANS, LeptonB200Codec
    monkeypatch.setenv("LEPB200_DEC_MODE", "2")
    monkeypatch.setenv("LEPB200_DEC_LANES", lanes)
    monkeypatch.setenv("LEPB200_DEC_THREADS", "32")          # several launches of one coder
    imgs, streams, want = batch(2)
    codec = LeptonB200Codec(0)
    try:
        st = codec.decode_images(imgs, streams, coders=[CODER_ANS] * len(imgs))
    finally:
        codec.close()
    assert st == [0] * sum(im.nseg for im in imgs)
    for img, planes in zip(imgs, want):
        for c in range(img.ncmp):
            assert np.array_equal(img.planes[c], planes[c])


@pytest.mark.parametrize("mode", ["0", "1", "2"])
def test_mixed_batch_equals_separate_batches(mode, monkeypatch):
    """Version-1 and version-3 streams of the same images in one batch give what each gives in a batch of its own."""
    from lepton_b200 import CODER_ANS, CODER_BOOL, LeptonB200Codec
    monkeypatch.setenv("LEPB200_DEC_MODE", mode)
    names = ["iphonecrop2_t4", "geo_y22_odd", "all22_tall_t8", "dense_grey_gauss74", "android"]
    loaded = [load_ans_case(n) for n in names]

    def run(which):
        imgs, streams, coders = [], [], []
        for lf, planes, bool_streams, st, _ in loaded:
            for coder, s in ((CODER_ANS, st), (CODER_BOOL, bool_streams)):
                if coder in which:
                    imgs.append(coef_image_from_lep(lf, [np.full_like(p, 5) for p in planes]))
                    streams.append(s)
                    coders.append(coder)
        codec = LeptonB200Codec(0)
        try:
            st = codec.decode_images(imgs, streams, coders=coders)
        finally:
            codec.close()
        assert st == [0] * len(st)
        return [[p.copy() for p in im.planes] for im in imgs]

    mixed, ans_only, bool_only = run((CODER_ANS, CODER_BOOL)), run((CODER_ANS,)), run((CODER_BOOL,))
    assert len(mixed) == 2 * len(names)
    for k in range(len(names)):
        for c in range(len(mixed[2 * k])):
            assert np.array_equal(mixed[2 * k][c], ans_only[k][c])
            assert np.array_equal(mixed[2 * k + 1][c], bool_only[k][c])
            assert np.array_equal(ans_only[k][c], loaded[k][1][c])


@pytest.mark.parametrize("key", ["plain", "zlib0"])
def test_file_api_restores_every_fixture(key):
    """Every fixture in ONE call, next to version-1 files, then concatenated streams of version-3 members mixed with
    version-1 and -2 members: the reference's md5 and exit code for each, or 200 and no bytes without libbrotlidec."""
    from lepton_b200 import LeptonB200FileCodec
    names = ans_cases()
    ordinary = ["android.lep", "androidprogressive.lep", "iphonecrop2_t8.lep"]
    fc = LeptonB200FileCodec(0, host_threads=8, zlib0=key == "zlib0")
    try:
        alone = fc.decompress([read_golden(n) for n in ordinary])
        got = fc.decompress([read_golden(ordinary[0])] + [ans_lep(n) for n in names] + [read_golden(n) for n in ordinary[1:]])
        assert [(s, md5(b)) for s, b in [got[0]] + got[1 + len(names):]] == [(s, md5(b)) for s, b in alone]
        if not brotli_available():
            print("libbrotlidec missing: every version-3 file is refused with 200")
            assert all(s == 200 and b == b"" for s, b in got[1:1 + len(names)])
            return
        print("libbrotlidec present: version-3 files restored")
        for n, (s, b) in zip(names, got[1:1 + len(names)]):
            want_rc, want_md5 = restore_want(n, key)
            assert s == want_rc and md5(b) == want_md5, (n, key, s)
        # concatenated streams: members of version 3, 1 and 2 (tests/golden/future/narrowrst.lep) in one stream each
        v2 = read_golden("future/narrowrst.lep")
        streams = [ans_lep("android") + read_golden("androidcrop.lep"), ans_lep("androidcrop") + v2 + ans_lep("geo_y22_odd"),
                   v2 + ans_lep("iphonecrop2_t4")]
        parts = [[ans_lep("android"), read_golden("androidcrop.lep")], [ans_lep("androidcrop"), v2, ans_lep("geo_y22_odd")],
                 [v2, ans_lep("iphonecrop2_t4")]]
        fc_plain = LeptonB200FileCodec(0, host_threads=8)
        try:
            member_jpegs = [[fc_plain.decompress([m])[0] for m in p] for p in parts]
        finally:
            fc_plain.close()
        got = fc.decompress(streams)
        for k, (s, b) in enumerate(got):
            assert all(ms == 0 for ms, _ in member_jpegs[k])
            joined = b"".join(mb for _, mb in member_jpegs[k])
            assert s == 0, (k, s)
            assert (zlib.decompress(b) if key == "zlib0" else b) == joined, k
    finally:
        fc.close()


@pytest.mark.parametrize("key", ["plain", "zlib0"])
def test_cli_single_file_and_batch_mode(key, tmp_path):
    names = ans_cases()
    flags = ["-zlib0"] if key == "zlib0" else []
    have = brotli_available()
    print("libbrotlidec %s" % ("present: version-3 files restored" if have else "missing: version-3 files refused with 200"))
    for n in names[:6]:
        src, out = tmp_path / (n + ".lep"), tmp_path / (n + ".out")
        src.write_bytes(ans_lep(n))
        r = subprocess.run([EXE] + flags + [str(src), str(out)], capture_output=True)
        want_rc, want_md5 = restore_want(n, key) if have else (200, None)
        assert r.returncode == want_rc, (n, r.returncode, r.stderr[-300:])
        if want_md5:
            assert md5(out.read_bytes()) == want_md5, n
    outdir = tmp_path / "outdir"
    outdir.mkdir()
    srcs = []
    for n in names:
        p = tmp_path / (n + ".lep")
        p.write_bytes(ans_lep(n))
        srcs.append(str(p))
    r = subprocess.run([EXE, "-outdir=" + str(outdir)] + flags + srcs, capture_output=True)
    if have:
        assert r.returncode == 0, r.stderr[-500:]
        for n in names:
            outs = [f for f in os.listdir(outdir) if f.startswith(n + ".")]
            assert len(outs) == 1, (n, outs)
            assert md5((outdir / outs[0]).read_bytes()) == restore_want(n, key)[1], n
    else:
        assert r.returncode != 0
