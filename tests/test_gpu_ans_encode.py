"""Coding rANS segment streams (container version 3) on the GPU through the C ABI: kernel A with the rANS model and the
rANS pass, against the reference's fixtures (tests/golden/ans.json) and the oracle's writer; mixed bool / rANS batches;
and the bool-only batches, whose kernels and streams stay what they were."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if os.path.join(os.path.dirname(HERE), "oracle") not in sys.path:
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "oracle"))

import oracle_ans  # noqa: E402
from ans_helpers import ans_cases, image_geometry, image_segments, load_ans_case  # noqa: E402
from helpers import coef_image_from_lep, oracle_encode_image, random_coef_image  # noqa: E402
from test_gpu_kernel_edges import codec_with  # noqa: E402

pytestmark = pytest.mark.gpu

BOOL, ANS = 0, 1
RC_FORMS = {"parallel": {"LEPB200_RC_MODE": "1"}, "parallel_regfeed": {"LEPB200_RC_MODE": "1", "LEPB200_RC_FEED": "0"},
            "serial": {"LEPB200_RC_MODE": "0"}}
# count pre-pass + token offsets (2), kernel A (1), range pass + digit offsets + pieces + carries (4), compaction (1)
PHOTO_ENCODE_LAUNCHES = 8


def tok(p, bit):
    return p | (bit << 8)


def oracle_ans_image(img):
    g = image_geometry(img)
    return [oracle_ans.encode_segment(g, img.planes, *seg) for seg in image_segments(img)]


@pytest.mark.parametrize("form", list(RC_FORMS))
def test_reference_fixture_streams(monkeypatch, form):
    """Every version-3 fixture in one batch (the planes and segments of its version-1 twin): the fixture's streams."""
    c = codec_with(monkeypatch, RC_FORMS[form])
    imgs, want = [], []
    for name in ans_cases():
        lf, planes, _, st, _ = load_ans_case(name)
        imgs.append(coef_image_from_lep(lf, planes))
        want.append(list(st))
    got = c.encode_images(imgs, coders=[ANS] * len(imgs))
    for name, g, w in zip(ans_cases(), got, want):
        assert [s.status for s in g] == [0] * len(w), name
        assert [s.data for s in g] == w, name
    c.close()


def token_corpus():
    rng = np.random.default_rng(77)
    streams = [(rng.integers(1, 256, n) | (rng.integers(0, 2, n) << 8)).astype(np.uint16) for n in list(range(41)) + [255, 256, 257, 777]]
    for t in (tok(1, 0), tok(255, 1), tok(128, 0)):
        for n in (1, 40, 333, 4097):
            streams.append(np.full(n, t, np.uint16))
    for k in range(8):                       # states on the emission threshold 2^55 * 2^k (test_emu_ans_encode)
        per_state = [tok(1, 0)] * 2 + [tok(64, 0)] * 2 + [tok(128, 0)] * k + [tok(2 ** k, 0)]
        t = np.array([v for v in per_state for _ in range(2)][::-1] * 3, np.uint16)
        streams += [t, t[1:]]
    big = (rng.integers(1, 256, (1 << 20) + 4097) | (rng.integers(0, 2, (1 << 20) + 4097) << 8)).astype(np.uint16)
    big[: len(big) // 3] = tok(1, 0)
    streams.append(big)
    return streams


@pytest.mark.parametrize("form", list(RC_FORMS))
def test_token_streams_next_to_bool_ones(monkeypatch, form):
    """The token entry with a coder per segment: the rANS streams equal the oracle's writer and stay inside their token
    slots (canaries); bool streams in the same batch equal a bool-only batch's."""
    c = codec_with(monkeypatch, RC_FORMS[form])
    ans = token_corpus()
    rng = np.random.default_rng(3)
    bools = [(rng.integers(1, 256, n) | (rng.integers(0, 2, n) << 8)).astype(np.uint16) for n in (0, 5, 1000, 20000)]
    caps = [len(t) + 4096 for t in bools]
    ref, bad = c.range_code(bools, caps)
    assert bad == 0
    streams, coders = [], []
    for i, a in enumerate(ans):                     # the bool streams between the first rANS ones
        streams.append(a), coders.append(ANS)
        if i < len(bools):
            streams.append(bools[i]), coders.append(BOOL)
    got, bad = c.range_code(streams, [len(s) + 4096 for s in streams], coders=coders)
    assert bad == 0
    k = 0
    for s, cd, (st, data, moved) in zip(streams, coders, got):
        if cd == ANS:
            assert (st, data) == oracle_ans.ans_encode(s), len(s)
            assert moved
            assert len(data) <= len(s) + 29 + ((len(s) + 9) >> 25)
        else:
            assert (st, data, moved) == ref[k]
            k += 1
    c.close()


def test_probability_0_tokens_give_status_1():
    """Long (0, 0) / (0, 1) streams through the token entry (the reference's writer asserts on them): status 1, and the
    segments next to them in the token arena, rANS and bool, still come out right."""
    from lepton_b200 import LeptonB200Codec
    c = LeptonB200Codec(0)
    rng = np.random.default_rng(8)
    good = (rng.integers(1, 256, 30001) | (rng.integers(0, 2, 30001) << 8)).astype(np.uint16)
    mixed = good.copy()
    mixed[::5] = tok(0, 0)
    streams = [np.full(100000, tok(0, 0), np.uint16), good, np.full(5000, tok(0, 1), np.uint16), mixed, good[:777], good]
    coders = [ANS, ANS, ANS, ANS, BOOL, ANS]
    got, bad = c.range_code(streams, [len(x) + 4096 for x in streams], coders=coders)
    assert bad == 0
    assert [st for st, _, _ in got] == [1, 0, 1, 1, 0, 0]
    assert got[1][:2] == got[5][:2] == oracle_ans.ans_encode(good)
    ref, _ = c.range_code([good[:777]], [777 + 4096])
    assert got[4] == ref[0]
    c.close()


def test_fetch_files_refuses_rans_segments():
    from lepton_b200 import LeptonB200Codec, LeptonB200Error
    c = LeptonB200Codec(0)
    with pytest.raises(LeptonB200Error, match="rANS"):
        c.range_code([np.full(10, tok(9, 1), np.uint16)], [4096], files=[1], headers=[b"x"], coders=[ANS])
    c.close()


def test_large_mixed_batch_round_trip():
    """1200 images of 2..4 segments, bool and rANS interleaved: every rANS stream is the oracle's and decodes back to
    the planes on the GPU; every bool stream is what the bool-only batch gives."""
    from lepton_b200 import CoefImage, LeptonB200Codec
    rng = np.random.default_rng(2024)
    imgs = [random_coef_image(rng, ncmp=3, mcuh=int(rng.integers(1, 4)), mcuv=int(rng.integers(2, 5)), nseg=int(rng.integers(2, 5)),
                              density=float(rng.uniform(0.05, 0.6))) for _ in range(1200)]
    for im in imgs:
        assert im.nseg >= 2
    coders = [int(x) for x in rng.integers(0, 2, len(imgs))]
    c = LeptonB200Codec(0)
    bool_only = c.encode_images(imgs)
    got = c.encode_images(imgs, coders=coders)
    ans_imgs, ans_streams = [], []
    for img, cd, g, b in zip(imgs, coders, got, bool_only):
        assert [s.status for s in g] == [0] * img.nseg
        if cd == BOOL:
            assert [s.data for s in g] == [s.data for s in b]
        else:
            want = oracle_ans_image(img)
            assert [s.data for s in g] == [s for _, s, _ in want]
            assert [s.ndecisions for s in g] == [n for _, _, n in want]
            ans_imgs.append(img)
            ans_streams.append([s.data for s in g])
    assert len(ans_imgs) > 400
    out = [CoefImage(ncmp=im.ncmp, mcuv=im.mcuv, bch=im.bch, bcv=im.bcv, qtables_zigzag=im.qtables_zigzag,
                     planes=[np.full_like(p, -3) for p in im.planes], luma_y_start=im.luma_y_start) for im in ans_imgs]
    st = c.decode_images(out, ans_streams, coders=[ANS] * len(out))
    assert st == [0] * len(st)
    for o, im in zip(out, ans_imgs):
        for a, b in zip(o.planes, im.planes):
            assert np.array_equal(a, b)
    c.close()


@pytest.mark.parametrize("form", list(RC_FORMS))
def test_bool_batches_are_unchanged(monkeypatch, form):
    """An all-bool batch, with no coders and with every coder CODER_BOOL: the parent's kernels (PHOTO_ENCODE_LAUNCHES under
    the parallel range coder) and the oracle's streams."""
    c = codec_with(monkeypatch, RC_FORMS[form])
    rng = np.random.default_rng(11)
    imgs = [random_coef_image(rng, ncmp=3, mcuh=3, mcuv=3, nseg=2) for _ in range(5)]
    want = [[r[1] for r in oracle_encode_image(im)] for im in imgs]
    counts = []
    for coders in (None, [BOOL] * len(imgs)):
        before = c.kernel_launches
        got = c.encode_images(imgs, coders=coders)
        counts.append(c.kernel_launches - before)
        assert [[s.data for s in g] for g in got] == want
    assert counts[0] == counts[1]
    if form != "serial":
        assert counts[0] == PHOTO_ENCODE_LAUNCHES
    c.close()


def case_input(e):
    """The input the reference coded for a case of ans.json (tests/golden/make_ans.py): its source, cut to input_size
    bytes, or behind a prefix of the generated bytes (i * 37 + 11) & 255 (the -embedding cases)."""
    import hashlib
    from helpers import GOLDEN
    data = open(os.path.join(GOLDEN, e["source"]), "rb").read()
    n = e["input_size"]
    data = data[:n] if n <= len(data) else bytes((i * 37 + 11) & 255 for i in range(n - len(data))) + data
    assert hashlib.md5(data).hexdigest() == e["input_md5"]
    return data


# What the adapter's decoder does not restore as the reference does, whatever the coder (the bool-coded build,
# oracle/_ref/lepton-b200plug, does the same on the file's version-1 twin).  The row entry (threaded or -singlethread)
# refuses truncated files and files with restart intervals with 33; the verify pass of an encode goes through that entry,
# so their verified encode fails with 41.  The full-plane entry restores the -embedding file to other bytes.
ROW_ENTRY_REFUSES = {"cut_android_40000", "cut_grayscale_30000_t4", "cut_iphonecrop2_9001", "narrowrst"}
RESTORE_DIFFERS = {("emb_androidcrop_p1001", "-forceprogressive")}


def test_reference_cli_writes_and_restores_ans_files(tmp_path):
    """oracle/_ref/lepton-b200plug-ans = the reference's CLI built with -DENABLE_ANS_EXPERIMENTAL and the GPU coder behind
    its encoder and decoder factory lines (lepton_b200/adapter/Makefile.plug).  For every case of tests/golden/ans.json,
    `-ans <flags> input out.lep` with -skipverify writes the bytes the reference wrote; with verify on (the GPU decoder
    restores the file before it is written) it does too, and the fixture restores to the recorded bytes through every
    decoder entry -- except for the runs named in ROW_ENTRY_REFUSES / RESTORE_DIFFERS, which must fail or differ exactly
    as the bool-coded build does."""
    import hashlib
    import subprocess
    from ans_helpers import ANS, ANS_DIR
    from helpers import GOLDEN
    ref = os.path.join(os.path.dirname(GOLDEN), "..", "oracle", "_ref")
    exe, plain = os.path.join(ref, "lepton-b200plug-ans"), os.path.join(ref, "lepton-b200plug")
    assert os.path.exists(exe), "oracle/_ref/lepton-b200plug-ans missing: __graft_entry__.build() makes it where the reference tree exists"
    md5 = lambda p: hashlib.md5(open(p, "rb").read()).hexdigest() if os.path.exists(p) else None  # noqa: E731
    run = lambda args: subprocess.run(args, capture_output=True, timeout=300)  # noqa: E731

    def fresh(*paths):
        for f in paths:
            if os.path.exists(f):
                os.remove(f)
        return paths[0]

    assert ROW_ENTRY_REFUSES | {n for n, _ in RESTORE_DIFFERS} <= set(ans_cases())
    for name in ans_cases():
        e = ANS[name]
        src, lep, back, p = (str(tmp_path / n) for n in ("in.jpg", "o.lep", "o.jpg", "p.out"))
        with open(src, "wb") as f:
            f.write(case_input(e))
        r = run([exe, "-unjailed", "-skipverify", "-ans"] + e["flags"] + [src, fresh(lep)])
        assert (r.returncode, md5(lep)) == (0, e["lep_md5"]), (name, r.stderr[-2000:])
        r = run([exe, "-unjailed", "-ans"] + e["flags"] + [src, fresh(lep)])
        if name in ROW_ENTRY_REFUSES:
            assert r.returncode == 41, name
            assert run([plain, "-unjailed"] + e["flags"] + [src, fresh(p)]).returncode == 41, name
        else:
            assert (r.returncode, md5(lep)) == (0, e["lep_md5"]), (name, r.stderr[-2000:])
        for flags in (["-forceprogressive"], [], ["-singlethread"]):
            r = run([exe, "-unjailed"] + flags + [os.path.join(ANS_DIR, name + ".lep"), fresh(back)])
            got = (r.returncode, md5(back) if r.returncode == 0 else None)
            if (name in ROW_ENTRY_REFUSES and flags != ["-forceprogressive"]) or (name, "".join(flags)) in RESTORE_DIFFERS:
                assert got != (e["restore"]["rc"], e["restore"]["md5"]), (name, flags, "now restores: drop it from the list")
                r1 = run([plain, "-unjailed"] + flags + [os.path.join(ANS_DIR, name + ".v1.lep"), fresh(p)])
                assert got == (r1.returncode, md5(p) if r1.returncode == 0 else None), (name, flags, r.stderr[-2000:])
            else:
                assert got == (e["restore"]["rc"], e["restore"]["md5"]), (name, flags, r.stderr[-2000:])
