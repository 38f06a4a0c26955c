"""Pins the CPU oracle (oracle/lepton_oracle.c) against files written by the UNMODIFIED reference.

tests/golden/*.lep were written by oracle/_ref/lepton (the reference CLI compiled from /root/reference by
oracle/Makefile.ref); manifest.json holds sha256s of the coefficient planes from the reference's own -ujg dump.
 * oracle decode of the reference's segment streams must reproduce the reference's coefficient planes;
 * oracle encode of those planes must reproduce the reference's segment streams byte for byte.
The reference repository's own golden vector images/iphone16.lep (test_suite/test_16threads.sh) is checked in-container.
"""
import hashlib
import os

import numpy as np
import pytest

import lepfmt
import oracle
from helpers import (EXTREMES, GOLDEN, MANIFEST, extreme_jpegs, extreme_leps, geometry_of, golden_leps, load_extreme_lep, load_lep,
                     oracle_decode_planes, oracle_encode_image, plane_hashes, read_golden, segments_of)


@pytest.mark.parametrize("name", golden_leps())
def test_oracle_roundtrips_reference_streams(name):
    lf = load_lep(name)
    planes, streams = oracle_decode_planes(lf)
    src = MANIFEST.get(name[:-4] + ".jpg") or MANIFEST.get(MANIFEST.get(name, {}).get("source", ""), {})
    if "plane_sha256" in src:
        assert plane_hashes(planes) == src["plane_sha256"], "oracle decode != reference -ujg coefficient dump"
    g, _, _ = geometry_of(lf)
    for i, (y0, y1, last) in enumerate(segments_of(lf)):
        rc, s, nd = oracle.encode_segment(g, planes, y0, y1, last)
        assert rc == 0
        assert s == streams[i], "oracle encode != reference stream for segment %d" % i
        assert nd > 0


@pytest.mark.skipif(not os.path.isdir("/root/reference/images"), reason="reference tree only exists in the build container")
@pytest.mark.slow
def test_reference_repo_golden_vector_iphone16(tmp_path):
    """images/iphone16.lep (16 thread segments) is the reference's own golden vector: test_suite/test_16threads.sh
    expects it to decode to iphone.jpg (md5 8ea9fcf1b2c24877aa838dd6ac1df413).  The oracle must decode its 16
    streams to exactly the coefficient planes the reference dumps for iphone.jpg, and re-encode them bit-exactly."""
    import hashlib
    import subprocess
    from conftest import REF_LEPTON
    jpg = "/root/reference/images/iphone.jpg"
    assert hashlib.md5(open(jpg, "rb").read()).hexdigest() == "8ea9fcf1b2c24877aa838dd6ac1df413"
    lf = lepfmt.parse_container(open("/root/reference/images/iphone16.lep", "rb").read())
    assert lf.nseg == 16
    planes, streams = oracle_decode_planes(lf)
    ujg = str(tmp_path / "a.ujg")
    assert subprocess.run([REF_LEPTON, "-ujg", "-skipverify", jpg, ujg], capture_output=True).returncode == 0
    _, ref_planes = lepfmt.parse_ujg_planes(open(ujg, "rb").read())
    for a, b in zip(planes, ref_planes):
        assert np.array_equal(a, b)
    g, _, _ = geometry_of(lf)
    for i, (y0, y1, last) in enumerate(segments_of(lf)):
        rc, s, _ = oracle.encode_segment(g, planes, y0, y1, last)
        assert rc == 0 and s == streams[i]


def _pin_against_reference_lep(lf, jpg_path, tmp_path, nseg, streams=None):
    """Oracle decode of the container's streams == planes the reference dumps for the JPEG; oracle re-encode == streams.
    ``streams``: decode these instead of lf's own (a golden container whose header blob this image cannot read)."""
    import subprocess
    from conftest import REF_LEPTON
    assert len(lf.handoffs) == nseg
    if streams is None:
        streams = lepfmt.demux(lf.payload, lf.version)
    f = lf.frame
    g, _, _ = geometry_of(lf)
    planes = [np.zeros((f.bch[c] * f.bcv[c], 64), dtype=np.int16) for c in range(f.ncmp)]
    for i, (y0, y1, last) in enumerate(segments_of(lf)):
        rc, _ = oracle.decode_segment(g, planes, y0, y1, last, streams[i])
        assert rc == 0, (i, rc)
    ujg = str(tmp_path / "a.ujg")
    assert subprocess.run([REF_LEPTON, "-ujg", "-skipverify", jpg_path, ujg], capture_output=True).returncode == 0
    _, ref_planes = lepfmt.parse_ujg_planes(open(ujg, "rb").read())
    for a, b in zip(planes, ref_planes):
        assert np.array_equal(a, b)
    for i, (y0, y1, last) in enumerate(segments_of(lf)):
        rc, s, _ = oracle.encode_segment(g, planes, y0, y1, last)
        assert rc == 0 and s == streams[i], i


@pytest.mark.skipif(not os.path.isdir("/root/reference/images"), reason="reference tree only exists in the build container")
@pytest.mark.slow
def test_reference_repo_golden_vector_gold_legacy(tmp_path):
    """images/gold-legacy.lep (test_suite/test_legacy.sh expects md5 9ffbfc24d1157d0b1ed7a9b53bef4c23 after decoding):
    a version-1 file from before the handoff table existed -- the payload opens with the segment count and the luma
    split rows (src/lepton/vp8_decoder.cc:337-369).  The JPEG it decodes to is not in images/, so the reference
    binary produces it here and its md5 is the one the reference's test pins."""
    import hashlib
    import subprocess
    from conftest import REF_LEPTON
    jpg = str(tmp_path / "legacy.jpg")
    assert subprocess.run([REF_LEPTON, "-unjailed", "/root/reference/images/gold-legacy.lep", jpg],
                          capture_output=True).returncode == 0
    assert hashlib.md5(open(jpg, "rb").read()).hexdigest() == "9ffbfc24d1157d0b1ed7a9b53bef4c23"
    lf = lepfmt.parse_container(open("/root/reference/images/gold-legacy.lep", "rb").read())
    _pin_against_reference_lep(lf, jpg, tmp_path, nseg=4)


@pytest.mark.skipif(not os.path.isdir("/root/reference/images"), reason="reference tree only exists in the build container")
def test_reference_repo_golden_vector_narrowrst(tmp_path):
    """images/narrowrst.lep (test_suite/test_future_compat.sh expects md5 07e9021d35114bd69f44f5bc1c3788e3 = the md5
    of images/narrowrst.jpg): container version 4, brotli header blob (no brotli decoder in this image), one
    thread-segment, a truncated JPEG with restart markers.  The blob is skipped by its length field; the frame and the
    truncation bounds come from the version-1 container the reference writes for narrowrst.jpg today, whose
    coefficient stream must be byte-identical with the golden file's.  The oracle then has to decode the GOLDEN
    stream to the reference's planes and re-create it."""
    import hashlib
    import subprocess
    from conftest import REF_LEPTON
    jpg = "/root/reference/images/narrowrst.jpg"
    data = open(jpg, "rb").read()
    assert hashlib.md5(data).hexdigest() == "07e9021d35114bd69f44f5bc1c3788e3"
    lf4 = lepfmt.parse_container(open("/root/reference/images/narrowrst.lep", "rb").read(), data)
    assert lf4.version == 4 and lf4.nseg == 1 and lf4.jpeg_size == len(data)
    golden_streams = lepfmt.demux(lf4.payload, lf4.version)
    lep1 = str(tmp_path / "v1.lep")
    assert subprocess.run([REF_LEPTON, "-skipverify", jpg, lep1], capture_output=True).returncode == 0
    lf1 = lepfmt.parse_container(open(lep1, "rb").read())
    assert lf1.version == 1 and "EEE" in lf1.sections
    assert lepfmt.demux(lf1.payload, 1) == golden_streams
    _pin_against_reference_lep(lf1, jpg, tmp_path, nseg=1, streams=golden_streams)


def test_branch_update_matches_reference_semantics():
    """Branch::record_obs_and_update corner cases (src/vp8/model/branch.hh:82-100) through a tiny stream."""
    # An all-zero 1x1-block grayscale image exercises the identity priors; encode/decode must agree.
    q = [[16] * 64]
    g = oracle.make_geometry(1, [1], [1], 1, q)
    planes = [np.zeros((1, 64), dtype=np.int16)]
    rc, s, nd = oracle.encode_segment(g, planes, 0, 1, True)
    assert rc == 0 and nd == 6 + 3 + 3 + 1
    out = [np.ones((1, 64), dtype=np.int16)]
    rc, nd2 = oracle.decode_segment(g, out, 0, 1, True, s)
    assert rc == 0 and nd2 == nd and not out[0].any()


def test_out_of_range_coefficient_is_rejected():
    """COEFFICIENT_OUT_OF_RANGE (exit code 6): src/vp8/encoder/encoder.cc:124,265,343."""
    q = [[16] * 64]
    g = oracle.make_geometry(1, [1], [1], 1, q)
    planes = [np.zeros((1, 64), dtype=np.int16)]
    planes[0][0, 3] = 4096
    rc, _, _ = oracle.encode_segment(g, planes, 0, 1, True)
    assert rc == 6


@pytest.mark.skipif(not os.path.isdir("/root/reference/images"), reason="reference tree only exists in the build container")
@pytest.mark.slow
def test_oracle_vs_live_reference_on_a_large_fixture(tmp_path):
    import subprocess
    from conftest import REF_LEPTON
    jpg = "/root/reference/images/iphonecrop.jpg"
    lep, ujg = str(tmp_path / "a.lep"), str(tmp_path / "a.ujg")
    assert subprocess.run([REF_LEPTON, "-skipverify", jpg, lep], capture_output=True).returncode == 0
    assert subprocess.run([REF_LEPTON, "-ujg", "-skipverify", jpg, ujg], capture_output=True).returncode == 0
    lf = lepfmt.parse_container(open(lep, "rb").read())
    _, planes = lepfmt.parse_ujg_planes(open(ujg, "rb").read())
    g, _, _ = geometry_of(lf)
    streams = lepfmt.demux(lf.payload, lf.version)
    assert lf.nseg == 4
    for i, (y0, y1, last) in enumerate(segments_of(lf)):
        rc, s, _ = oracle.encode_segment(g, planes, y0, y1, last)
        assert rc == 0 and s == streams[i]


# ---- the extreme corpus (tests/golden/make_extremes.py): coefficients, quantisers and Huffman codes at their limits
@pytest.mark.parametrize("name,source", extreme_leps())
def test_oracle_extremes_decode_to_the_reference_planes_and_reencode(name, source):
    """Every reference-written .lep of the extreme corpus: the oracle decodes the reference's streams to the planes of the
    reference's -ujg dump and re-encodes them to the same streams."""
    raw = read_golden("extremes/" + name)
    assert hashlib.md5(raw).hexdigest() == EXTREMES[name if name in EXTREMES else source]["lep_md5"]
    lf = load_extreme_lep(name)
    planes, streams = oracle_decode_planes(lf)
    assert plane_hashes(planes) == EXTREMES[source]["plane_sha256"], "oracle decode != reference -ujg coefficient dump"
    g, _, _ = geometry_of(lf)
    for i, (y0, y1, last) in enumerate(segments_of(lf)):
        rc, s, _ = oracle.encode_segment(g, planes, y0, y1, last)
        assert rc == 0 and s == streams[i], "segment %d" % i


def test_oracle_refuses_the_files_the_reference_refuses():
    """dc_out_of_range (a DC beyond +-1024), dc_residual_long (a DC residual that round-trips but needs 12 bits) and cat12
    (a 12-bit AC magnitude): the reference exits with COEFFICIENT_OUT_OF_RANGE; so does the oracle, on the front end's
    planes."""
    from lepton_b200 import HostJpeg
    refused = [n for n in extreme_jpegs() if EXTREMES[n]["status_want"]]
    assert sorted(refused) == ["cat12.jpg", "dc_out_of_range.jpg", "dc_residual_long.jpg"]
    for n in refused:
        assert EXTREMES[n]["exit_name"] == "COEFFICIENT_OUT_OF_RANGE" and EXTREMES[n]["status_want"] == 6
        hj = HostJpeg(read_golden(EXTREMES[n]["path"]))
        assert hj.status == 0, n
        assert [r[0] for r in oracle_encode_image(hj.coef_image())] == [6], n


# every place where the reference's arithmetic wraps, truncates or caps (oracle/lepton_oracle.c, "regime counters")
REGIME_SITES = ["idct_int32_wrap", "idct_int16_pixel", "dc_est_int16", "edge_int16", "qdc_int16", "lak_uint32_wrap",
                "sign_ctx_int16", "thr_ctx_mask", "thr_ctx_cap255", "bsr_cap1023", "len_mxm_cap11", "thr_so_sat127",
                "adv_wrap_pos", "adv_wrap_neg", "ac_len11", "refuse_dc", "refuse_dc_len", "refuse_ac"]


def test_extreme_corpus_reaches_every_wrap_and_cap_site():
    """The oracle computes each wrapped or capped value exactly as well and counts where the two differ.  Coding the
    extreme corpus has to reach every such site several times -- so a regenerated corpus cannot drift back into the range
    photos live in, where a wrong cast, mask or division domain in the kernels would go unnoticed -- while the golden
    photos reach almost none of them."""
    from lepton_b200 import HostJpeg
    assert sorted(oracle.regime_counts(reset=True)) == sorted(REGIME_SITES)
    for n in extreme_jpegs():
        oracle_encode_image(HostJpeg(read_golden(EXTREMES[n]["path"])).coef_image())
    for name, _ in extreme_leps():
        oracle_decode_planes(load_extreme_lep(name))
    hit = oracle.regime_counts(reset=True)
    assert all(hit[k] >= 3 for k in REGIME_SITES if not k.startswith("refuse")), hit
    assert hit["refuse_dc"] >= 1 and hit["refuse_dc_len"] >= 1 and hit["refuse_ac"] >= 1, hit
    for name in golden_leps():
        oracle_decode_planes(load_lep(name))
    photo = oracle.regime_counts(reset=True)
    assert sum(photo[k] > 0 for k in REGIME_SITES) <= 3, photo


def _div_trunc_small_f32(n, d):
    """lep_predict.cuh div_trunc_small in numpy float32: __uint2float_rz of |n| and d (exact below 2^24), __frcp_rn
    (the correctly rounded reciprocal), a round-to-nearest product truncated to an integer, one correction each way."""
    a = np.abs(n).astype(np.int64)
    rcp = np.float32(1) / d.astype(np.float32)
    q = (a.astype(np.float32) * rcp).astype(np.int64)
    rem = a - q * d
    q = np.where(rem < 0, q - 1, q)
    rem = np.where(rem < 0, rem + d, rem)
    q = np.where(rem >= d, q + 1, q)
    return np.where(n < 0, -q, q)


def test_div_trunc_small_is_exact_over_the_callers_domain():
    """div_trunc_small claims exact truncating division for |n| < 2^24, 1 <= d < 2^16 with a float reciprocal and one
    correction step.  Its callers divide |avgmed| <= 2^18 (sums of eight int16 estimates) by q0 and |t| <= 2^18 (a 32-bit
    sum shifted right by 13) by a quantiser.  Checked for every d < 2^16 at n = k d - 1, k d, k d + 1 for every multiple
    k d up to 2^20, and at the multiples just below 2^24, both signs."""
    for lo in range(1, 1 << 16, 4096):
        d = np.arange(lo, min(lo + 4096, 1 << 16), dtype=np.int64)
        for top in (1 << 20, 1 << 24):
            kmax = top // d
            kmin = np.maximum(kmax - 8, 1) if top == 1 << 24 else np.ones_like(d)
            cnt = kmax - kmin + 1
            dd = np.repeat(d, cnt)
            k = np.repeat(kmin - np.cumsum(np.r_[0, cnt[:-1]]), cnt) + np.arange(cnt.sum())
            n = (k * dd)[:, None] + np.array([-1, 0, 1])
            dd = np.broadcast_to(dd[:, None], n.shape).ravel()
            n = n.ravel()
            keep = np.abs(n) < (1 << 24)
            n, dd = n[keep], dd[keep]
            for sgn in (1, -1):
                got = _div_trunc_small_f32(sgn * n, dd)
                want = sgn * (n // dd)
                bad = np.nonzero(got != want)[0]
                assert bad.size == 0, (int(sgn * n[bad[0]]), int(dd[bad[0]]), int(got[bad[0]]))
