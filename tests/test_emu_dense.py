"""The dense corpus (tests/golden/dense/, white noise at quality 100: every thread-segment needs more range-coder stream
than the 64 bytes per block plus 4 KB it starts with) through the emulated kernels, against the reference's streams,
planes and scans; and random noise planes against the oracle."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu  # noqa: E402
import lepfmt  # noqa: E402
from helpers import (DENSE, coef_image_from_lep, dense_jpegs, dense_leps, load_dense_lep, oracle_decode_planes,  # noqa: E402
                     oracle_encode_image, plane_hashes, random_coef_image, read_golden)

KERNELS = [0, 1, 2]          # range coder: parallel, serial, parallel with the register token feed


def dense_batch():
    """Every .lep record of the dense corpus as the encoder gets it -> (images, reference streams per image, names)."""
    imgs, want, names = [], [], []
    for name, source in dense_leps():
        lf = load_dense_lep(name)
        planes, streams = oracle_decode_planes(lf)
        imgs.append(coef_image_from_lep(lf, planes))
        want.append(list(streams[:lf.nseg]))
        names.append((name, source))
    return imgs, want, names


def test_corpus_outgrows_the_initial_stream_slot():
    """What makes the corpus worth having: every segment's reference stream is longer than its initial slot."""
    for name, _ in dense_leps():
        e = DENSE[name if name in DENSE else name[:-4] + ".jpg"]
        lf = load_dense_lep(name)
        streams = lepfmt.demux(lf.payload, lf.version)[:lf.nseg]
        assert [len(s) for s in streams] == e["seg_stream_bytes"], name
        assert all(n > s for n, s in zip(e["seg_stream_bytes"], e["seg_slot_bytes"])), name
        assert e["min_margin"] > 1, name


@pytest.mark.parametrize("kernel", KERNELS)
def test_dense_batch_encode_matches_reference_streams(kernel):
    """Kernel A + B over the whole corpus in one batch, three persistent CTAs: the reference's streams (status 100
    before the streams could grow past their slot)."""
    imgs, want, names = dense_batch()
    got = emu.encode_images(imgs, grid_cap=3, kernel=kernel)
    for (name, _), g, w in zip(names, got, want):
        assert [x[0] for x in g] == [0] * len(w), name
        assert [x[1] for x in g] == w, name


def test_token_bounds_cover_the_decisions():
    """The token bound of every segment -- the count pre-pass's, and the one the GPU Huffman decoder's row counters give
    (start_tok in lep_file.cc) -- is at least the number of decisions the oracle codes."""
    imgs, _, names = dense_batch()
    res, caps = emu.encode_images(imgs, kernel=0, tok_caps=True)
    k = 0
    for img, r, (name, source) in zip(imgs, res, names):
        ref = oracle_encode_image(img)
        for (rc, _, nd), (st, _, gnd) in zip(ref, r):
            assert rc == 0 and st == 0 and gnd == nd, name
            assert caps[k] >= nd + 64, (name, caps[k], nd)
            k += 1
    # the Huffman decoder's counters: decisions of the rows of each segment of the single-segment records
    jpegs = [read_golden(DENSE[n]["path"]) for n in dense_jpegs()]
    huff, _ = emu.huffman_decode(emu.HUFF_SERIAL, jpegs)
    for n, h in zip(dense_jpegs(), huff):
        assert h is not None and h["status"] == 0, n
        lf = load_dense_lep(n[:-4] + ".lep")
        img = imgs[[x for x, _ in names].index(n[:-4] + ".lep")]
        ref = oracle_encode_image(img)
        rows = h["rows"]
        for t, hd in enumerate(lf.handoffs):
            r0 = next(i for i, row in enumerate(rows) if row[2] * (img.bcv[0] // img.mcuv) >= hd.luma_y_start)
            r1 = next((i for i, row in enumerate(rows) if t + 1 < len(lf.handoffs) and
                       row[2] * (img.bcv[0] // img.mcuv) >= lf.handoffs[t + 1].luma_y_start), len(rows) - 1)
            bound = max(1, rows[r1][3] - rows[r0][3])
            assert bound >= ref[t][2], (n, t, bound, ref[t][2])


@pytest.mark.parametrize("kernel", [emu.KERNEL_WARP] + [pytest.param(emu.KERNEL_G2(g), marks=pytest.mark.slow) if g < 4
                                                        else emu.KERNEL_G2(g) for g in (1, 2, 4, 8, 16, 32)])
def test_dense_corpus_decodes_to_the_reference_planes(kernel):
    imgs, want, names = dense_batch()
    out = [coef_image_from_lep(load_dense_lep(n), [np.full_like(p, 77) for p in img.planes]) for img, (n, _) in zip(imgs, names)]
    st, _ = emu.decode_images(kernel, out, want, grid_cap=3)
    assert all(s == 0 for s in st), st
    for (name, source), img in zip(names, out):
        assert plane_hashes(img.planes) == DENSE[source]["plane_sha256"], name


@pytest.mark.parametrize("sub_bits", [1024, 4096])
def test_dense_jpegs_both_huffman_kernels_match_the_host_decoder(sub_bits):
    names = dense_jpegs()
    jpegs = [read_golden(DENSE[n]["path"]) for n in names]
    ser, _ = emu.huffman_decode(emu.HUFF_SERIAL, jpegs)
    par, _ = emu.huffman_decode(emu.HUFF_SUBSEQ, jpegs, sub_bits=sub_bits)
    for n, s, p in zip(names, ser, par):
        assert s is not None and p is not None and s["status"] == 0 and p["status"] == 0, n
        for got, want in zip(s["planes"], s["host_planes"]):
            assert np.array_equal(got, want), n
        for got, want in zip(p["planes"], s["planes"]):
            assert np.array_equal(got, want), n
        assert (p["padbit"], p["end_bitpos"], p["rows"]) == (s["padbit"], s["end_bitpos"], s["rows"]), n


def test_huffman_encode_kernel_recreates_the_dense_scans():
    from lepton_b200 import HostJpeg, HostLep
    for name, source in dense_leps():
        jpg = read_golden(DENSE[source]["path"])
        hl = HostLep(read_golden("dense/" + name))
        assert hl.status == 0, hl.error
        off, n = hl.scan_layout()
        job = emu.henc_job(hl)
        scan, segs = emu.huffman_encode(job, HostJpeg(jpg).coef_image())
        assert [st for st, _ in segs] == [0] * job.nseg, (name, segs)
        assert scan == jpg[off:off + n], name


def test_dense_leps_reassembled_by_the_gather_kernel():
    from test_emu_mux import split_lep
    names = [n for n, _ in dense_leps()]
    raws = [read_golden("dense/" + n) for n in names]
    got = emu.mux_files([split_lep(r) for r in raws], grid=3)
    for n, g, r in zip(names, got, raws):
        assert g == r, n


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("cfg", [
    dict(ncmp=1, mcuh=16, mcuv=32, sf=((1, 1),), nseg=1, noise="uniform", amp=1023),
    dict(ncmp=1, mcuh=32, mcuv=32, sf=((1, 1),), nseg=2, noise="gauss", amp=120),
    dict(ncmp=3, mcuh=12, mcuv=12, sf=((2, 2), (1, 1), (1, 1)), nseg=1, noise="uniform", amp=700),
])
def test_random_noise_planes_encode_vs_oracle(kernel, cfg):
    """iid noise at every AC position, 512 blocks or more per segment (so the 4 KB of slack cannot hide the stream's
    length): the oracle's streams and decision counts, and every stream is longer than its initial slot."""
    rng = np.random.default_rng(2468)
    img = random_coef_image(rng, **cfg)
    ref = oracle_encode_image(img)
    got = emu.encode_images([img], kernel=kernel)[0]
    nb = img.blocks() // len(ref)
    assert nb >= 512
    for g, r in zip(got, ref):
        assert r[0] == 0 and len(r[1]) > nb * 64 + 4096
        assert (g[0], g[1], g[2]) == r
