"""JPEGs embedded in larger files (-embedding=N) and -d on the GPU, through the file API and the CLI, against what the
unmodified reference CLI did with every case of tests/golden/embedded.json (tests/golden/make_embedded.py)."""
import hashlib
import json
import os
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from helpers import GOLDEN, read_golden  # noqa: E402
from make_embedded import LEP_FIXTURES, case_bytes, embedding_of, expected_status  # noqa: E402

pytestmark = pytest.mark.gpu

EMB = json.load(open(os.path.join(GOLDEN, "embedded.json")))
CASES = sorted(EMB["cases"])
EXE = os.path.join(os.path.dirname(GOLDEN), "..", "lepton_b200", "bin", "lepton-b200")
THREADS = {"skipverify": 1, "t4": 4, "t8": 8}


def md5(b):
    return hashlib.md5(b).hexdigest()


def groups():
    """Cases by their flags: the codec settings apply to a whole call, as the reference's flags to one invocation."""
    out = {}
    for n in CASES:
        out.setdefault(tuple(EMB["cases"][n]["flags"]), []).append(n)
    return out


def compress_all(run, gpu_huffman, verify=False):
    """{case: (status, .lep)} for every case, one call per group of equal flags."""
    from lepton_b200 import LeptonB200FileCodec
    got = {}
    for flags, names in groups().items():
        off, discard = embedding_of(list(flags))
        fc = LeptonB200FileCodec(0, host_threads=8, gpu_huffman=gpu_huffman, min_encode_threads=THREADS.get(run, 1),
                                 verify=verify, embedding=off, discard_meta=discard)
        try:
            for n, r in zip(names, fc.compress([case_bytes(n) for n in names])):
                got[n] = r
        finally:
            fc.close()
    return got


def verify_status(e):
    """The status with verification on: the reference's, except that a file the coder refuses keeps the coder's status
    (the reference reports 41 for it, its verification having nothing to compare)."""
    r = e["verify"]
    if r["rc"] == 0 and r["lep_md5"]:
        return 0
    if r["names"][:1] == ["ROUNDTRIP_FAILURE"]:
        return 41
    return expected_status(e["skipverify"])


@pytest.mark.parametrize("gpu_huffman", [True, False])
@pytest.mark.parametrize("run", sorted(THREADS))
def test_file_api_compresses_like_the_reference(run, gpu_huffman):
    """Every case compresses to the reference's .lep md5 and status, with the device or the host Huffman decoder."""
    got = compress_all(run, gpu_huffman)
    for n in CASES:
        r = EMB["cases"][n][run]
        st, lep = got[n]
        assert st == expected_status(r), (n, run, st, r)
        if st == 0:
            assert md5(lep) == r["lep_md5"], (n, run)


def test_file_api_with_verification():
    """Verification compares the whole input, prefix and trailer included: the progressive file behind a prefix and every
    -d file fail with 41, as with the reference; the rest are written."""
    got = compress_all("verify", True, verify=True)
    for n in CASES:
        e = EMB["cases"][n]
        st, lep = got[n]
        assert st == verify_status(e), (n, st, e["verify"])
        if st == 0:
            assert md5(lep) == e["verify"]["lep_md5"], n
    assert got["prog_p500"][0] == 41 and got["d_android"][0] == 41 and got["android.jpg_p70000_t1"][0] == 0


@pytest.mark.parametrize("gpu_huffman", [True, False])
def test_restore_every_case(gpu_huffman):
    """Every .lep restores to what the reference restores from it -- the input, except for the progressive file (its
    prefix is dropped) and the -d files (their metadata is gone) -- plainly and with zlib0.  The device re-encode takes
    the complete baseline files with a prefix; the host re-encoders take the truncated, progressive and -d ones."""
    from lepton_b200 import LeptonB200FileCodec
    names = [n for n in CASES for run in THREADS if EMB["cases"][n][run].get("restore")]
    runs = [run for n in CASES for run in THREADS if EMB["cases"][n][run].get("restore")]
    got = {}
    for run in THREADS:
        for n, r in compress_all(run, True).items():
            got[(n, run)] = r
    leps = [got[(n, run)][1] for n, run in zip(names, runs)]
    fp = LeptonB200FileCodec(0, host_threads=8, gpu_huffman=gpu_huffman)
    fz = LeptonB200FileCodec(0, host_threads=8, gpu_huffman=gpu_huffman, zlib0=True)
    try:
        plain = fp.decompress(leps)
        recoded = fp.last_gpu_recoded
        zl = fz.decompress(leps)
    finally:
        fp.close()
        fz.close()
    device = 0
    for n, run, (st, j), (zst, z) in zip(names, runs, plain, zl):
        rec = EMB["cases"][n][run]
        assert st == 0 and md5(j) == rec["restore"]["md5"], (n, run, st)
        assert zst == 0 and md5(z) == rec["restore_zlib0"]["md5"], (n, run, zst)
        if not (n.startswith(("d_", "prog", "trunc"))):
            assert j == case_bytes(n), (n, run)
            device += 1
    assert recoded == (device if gpu_huffman else 0), (recoded, device)


def test_restore_the_reference_files():
    """The .lep files the reference wrote with -embedding come back as it restores them."""
    from lepton_b200 import LeptonB200FileCodec
    leps = [read_golden("embedded/%s.lep" % n) for n in LEP_FIXTURES]
    fc = LeptonB200FileCodec(0, host_threads=4)
    try:
        back = fc.decompress(leps)
    finally:
        fc.close()
    for n, (st, j) in zip(LEP_FIXTURES, back):
        assert st == 0 and md5(j) == EMB["cases"][n]["skipverify"]["restore"]["md5"], (n, st)


def run_cli(args, **kw):
    return subprocess.run([EXE] + args, capture_output=True, **kw)


def test_cli_single_file(tmp_path):
    """-embedding=N and -d in single-file mode give the reference CLI's bytes and statuses (verification on by default)."""
    assert os.path.exists(EXE), "build() did not produce the CLI"
    for n in ("android.jpg_p4096_t1", "trailingrst.jpg_p1_t0", "android.jpg_e0", "d_android", "d_emb_androidcropoptions",
              "prog_p500", "notsoi_p1001", "past_end", "lep_e5", "plain_e2", "trunc_p1001"):
        e = EMB["cases"][n]
        src, dst, back = tmp_path / "in.bin", tmp_path / "o.lep", tmp_path / "b.jpg"
        src.write_bytes(case_bytes(n))
        for key, extra in (("skipverify", ["-skipverify"]), ("verify", [])):
            if dst.exists():
                dst.unlink()
            r = run_cli(e["flags"] + extra + [str(src), str(dst)])
            want = expected_status(e[key]) if key == "skipverify" else verify_status(e)
            assert r.returncode == want, (n, key, r.returncode, r.stderr)
            if want == 0:
                assert md5(dst.read_bytes()) == e[key]["lep_md5"], (n, key)
                r = run_cli([str(dst), str(back)])
                assert r.returncode == 0 and md5(back.read_bytes()) == e["skipverify"]["restore"]["md5"], (n, r.stderr)
    # default output name: <stem>.lep, whatever the input's first bytes
    src = tmp_path / "wrapped.bin"
    src.write_bytes(case_bytes("android.jpg_p255_t0"))
    r = run_cli(["-embedding=255", str(src)])
    assert r.returncode == 0 and md5((tmp_path / "wrapped.lep").read_bytes()) == EMB["cases"]["android.jpg_p255_t0"]["verify"]["lep_md5"]


def test_cli_batch_mode(tmp_path):
    """Batch mode with -embedding=N takes every input as a JPEG: the embedded files give the reference's .lep, a .lep in the
    same batch is refused as the reference refuses it; the .lep files then restore in one batch.  -d in batch mode too."""
    out, back = tmp_path / "out", tmp_path / "back"
    out.mkdir()
    back.mkdir()
    names = ["android.jpg_p255_t0", "android.jpg_p255_t1", "trailingrst.jpg_p255_t1", "grayscale.jpg_p255_t0"]
    for n in names:
        (tmp_path / (n + ".bin")).write_bytes(case_bytes(n))
    (tmp_path / "other.lep").write_bytes(read_golden("android.lep"))
    r = run_cli(["-embedding=255", "-outdir=" + str(out)] + [str(tmp_path / (n + ".bin")) for n in names] + [str(tmp_path / "other.lep")])
    assert r.returncode == 42, (r.returncode, r.stderr)                 # UNSUPPORTED_JPEG, as the reference says for it
    for n in names:
        assert md5((out / (n + ".lep")).read_bytes()) == EMB["cases"][n]["verify"]["lep_md5"], n
    assert not (out / "other.lep").exists() and not (out / "other.jpg").exists()
    (out / "plain.lep").write_bytes(read_golden("android.lep"))
    r = run_cli(["-outdir=" + str(back)] + [str(out / (n + ".lep")) for n in names] + [str(out / "plain.lep")])
    assert r.returncode == 0, r.stderr
    for n in names:
        assert (back / (n + ".jpg")).read_bytes() == case_bytes(n), n
    assert (back / "plain.jpg").read_bytes() == read_golden("android.jpg")
    dd = tmp_path / "d"
    dd.mkdir()
    r = run_cli(["-d", "-skipverify", "-outdir=" + str(dd)] + [os.path.join(GOLDEN, s + ".jpg") for s in ("android", "iphonecrop2")])
    assert r.returncode == 0, r.stderr
    for s in ("android", "iphonecrop2"):
        assert md5((dd / (s + ".lep")).read_bytes()) == EMB["cases"]["d_" + s]["skipverify"]["lep_md5"], s
