"""Streams of concatenated .lep files on the GPU, through the file API and the CLI, against what the unmodified reference
CLI restored from every case of tests/golden/concat.json (tests/golden/make_concat.py)."""
import hashlib
import json
import os
import subprocess
import sys
import zlib

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from helpers import GOLDEN, read_golden  # noqa: E402
from make_concat import case_bytes, expected, member  # noqa: E402

pytestmark = pytest.mark.gpu

CON = json.load(open(os.path.join(GOLDEN, "concat.json")))
CASES = sorted(CON["cases"])
EXE = os.path.join(os.path.dirname(GOLDEN), "..", "lepton_b200", "bin", "lepton-b200")
ORDINARY = ["android.lep", "androidprogressive.lep", "narrowrst.lep", "iphonecrop2_t8.lep"]     # version-1 single files


def md5(b):
    return hashlib.md5(b).hexdigest()


@pytest.fixture(autouse=True)
def brotli():
    from lepton_b200 import lib
    if not lib().lepb200_host_brotli_available():
        pytest.skip("libbrotlidec (libbrotlidec.so.1) not found: the version-2 members of concat.json cannot be read")


def ordinary_expected(key):
    """(status, md5) of the ordinary files, from a call with nothing but them."""
    from lepton_b200 import LeptonB200FileCodec
    fc = LeptonB200FileCodec(0, host_threads=8, zlib0=key == "zlib0")
    try:
        return [(st, md5(b)) for st, b in fc.decompress([read_golden(n) for n in ORDINARY])]
    finally:
        fc.close()


def check(got, key, names):
    for n, (st, out) in zip(names, got):
        want_st, want_md5 = expected(n, CON["cases"][n], key)
        assert st == want_st, (n, key, st)
        if want_md5:
            assert md5(out) == want_md5, (n, key)


@pytest.mark.parametrize("gpu_huffman", [True, False])
@pytest.mark.parametrize("key", ["plain", "zlib0"])
def test_file_api(key, gpu_huffman):
    """Every case in ONE call, between ordinary .lep files: the reference's md5 and status for each, plainly and as one zlib
    stream, with the device or the host re-encoder."""
    from lepton_b200 import LeptonB200FileCodec
    ords = ordinary_expected(key)
    inputs = [read_golden(ORDINARY[0])] + [case_bytes(CON["cases"][n]["parts"]) for n in CASES] + [read_golden(n) for n in ORDINARY[1:]]
    fc = LeptonB200FileCodec(0, host_threads=8, gpu_huffman=gpu_huffman, zlib0=key == "zlib0")
    try:
        got = fc.decompress(inputs)
        if gpu_huffman:
            assert fc.last_gpu_recoded > 0
    finally:
        fc.close()
    check(got[1:1 + len(CASES)], key, CASES)
    assert [(st, md5(b)) for st, b in [got[0]] + got[1 + len(CASES):]] == ords
    if key == "zlib0":
        e = CON["cases"]["embedded_doubled"]
        assert md5(zlib.decompress(got[1 + CASES.index("embedded_doubled")][1])) == e["jpeg_md5"]     # test_embedded.sh


def test_zeta_stream_without_the_setting():
    """A stream whose first member is CE B6 goes out as one zlib stream without -zlib0; a CE B6 member behind a CF 84 one
    ends the stream."""
    from lepton_b200 import LeptonB200FileCodec
    fc = LeptonB200FileCodec(0, host_threads=8)
    try:
        names = ["zeta_first", "zeta_second"]
        got = fc.decompress([case_bytes(CON["cases"][n]["parts"]) for n in names])
    finally:
        fc.close()
    assert got[0][0] == 0 and md5(got[0][1]) == CON["cases"]["zeta_first"]["plain"]["md5"]
    assert got[1][0] == 0 and md5(got[1][1]) == CON["cases"]["zeta_second"]["plain"]["md5"]


def run_cli(args, stdin=None):
    return subprocess.run([EXE] + args, input=stdin, capture_output=True)


def cli_status(st):
    return 42 if st == 200 else st


@pytest.mark.parametrize("key", ["plain", "zlib0"])
def test_cli_stdin(key):
    """`cat a.lep b.lep | lepton-b200 -`: the reference's stdout and exit code for every case."""
    assert os.path.exists(EXE), "build() did not produce the CLI"
    flags = ["-zlib0"] if key == "zlib0" else []
    for n in CASES:
        r = run_cli(flags + ["-"], case_bytes(CON["cases"][n]["parts"]))
        want_st, want_md5 = expected(n, CON["cases"][n], key)
        assert r.returncode == cli_status(want_st), (n, key, r.returncode, r.stderr[-400:])
        if want_md5:
            assert md5(r.stdout) == want_md5, (n, key)


def test_cli_single_file(tmp_path):
    """Single-file mode with an output name, and with the default one (<stem>.jpg, <stem>.jpg.z for zlib0)."""
    for n in ("pair_androidcrop_trailingrst2", "lepcat3", "embedded_doubled", "baseline_then_progressive"):
        src = tmp_path / (n + ".lep")
        src.write_bytes(case_bytes(CON["cases"][n]["parts"]))
        for key, flags, default in (("plain", [], n + ".jpg"), ("zlib0", ["-zlib0"], n + ".jpg.z")):
            want_st, want_md5 = expected(n, CON["cases"][n], key)
            dst = tmp_path / "out.bin"
            r = run_cli(flags + [str(src), str(dst)])
            assert r.returncode == cli_status(want_st), (n, key, r.returncode, r.stderr[-400:])
            if want_md5:
                assert md5(dst.read_bytes()) == want_md5, (n, key)
                r = run_cli(flags + [str(src)])
                assert r.returncode == 0 and md5((tmp_path / default).read_bytes()) == want_md5, (n, key)


@pytest.mark.parametrize("devices", [None, "-devices=0"])
@pytest.mark.parametrize("key", ["plain", "zlib0"])
def test_cli_batch(tmp_path, key, devices):
    """-outdir= batch mode (one library call) with every case and ordinary files; exit code = the first failure's."""
    out = tmp_path / "out"
    out.mkdir()
    paths = []
    for n in CASES:
        p = tmp_path / (n + ".lep")
        p.write_bytes(case_bytes(CON["cases"][n]["parts"]))
        paths.append(str(p))
    for n in ORDINARY:
        p = tmp_path / ("ord_" + n)
        p.write_bytes(read_golden(n))
        paths.append(str(p))
    flags = (["-zlib0"] if key == "zlib0" else []) + ([devices] if devices else [])
    r = run_cli(flags + ["-outdir=" + str(out)] + paths)
    assert r.returncode != 0                      # cut_in_second and the rest that fail
    suffix = ".jpg.z" if key == "zlib0" else ".jpg"
    for n in CASES:
        want_st, want_md5 = expected(n, CON["cases"][n], key)
        f = out / (n + (".jpg.z" if n == "zeta_first" else suffix))       # a CE B6 stream is always written as zlib
        if want_st:
            assert not f.exists(), n
            assert ("%s.lep: exit code %d" % (n, cli_status(want_st))) in r.stderr.decode(), n
        else:
            assert md5(f.read_bytes()) == want_md5, (n, key)
    for n, (st, m) in zip(ORDINARY, ordinary_expected(key)):
        assert st == 0 and md5((out / ("ord_" + n[:-4] + suffix)).read_bytes()) == m, n


def test_2048_members_share_batches():
    """A stream of 2 048 small reference .lep files restores byte for byte, with as many kernel launches as the same 2 048
    files passed as separate buffers: the members go through the same batches."""
    from lepton_b200 import LeptonB200FileCodec
    names = ["colorswap", "tall_t1", "tall_t4", "tall_t8", "narrowrst"]
    files = [member(names[i % len(names)]) for i in range(2048)]
    stream = b"".join(files)
    fc = LeptonB200FileCodec(0, host_threads=8)
    try:
        fc.decompress([stream])                                # warm-up: arenas and modules
        k0 = fc.kernel_launches
        sep = fc.decompress(files)
        k1 = fc.kernel_launches
        one = fc.decompress([stream])
        k2 = fc.kernel_launches
    finally:
        fc.close()
    for i, (st, b) in enumerate(sep):
        assert st == 0 and md5(b) == CON["members"][names[i % len(names)]]["jpeg_md5"], i
    assert one[0][0] == 0 and one[0][1] == b"".join(b for _, b in sep)
    assert k2 - k1 == k1 - k0, (k1 - k0, k2 - k1)
