"""zlib0 output on the GPU: .lep files restored as zlib streams of stored blocks (-zlib0, and containers with the zeta magic
CE B6) through the file API and the CLI, against what the unmodified reference CLI wrote (tests/golden/zlib0.json,
tests/golden/make_zlib0.py)."""
import hashlib
import json
import os
import subprocess
import sys
import zlib

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from helpers import GOLDEN, read_golden  # noqa: E402
from make_zlib0 import sweep_jpeg, zeta  # noqa: E402

pytestmark = pytest.mark.gpu

ZLIB0 = json.load(open(os.path.join(GOLDEN, "zlib0.json")))
LEPS = sorted(ZLIB0["leps"])
EXE = os.path.join(os.path.dirname(GOLDEN), "..", "lepton_b200", "bin", "lepton-b200")


def md5(b):
    return hashlib.md5(b).hexdigest()


def brotli():
    from lepton_b200 import lib
    return lib().lepb200_host_brotli_available() == 1


def check_blocks(z, n):
    """78 01, stored blocks of 65535 bytes, the last one BFINAL and not empty, then 4 bytes: 2 + n + 5 ceil(n / 65535) + 4."""
    assert z[:2] == b"\x78\x01" and len(z) == 2 + n + 5 * -(-n // 65535) + 4
    p, got = 2, 0
    while True:
        ln = int.from_bytes(z[p + 1:p + 3], "little")
        assert z[p] == (1 if got + ln == n else 0) and ln == min(65535, n - got) and ln > 0
        assert int.from_bytes(z[p + 3:p + 5], "little") == ln ^ 0xFFFF
        p += 5 + ln
        got += ln
        if got == n:
            break
    assert p + 4 == len(z)


def check_against_reference(rel, plain, got, ref):
    """got = (status, bytes) with zlib0 output; plain = (status, bytes) of the same file without it."""
    assert got[0] == plain[0], (rel, got[0], plain[0])
    if plain[0] != 0:
        # the one file the reference restores and this build may refuse: a brotli header blob on a host without libbrotlidec
        assert ref["rc"] != 0 or (rel == "future/narrowrst.lep" and plain[0] == 200 and not brotli()), (rel, plain[0], ref)
        return
    assert zlib.decompress(got[1]) == plain[1], rel
    check_blocks(got[1], len(plain[1]))
    if ref["rc"] == 0 and ref["exit_name"] is None:
        assert md5(got[1]) == ref["md5"] and len(got[1]) == ref["size"], rel
    else:
        # the reference's own decoder refuses a few truncated multi-segment records that this build restores
        assert rel.startswith("truncated/") and "_t" in rel, rel


@pytest.mark.parametrize("gpu_huffman,parts", [(True, "1"), (True, "4"), (False, "4")])
def test_file_api_matches_reference(monkeypatch, gpu_huffman, parts):
    """Every committed .lep restored with zlib0=True, and its zeta copy restored with and without it, gives the reference's
    -zlib0 bytes, in one batch of 388 files (large enough for the device re-encode to run in parts); tau files of the same
    batch stay plain JPEGs.  Statuses are those of the plain restore."""
    from lepton_b200 import LeptonB200FileCodec
    monkeypatch.setenv("LEPB200_HENC_PARTS", parts)
    leps = [read_golden(r) for r in LEPS]
    zetas = [zeta(l) for l in leps]
    fp = LeptonB200FileCodec(0, host_threads=8, gpu_huffman=gpu_huffman)
    fz = LeptonB200FileCodec(0, host_threads=8, gpu_huffman=gpu_huffman, zlib0=True)
    try:
        plain = fp.decompress(leps)
        plain_recoded = fp.last_gpu_recoded
        both = fz.decompress(leps + zetas)
        z_recoded = fz.last_gpu_recoded
        mixed = fp.decompress(leps + zetas)
    finally:
        fp.close()
        fz.close()
    n = len(leps)
    for k, rel in enumerate(LEPS):
        ref = ZLIB0["leps"][rel]
        assert ref["plain"] == ref["zeta"], rel
        check_against_reference(rel, plain[k], both[k], ref["plain"])
        check_against_reference(rel, plain[k], both[n + k], ref["zeta"])
        check_against_reference(rel, plain[k], mixed[n + k], ref["zeta"])
        assert mixed[k] == plain[k], rel
    if gpu_huffman:
        assert plain_recoded > 100 and z_recoded == 2 * plain_recoded, (plain_recoded, z_recoded)
    else:
        assert z_recoded == 0


def test_length_sweep_through_the_library():
    """The sweep's JPEGs (one block; one byte short of, at and past one and two blocks; three full blocks) compress to the
    reference's .lep and come back as the reference's -zlib0 bytes, on the device re-encode path."""
    from lepton_b200 import LeptonB200FileCodec
    jpegs = [sweep_jpeg(r["total"]) for r in ZLIB0["sweep"]]
    fz = LeptonB200FileCodec(0, host_threads=4, zlib0=True)
    try:
        leps = fz.compress(jpegs)
        assert [md5(l) for _, l in leps] == [r["lep_md5"] for r in ZLIB0["sweep"]]
        back = fz.decompress([l for _, l in leps])
        assert fz.last_gpu_recoded == len(jpegs)
    finally:
        fz.close()
    for r, j, (st, z) in zip(ZLIB0["sweep"], jpegs, back):
        assert st == 0 and md5(z) == r["zlib0_md5"] and zlib.decompress(z) == j, r["total"]


def test_damaged_files_keep_their_status():
    """A batch of tau files, zeta files and damaged ones of both kinds: with zlib0 every file has the status it has without."""
    from lepton_b200 import LeptonB200FileCodec
    base = [read_golden(r) for r in ("android.lep", "androidprogressive.lep", "extremes/odd_rst_t4.lep", "grayscale.lep")]
    damaged = []
    for l in base:
        damaged += [l[:len(l) // 2], l[:40], l[:-9] + l[-4:], l[:len(l) - 200] + bytes(196) + l[-4:]]
    tau = base + damaged
    batch = tau + [zeta(l) for l in tau]
    fp = LeptonB200FileCodec(0, host_threads=4)
    fz = LeptonB200FileCodec(0, host_threads=4, zlib0=True)
    try:
        plain = fp.decompress(tau)
        got = fz.decompress(batch)
        mixed = fp.decompress(batch)
    finally:
        fp.close()
        fz.close()
    want = [st for st, _ in plain] * 2
    assert [st for st, _ in got] == want
    assert [st for st, _ in mixed] == want
    assert any(want) and want.count(0) >= 8
    for (st, j), (_, z) in zip(plain * 2, got):
        if st == 0:
            assert zlib.decompress(z) == j


def run(args, **kw):
    return subprocess.run([EXE] + args, capture_output=True, **kw)


def test_cli_single_file_stdin_and_default_names(tmp_path):
    """-zlib0 and zeta inputs in single-file mode: explicit output, default <stem>.jpg.z, and stdin to stdout."""
    assert os.path.exists(EXE), "build() did not produce the CLI"
    for rel in ("android.lep", "iphoneprogressive.lep", "extremes/color420_long_t8.lep"):
        lep = read_golden(rel)
        want = ZLIB0["leps"][rel]["plain"]["md5"]
        t, z = tmp_path / "t.lep", tmp_path / "z.lep"
        t.write_bytes(lep)
        z.write_bytes(zeta(lep))
        r = run(["-zlib0", str(t), str(tmp_path / "o1")])
        assert r.returncode == 0 and md5((tmp_path / "o1").read_bytes()) == want, (rel, r.stderr)
        r = run(["-zlib0", str(t)])
        assert r.returncode == 0 and md5((tmp_path / "t.jpg.z").read_bytes()) == want, (rel, r.stderr)
        r = run([str(z)])
        assert r.returncode == 0 and md5((tmp_path / "z.jpg.z").read_bytes()) == want, (rel, r.stderr)
        r = run(["-zlib0", "-"], input=lep)
        assert r.returncode == 0 and md5(r.stdout) == want, rel
        r = run(["-", "-"], input=zeta(lep))
        assert r.returncode == 0 and md5(r.stdout) == want, rel
        r = run([str(t)])                                           # tau without the flag: a plain JPEG, as before
        assert r.returncode == 0 and (tmp_path / "t.jpg").exists() and (tmp_path / "t.jpg").read_bytes()[:2] == b"\xff\xd8"
        for f in ("t.jpg", "t.jpg.z", "z.jpg.z", "o1"):
            (tmp_path / f).unlink()


def test_cli_batch_mode(tmp_path):
    """Batch mode: tau files become DIR/<name>.jpg.z with -zlib0, zeta files always; JPEG inputs still give the .lep."""
    out = tmp_path / "out"
    out.mkdir()
    names = ["android.lep", "grayscale.lep", "iphonecrop2_t8.lep"]
    for n in names:
        (tmp_path / n).write_bytes(read_golden(n))
        (tmp_path / ("z_" + n)).write_bytes(zeta(read_golden(n)))
    ins = [str(tmp_path / n) for n in names] + [str(tmp_path / ("z_" + n)) for n in names]
    r = run(["-outdir=" + str(out)] + ins + [os.path.join(GOLDEN, "androidcrop.jpg")])
    assert r.returncode == 0, r.stderr
    for n in names:
        want = ZLIB0["leps"][n]["plain"]["md5"]
        assert (out / (n[:-4] + ".jpg")).read_bytes()[:2] == b"\xff\xd8"
        assert md5((out / ("z_" + n[:-4] + ".jpg.z")).read_bytes()) == want, n
    assert (out / "androidcrop.lep").read_bytes() == read_golden("androidcrop.lep")
    out2 = tmp_path / "out2"
    out2.mkdir()
    r = run(["-zlib0", "-outdir=" + str(out2)] + ins)
    assert r.returncode == 0, r.stderr
    for n in names:
        want = ZLIB0["leps"][n]["plain"]["md5"]
        assert md5((out2 / (n[:-4] + ".jpg.z")).read_bytes()) == want, n
        assert md5((out2 / ("z_" + n[:-4] + ".jpg.z")).read_bytes()) == want, n


def test_cli_zlib0_on_jpeg_input_writes_the_reference_lep(tmp_path):
    """The JPEG -> .lep direction ignores -zlib0 (with the default verification and with -skipverify)."""
    for name in ("android.jpg", "iphoneprogressive.jpg", "gray2sf.jpg"):
        for flags in ([], ["-skipverify"]):
            dst = tmp_path / "o.lep"
            r = run(["-zlib0"] + flags + [os.path.join(GOLDEN, name), str(dst)])
            assert r.returncode == 0, (name, r.stderr)
            assert dst.read_bytes() == read_golden(name[:-4] + ".lep"), name
            dst.unlink()
