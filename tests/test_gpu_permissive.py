"""-permissive on the GPU, through the file API, the _multi entry and the CLI, against what the unmodified reference CLI
did with every case of tests/golden/permissive.json (tests/golden/make_permissive.py): the files the coder cannot take come
out in the generic container and restore byte for byte, while the ordinary JPEGs of the same batch keep their device
path, their bytes and their device re-encode."""
import hashlib
import json
import os
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from helpers import GOLDEN, read_golden  # noqa: E402
from make_permissive import LEP_FIXTURES, case_bytes  # noqa: E402

pytestmark = pytest.mark.gpu

PERM = json.load(open(os.path.join(GOLDEN, "permissive.json")))
CASES = sorted(PERM["cases"])
EXE = os.path.join(os.path.dirname(GOLDEN), "..", "lepton_b200", "bin", "lepton-b200")
# ordinary JPEGs with the reference's .lep beside them: baseline (device Huffman decode and re-encode), progressive (host
# Huffman paths), restart markers, greyscale
NORMAL = ["android", "androidcrop", "androidtrail", "colorswap", "grayscale", "iphonecrop2", "trailingrst", "trailingrst2",
          "androidprogressive", "iphoneprogressive"]


def md5(b):
    return hashlib.md5(b).hexdigest()


def settings(flags):
    off = [int(f.split("=")[1]) for f in flags if f.startswith("-embedding=")]
    return {"embedding": off[0] if off else None, "discard_meta": "-d" in flags}


def groups():
    """Cases by their flags: the codec settings apply to a whole call, as the reference's flags to one invocation."""
    out = {}
    for n in CASES:
        out.setdefault(tuple(PERM["cases"][n]["flags"]), []).append(n)
    return out


def expected(case):
    r = PERM["cases"][case]["skipverify"]
    return (0, r["lep_md5"]) if r["rc"] == 0 else (r["rc"], None)


def mixed(names, flags=()):
    """The fixture cases interleaved with the ordinary JPEGs: (labels, inputs).  Only calls without -d / -embedding get
    ordinary JPEGs: with those flags they would be generic themselves (restored differently, or no SOI at the offset)."""
    labels, inputs = [], []
    normal = iter(NORMAL * 4)
    for n in names:
        for _ in range(2 if not flags else 0):
            k = next(normal)
            labels.append(("jpeg", k))
            inputs.append(read_golden(k + ".jpg"))
        labels.append(("case", n))
        inputs.append(case_bytes(n))
    return labels, inputs


def codec(**kw):
    from lepton_b200 import LeptonB200FileCodec
    return LeptonB200FileCodec(0, host_threads=8, **kw)


def compress_mixed(permissive=True):
    """{flags: (labels, results)} for one compress call per group of equal flags."""
    out = {}
    for flags, names in groups().items():
        labels, inputs = mixed(names, flags)
        fc = codec(permissive=permissive, **settings(flags))
        try:
            out[flags] = (labels, fc.compress(inputs))
        finally:
            fc.close()
    return out


@pytest.fixture(scope="module")
def compressed():
    return compress_mixed()


def test_compress_matches_reference_in_mixed_batches(compressed):
    seen = set()
    for flags, (labels, res) in compressed.items():
        for (kind, name), (st, lep) in zip(labels, res):
            if kind == "case":
                seen.add(name)
                assert (st, md5(lep) if st == 0 else None) == expected(name), (flags, name, st)
            else:
                assert st == 0 and lep == read_golden(name + ".lep"), (flags, name, st)
    assert seen == set(CASES)


def test_ordinary_files_unchanged_by_permissive(compressed):
    """The ordinary JPEGs, and the cases the coder takes, give the same bytes with and without the setting in the same
    batch; the other cases fail without it."""
    labels, inputs = mixed(groups()[()])
    fc = codec()
    try:
        plain = fc.compress(inputs)
    finally:
        fc.close()
    for (kind, name), a, b in zip(labels, compressed[()][1], plain):
        if kind == "jpeg" or PERM["cases"][name]["skipverify"]["flag"] == "Z":
            assert a == b and a[0] == 0, name
        elif name != "roundtripfail":                            # the one whose .lep only verification refuses
            assert b[0] != 0 and b[1] == b"", name


def test_decompress_mixed_batch_plain_and_zlib0(compressed):
    """Generic containers and coded .lep files restored in one call, plainly and as zlib0; the generic members take no
    device re-encode, so last_gpu_recoded and the coded files' bytes are those of a call without them."""
    from lepton_b200.codec import zlib0_frame
    leps, want, want_z, ordinary = [], [], [], []
    for labels, res in compressed.values():
        for (kind, name), (st, lep) in zip(labels, res):
            if st:
                continue
            leps.append(lep)
            if kind == "case":
                r = PERM["cases"][name]["skipverify"]
                want.append(r["restore"]["md5"])
                want_z.append(r["restore_zlib0"]["md5"])
            else:
                jpg = read_golden(name + ".jpg")
                want.append(md5(jpg))
                want_z.append(md5(zlib0_frame(jpg)))
            if kind == "jpeg" or r["flag"] != "Y":
                ordinary.append(len(leps) - 1)                   # a coded .lep: the device path
    for zlib0, w in ((False, want), (True, want_z)):
        fc = codec(zlib0=zlib0)
        try:
            got = fc.decompress(leps)
            recoded = fc.last_gpu_recoded
            assert [(st, md5(b)) for st, b in got] == [(0, x) for x in w], zlib0
            alone = fc.decompress([leps[i] for i in ordinary])
            assert fc.last_gpu_recoded == recoded > 0, zlib0
            assert alone == [got[i] for i in ordinary], zlib0
        finally:
            fc.close()


def test_reference_generic_files_restore_in_a_large_batch():
    """The reference's generic files among 256+ ordinary ones (the device re-encode then runs in parts): every file comes
    back, and the device re-encode count and the ordinary files' bytes are those of the ordinary files alone."""
    base = [read_golden(k + ".lep") for k in NORMAL]
    ordinary = (base * 24)[:256]
    generic = [read_golden("permissive/%s.lep" % n) for n in LEP_FIXTURES]
    batch = list(ordinary)
    for i, g in enumerate(generic):
        batch.insert(37 * i + 5, g)
    fc = codec()
    try:
        alone = fc.decompress(ordinary)
        n_alone = fc.last_gpu_recoded
        got = fc.decompress(batch)
        assert fc.last_gpu_recoded == n_alone > 0
    finally:
        fc.close()
    gi = [batch.index(g) for g in generic]
    for n, i in zip(LEP_FIXTURES, gi):
        assert got[i] == (0, case_bytes(n)), n
    assert [r for i, r in enumerate(got) if i not in gi] == alone


def test_multi_on_one_device():
    from lepton_b200 import LeptonB200MultiGpuFileCodec
    names = groups()[()]
    labels, inputs = mixed(names)
    mc = LeptonB200MultiGpuFileCodec([0], host_threads_per_gpu=8, permissive=True)
    try:
        res = mc.compress(inputs)
    finally:
        mc.close()
    for (kind, name), (st, lep) in zip(labels, res):
        if kind == "case":
            assert (st, md5(lep) if st == 0 else None) == expected(name), name
        else:
            assert st == 0 and lep == read_golden(name + ".lep"), name


def cli(args, **kw):
    return subprocess.run([EXE] + args, capture_output=True, **kw)


def test_cli_single_file_and_stdin(tmp_path):
    assert os.path.exists(EXE), "build() did not produce the CLI"
    for name in ("one_byte", "two_bytes", "blob70k", "badzerorun", "android_lep", "androidcrop", "empty"):
        src, lep, back = tmp_path / (name + ".bin"), tmp_path / (name + ".lep"), tmp_path / (name + ".back")
        data = case_bytes(name)
        src.write_bytes(data)
        r = PERM["cases"][name]["verify"]
        p = cli(["-permissive", str(src), str(lep)])
        assert p.returncode == r["rc"], (name, p.returncode, p.stderr)
        if r["rc"]:
            assert not lep.exists()
            continue
        assert md5(lep.read_bytes()) == r["lep_md5"], name
        p = cli([str(lep), str(back)])
        assert p.returncode == 0 and md5(back.read_bytes()) == r["restore"]["md5"], name
        p = cli(["-zlib0", str(lep), "-"])
        assert p.returncode == 0 and md5(p.stdout) == r["restore_zlib0"]["md5"], name
        p = cli(["-permissive", "-skipverify", "-"], input=data)
        assert p.returncode == 0 and md5(p.stdout) == r["lep_md5"], name
    p = cli([str(tmp_path / "one_byte.bin"), str(tmp_path / "x.lep")])
    assert p.returncode == 3                                     # without -permissive: SHORT_READ as before


def test_cli_outdir(tmp_path):
    names = ["one_byte", "blob70k", "roundtripfail", "android_lep", "androidcrop", "trunc_head", "empty"]
    srcs = []
    for n in names:
        f = tmp_path / (n + ".in")
        f.write_bytes(case_bytes(n))
        srcs.append(str(f))
    out = tmp_path / "out"
    out.mkdir()
    p = cli(["-permissive", "-outdir=%s" % out] + srcs)
    assert p.returncode == 42 and b"empty.in: exit code 42" in p.stderr, p.stderr   # the empty input: no container
    for n in names:
        f = out / (n + ".lep")
        r = PERM["cases"][n]["verify"]
        if r["rc"]:
            assert not f.exists()
        else:
            assert md5(f.read_bytes()) == r["lep_md5"], n
    back = tmp_path / "back"
    back.mkdir()
    leps = [str(out / (n + ".lep")) for n in names if n != "empty"]
    p = cli(["-outdir=%s" % back] + leps)
    assert p.returncode == 0, p.stderr
    for n in names:
        if n != "empty":
            assert (back / (n + ".jpg")).read_bytes() == case_bytes(n), n
