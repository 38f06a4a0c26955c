"""-permissive on the host (CPU, no GPU): the generic container writer reproduces every generic .lep the unmodified
reference CLI wrote (tests/golden/permissive.json, tests/golden/make_permissive.py) byte for byte, system zlib's level 9
included; the .lep reader restores generic containers, plainly and as zlib0, to what the reference restores; files the
coder takes still give their ordinary .lep; and every 'Y' container other than the generic one stays refused with 200."""
import hashlib
import json
import os
import struct
import sys
import zlib

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from helpers import GOLDEN, oracle_encode_image, read_golden  # noqa: E402
from make_permissive import LEP_FIXTURES, case_bytes  # noqa: E402

PERM = json.load(open(os.path.join(GOLDEN, "permissive.json")))
CASES = sorted(PERM["cases"])
RUNS = sorted(PERM["runs"])
GENERIC = [c for c in CASES if PERM["cases"][c]["skipverify"]["flag"] == "Y"]
CODED = [c for c in CASES if PERM["cases"][c]["skipverify"]["flag"] in ("Z", "X")]


def md5(b):
    return hashlib.md5(b).hexdigest()


def generic(data):
    from lepton_b200.codec import generic_lep
    return generic_lep(data)


def test_cases_cover_the_ground():
    """Non-JPEGs of 1 B to 1 MB, damaged, arithmetic-coded and round-trip-failing JPEGs, .lep inputs, -d and a wrong
    -embedding offset all come out generic; good, truncated and embedded JPEGs come out coded; an empty input fails."""
    assert {"one_byte", "two_bytes", "blob70k", "blob1m", "badzerorun", "roundtripfail", "arithmetic_head",
            "android_lep", "gold_legacy_lep", "d_androidcropoptions", "emb5_androidcrop"} <= set(GENERIC)
    assert {"androidcrop", "trunc_head", "nofsync", "emb1001_android"} <= set(CODED)
    assert PERM["cases"]["empty"]["skipverify"]["rc"] == 42


@pytest.mark.parametrize("case", CASES)
def test_inputs_are_the_recorded_ones(case):
    e = PERM["cases"][case]
    data = case_bytes(case)
    assert (md5(data), len(data)) == (e["md5"], e["size"])


@pytest.mark.parametrize("run", RUNS)
@pytest.mark.parametrize("case", GENERIC)
def test_generic_writer_matches_reference(case, run):
    """The same container in every run: -skipverify and -maxencodethreads change nothing about it."""
    r = PERM["cases"][case][run]
    assert (r["rc"], r["flag"]) == (0, "Y")
    lep = generic(case_bytes(case))
    assert (md5(lep), len(lep)) == (r["lep_md5"], r["lep_size"]), (case, run)


def test_empty_input_has_no_container():
    assert generic(b"") == b""
    assert all(PERM["cases"]["empty"][run]["rc"] == 42 and PERM["cases"]["empty"][run]["lep_md5"] is None for run in RUNS)


@pytest.mark.parametrize("case", GENERIC)
def test_reader_restores_generic_containers(case):
    """Plain and zlib0 restores of what the host writer wrote, against what the reference restored from its own file."""
    from lepton_b200 import HostLep
    from lepton_b200.codec import zlib0_frame
    r = PERM["cases"][case]["skipverify"]
    data = case_bytes(case)
    hl = HostLep(generic(data))
    assert hl.status == 0, (hl.status, hl.error)
    plain, z = hl.restore_generic(), hl.restore_generic(zlib0=True)
    assert plain == data and md5(plain) == r["restore"]["md5"]
    assert md5(z) == r["restore_zlib0"]["md5"] and z == zlib0_frame(data)


@pytest.mark.parametrize("name", LEP_FIXTURES)
def test_reader_restores_reference_files(name):
    from lepton_b200 import HostLep
    from lepton_b200.codec import lep_members
    r = PERM["cases"][name]["skipverify"]
    lep = read_golden("permissive/%s.lep" % name)
    assert md5(lep) == r["lep_md5"]
    hl = HostLep(lep)
    assert hl.status == 0 and not hl.zlib0
    assert md5(hl.restore_generic()) == r["restore"]["md5"]
    assert md5(hl.restore_generic(zlib0=True)) == r["restore_zlib0"]["md5"]
    assert lep_members(lep) == [(0, len(case_bytes(name)), 0)]          # one member, nothing coded


def test_zeta_generic_restores_as_zlib0():
    from lepton_b200 import HostLep
    data = case_bytes("two_bytes")
    hl = HostLep(b"\xce\xb6" + generic(data)[2:])
    assert hl.status == 0 and hl.zlib0
    assert hl.restore_generic() == hl.restore_generic(zlib0=True)


def test_coded_containers_are_not_generic():
    from lepton_b200 import HostLep
    hl = HostLep(read_golden("androidcrop.lep"))
    assert hl.status == 0
    with pytest.raises(Exception):
        hl.restore_generic()


@pytest.mark.parametrize("case", CODED)
def test_coded_cases_give_the_ordinary_lep(case):
    """A file the coder takes gives under -permissive what it gives without: the front end takes it and the container
    writer, fed the CPU oracle's segment streams, writes the reference's bytes."""
    from lepton_b200 import HostJpeg
    e = PERM["cases"][case]
    off = [int(f.split("=")[1]) for f in e["flags"] if f.startswith("-embedding=")]
    hj = HostJpeg(case_bytes(case), embedding=off[0] if off else None)
    assert hj.status == 0, (case, hj.error)
    lep = hj.write_lep([s for _, s, _ in oracle_encode_image(hj.coef_image())])
    for run in RUNS:
        assert md5(lep) == e[run]["lep_md5"], (case, run)


def blob_of(lep):
    zlen = struct.unpack("<I", lep[24:28])[0]
    return zlib.decompress(lep[28:28 + zlen]), lep[28 + zlen:]


def with_blob(lep, blob, tail=None):
    """The .lep with its header blob (and what follows it) replaced."""
    zlen = struct.unpack("<I", lep[24:28])[0]
    z = zlib.compress(blob, 9)
    rest = lep[28 + zlen:] if tail is None else tail
    return lep[:24] + struct.pack("<I", len(z)) + z + rest


def sections(blob):
    """name -> (offset, length of the whole section) for the sections of a generic blob."""
    out, p = {}, 0
    while p < len(blob):
        tag = blob[p:p + 3]
        if tag == b"HDR" or tag == b"PGE" or tag == b"GRB":
            n = 7 + struct.unpack("<I", blob[p + 3:p + 7])[0]
        elif tag == b"P0D":
            n = 4
        else:
            assert blob[p:p + 2] == b"HH", tag
            n = 3 + 16 * blob[p + 2]
            tag = b"HH"
        out[tag.decode()] = (p, n)
        p += n
    return out


def damaged_generic_files():
    lep = generic(case_bytes("blob70k"))
    blob, tail = blob_of(lep)
    s = sections(blob)
    pge, grb = s["PGE"], s["GRB"]
    out = {
        "pgr_section": with_blob(lep, blob[:pge[0]] + b"PGR" + blob[pge[0] + 3:]),
        "siz_section": with_blob(lep, blob + b"SIZ" + struct.pack("<I", 70000)),
        "grb_not_empty": with_blob(lep, blob[:grb[0]] + b"GRB" + struct.pack("<I", 2) + b"\xff\xd9"),
        "no_grb": with_blob(lep, blob[:grb[0]]),
        "pge_shorter_than_file": with_blob(lep, blob[:pge[0]] + b"PGE" + struct.pack("<I", 69999) +
                                           blob[pge[0] + 7:pge[0] + 7 + 69999] + blob[grb[0]:]),
        "crs_section": with_blob(lep, blob + b"CRS" + struct.pack("<II", 1, 0)),
        "padbit_set": with_blob(lep, blob[:s["P0D"][0] + 3] + b"\x01" + blob[s["P0D"][0] + 4:]),
        "handoff_not_zero": with_blob(lep, blob[:s["HH"][0] + 3] + b"\x00\x00\x01" + blob[s["HH"][0] + 6:]),
        "other_header": with_blob(lep, blob[:7 + 20] + b"\x01" + blob[7 + 21:]),
        "mux_packet_behind_cmp": with_blob(lep, blob, tail=b"CMP" + b"\x00\x00\x00\x07" + tail[3:]),
    }
    # an ordinary container marked 'Y'
    lz = bytearray(read_golden("androidcrop.lep"))
    lz[3] = ord("Y")
    out["coded_marked_y"] = bytes(lz)
    return out


DAMAGED = sorted(damaged_generic_files())


@pytest.mark.parametrize("name", DAMAGED)
def test_other_y_containers_stay_refused(name):
    """Only the generic container opens: a -startbyte slice (PGR / SIZ sections) or any 'Y' container that differs from
    the generic one in any section is refused with 200, never restored to something else."""
    from lepton_b200 import HostLep
    hl = HostLep(damaged_generic_files()[name])
    assert hl.status == 200, (name, hl.status, hl.error)


def test_damaged_files_differ_from_the_generic_one():
    lep = generic(case_bytes("blob70k"))
    assert all(v != lep for v in damaged_generic_files().values())
