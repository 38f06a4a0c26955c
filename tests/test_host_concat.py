"""The member walk over streams of concatenated .lep files (no GPU): lepb200_host_lep_members on every case of
tests/golden/concat.json (tests/golden/make_concat.py) against the members the reference restored."""
import json
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from helpers import GOLDEN  # noqa: E402
from make_concat import DIFFERENCES, LEPCAT, case_bytes, expected, member, part_source, members as member_sources  # noqa: E402

CON = json.load(open(os.path.join(GOLDEN, "concat.json")))
CASES = sorted(CON["cases"])


def lib_or_skip():
    from lepton_b200 import lib
    L = lib()
    if not L.lepb200_host_brotli_available():
        pytest.skip("libbrotlidec (libbrotlidec.so.1) not found: container version 2 members cannot be read")
    return L


def expected_members(name):
    """[(status, JPEG size)] the walk must give: one entry per member the reference restored (what its output is made of),
    then the failing member where the reference failed."""
    e = CON["cases"][name]
    src = member_sources()
    sizes = []
    for p in e["parts"]:
        if p.startswith("@"):
            sizes += [len(src[m][0]) for m in LEPCAT[p[1:]]]
        elif p.startswith("!cut:"):
            sizes.append(len(src[p[5:]][0]))
        elif not p.startswith("#"):
            sizes.append(len(part_source(p, src)))
    st, _ = expected(name, e, "plain")
    if name == "v1_then_v2":
        return [(3, sizes[0])]                         # the version-1 member takes the rest of the stream as its mux packets
    if name.startswith("zeta_"):
        return [(0, sizes[0])]                         # the second member's magic differs from the first's: the stream ends
    if st == 0:
        assert sum(sizes) == e["plain"]["len"], name
        return [(0, s) for s in sizes]
    return [(0, s) for s in sizes[:-1]] + [(st, sizes[-1])]


@pytest.mark.parametrize("name", CASES)
def test_member_walk(name):
    lib_or_skip()
    from lepton_b200 import lep_members
    got = lep_members(case_bytes(CON["cases"][name]["parts"]))
    assert [(s, n) for s, n, _ in got] == expected_members(name), (name, got)


def test_thread_segments_of_members():
    """Members keep their own thread-segment counts, whatever the first member's (the reference's NUM_THREADS only goes down,
    and it still restores every member: t1_then_tall_t8 and tall_t8_then_t1 give the sources)."""
    lib_or_skip()
    from lepton_b200 import lep_members
    for name, want in (("t1_then_tall_t8", [1, 8]), ("tall_t8_then_t1", [8, 1]), ("tall_t1_then_t8", [1, 8]),
                       ("t1_then_tall_t4", [1, 4]), ("progressive_then_baseline", [2, 1])):
        e = CON["cases"][name]
        assert [k for _, _, k in lep_members(case_bytes(e["parts"]))] == want, name
        assert e["plain"]["md5"] == e["jpeg_md5"], name


@pytest.mark.parametrize("name", sorted(set(p for e in CON["cases"].values() for p in e["parts"]
                                            if not p[0] in "#!@")))
def test_one_member_stream_is_the_single_file(name):
    """A single member is what lepb200_host_lep_open makes of the file: status, geometry, segments and every stream byte."""
    lib_or_skip()
    from lepton_b200 import HostLep, lep_members
    data = member(name)
    single = HostLep(data)
    m = HostLep(data, member=0)
    assert lep_members(data) == [(single.status, CON["members"][name]["jpeg_len"], single.coef_image().nseg)]
    assert (m.status, m.error) == (single.status, single.error)
    a, b = single.coef_image(), m.coef_image()
    assert (a.ncmp, a.mcuv, a.bch, a.bcv, a.luma_y_start) == (b.ncmp, b.mcuv, b.bch, b.bcv, b.luma_y_start)
    assert single.streams(a.nseg) == m.streams(b.nseg)
    assert single.scan_layout() == m.scan_layout()


def test_members_open_like_files():
    """Member k of a stream opens with the header, handoffs and streams of the k-th file that went into it, -lepcat files
    included (their later members' headers come from the first member's blob)."""
    lib_or_skip()
    from lepton_b200 import HostLep
    for name in ("triple_colorswap_androidtrail_narrowrst", "lepcat3", "embedded_doubled", "tall_t1_then_t8"):
        parts = CON["cases"][name]["parts"]
        files = LEPCAT[parts[0][1:]] if parts[0].startswith("@") else parts
        data = case_bytes(parts)
        for k, f in enumerate(files):
            one, m = HostLep(member(f)), HostLep(data, member=k)
            assert m.status == 0 and one.status == 0, (name, k, m.error)
            a, b = one.coef_image(), m.coef_image()
            assert (a.ncmp, a.mcuv, a.bch, a.bcv, a.luma_y_start) == (b.ncmp, b.mcuv, b.bch, b.bcv, b.luma_y_start), (name, k)
            assert one.streams(a.nseg) == m.streams(b.nseg), (name, k)
            assert one.scan_layout() == m.scan_layout(), (name, k)


def test_lepcat_rules():
    """-lepcat: a later member whose own header blob is not empty fails with the reference's assertion (read_ujpg :4188),
    and without the walk (lepb200_host_lep_open) the CNT marker is unknown data in the header blob, as before."""
    lib_or_skip()
    from lepton_b200 import HostLep, lep_members
    cat, first = member("lepcat2"), member("androidcrop")
    le32 = lambda b, o: int.from_bytes(b[o:o + 4], "little")            # noqa: E731
    # lepcat2's first member (its blob ends in CNT + the second member's headers), then a member with a blob of its own
    end = 28 + le32(cat, 24) + len(first) - 28 - le32(first, 24)
    assert cat[end:end + 2] == b"\xcf\x84" and le32(cat, end + 24) == 0
    assert [s for s, _, _ in lep_members(cat[:end] + member("narrowrst"))] == [0, 1]
    assert [s for s, _, _ in lep_members(cat + member("narrowrst"))] == [0, 0, 0]     # no headers pending behind the last
    assert HostLep(cat).status == 42
    assert DIFFERENCES                                  # the documented differences are pinned by test_member_walk


def test_open_member_out_of_range():
    lib_or_skip()
    from lepton_b200 import HostLep, LeptonB200Error
    with pytest.raises(LeptonB200Error):
        HostLep(member("narrowrst"), member=1)
