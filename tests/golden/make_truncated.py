#!/usr/bin/env python
"""Regenerate tests/golden/truncated/ and tests/golden/truncated.json: small baseline JPEGs cut at every byte of their
scan, and what the UNMODIFIED reference CLI makes of every cut.

A JPEG that ends inside its scan (an interrupted upload, a partial download) is coded by the reference byte for byte:
the last blocks are cut short (eof fix-up), the coded extent of every component is recorded in the container (EEE)
and rounded up to whole MCU rows, and the bytes after the last whole byte of the scan are kept as a garbage tail.  The
sources here are small enough that every byte offset from 3 bytes before the end of the SOS header to the full length
is a cut: a cut inside the SOS header, a scan with no bytes, cuts inside stuffed FF 00 and inside restart markers, a
missing EOI, and the complete file.  Tests build each cut as src[:cut].

Run where oracle/_ref/lepton exists (oracle/Makefile builds it from the reference tree):
    python tests/golden/make_truncated.py
The output is deterministic: a second run reproduces every file byte for byte.  truncated.json holds

  sources[NAME]         path, jpg_md5, len, sos_end (offset of the first scan byte), first_cut (= sos_end - 3),
                        ncmp, sampling, width, height, restart
  runs[NAME][FLAG]      FLAG = t1 (plain), t4 / t8 (-minencodethreads=4 / =8), each run as
                        `lepton -unjailed -skipverify cut.jpg out.lep`:
                          codes      one character per cut (cut = first_cut + index), see `codes` and code_of():
                                     r / n a clean .lep that the reference's own decoder does / does not restore to
                                     the cut (most multi-segment records of a cut: its decoder asserts on the overhang
                                     bits of a handoff), c / t refused with COEFFICIENT_OUT_OF_RANGE (6) -- t when the
                                     other threads printed THREAD_PROTOCOL_ERROR (5) as well -- and u refused with
                                     UNSUPPORTED_JPEG (42).  A run that wrote an ExitCode name to stderr failed with
                                     that code even when the process exited with 0 (custom_exit ends one thread; see
                                     make_extremes.py and exit_name_of).  A failed multi-thread run may leave a partial
                                     file whose length depends on thread timing; it is not recorded.
                          lep_chain  md5 over the md5s of the clean .lep files in cut order (lep_chain()): a test
                                     that rebuilds every container compares the whole run at once.  The container
                                     holds the truncation bounds (EEE) and the splits (handoffs), so they are pinned too.
  leps[FILE]            the committed subset, tests/golden/truncated/FILE (select(): a few per selection class, from
                        the sources in turn): source, cut, flag, lep_md5, trunc_bcv, trunc_bc, splits, classes
  classes               every selection class and how many committed files carry it (each is asserted non-empty)
"""
import hashlib
import json
import multiprocessing
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from jpegwriter import AC_SYMBOLS, HuffTable, fit_lengths, geometry, write_baseline  # noqa: E402
from make_extremes import EXIT_CODES, LEPTON, long_tables  # noqa: E402

OUTDIR = os.path.join(HERE, "truncated")
OUT = os.path.join(HERE, "truncated.json")
FLAGS = {"t1": [], "t4": ["-minencodethreads=4"], "t8": ["-minencodethreads=8"]}
ZZ63 = 48                   # AlignedBlock index of zig-zag coefficient 63


def md5(b):
    return hashlib.md5(b).hexdigest()


def smooth_planes(rng, w, h, sampling, nnz=3, amp=40):
    """Photo-like sparse planes: a DC random walk and a few low-frequency AC coefficients per block, so that a scan
    stays a few hundred bytes long and every byte of it can be a cut."""
    _, _, grid, _ = geometry(w, h, sampling)
    planes = []
    for c, (bx, by) in enumerate(grid):
        n = by * bx
        p = np.zeros((n, 64), np.int64)
        pos = rng.integers(1, 15, size=(n, nnz))
        val = rng.integers(-amp, amp + 1, size=(n, nnz))
        np.put_along_axis(p, pos, val, axis=1)
        p[:, 0] = np.clip(np.cumsum(rng.integers(-30, 31, size=n)), -500 if c else -900, 500 if c else 900)
        planes.append(p.reshape(by, bx, 64))
    return planes


S420, S422, S444, GREY = [(2, 2), (1, 1), (1, 1)], [(2, 1), (1, 1), (1, 1)], [(1, 1)] * 3, [(1, 1)]


def corpus():
    """-> [(name, width, height, sampling, restart, jpeg bytes)].  Each file has its own seed."""
    files = []

    def rng(k):
        return np.random.default_rng(20261017 + k)

    def add(name, k, w, h, sampling, restart=0, **kw):
        q = [[6] + [4 + i // 8 for i in range(63)]] * (1 if len(sampling) == 1 else 2)
        files.append((name, w, h, sampling, restart, write_baseline(smooth_planes(rng(k), w, h, sampling), w, h, sampling,
                                                                     q, restart=restart, **kw)))

    # The bit reader reads zeros past the end of the data.  With the usual tables the all-zeros code is EOB, so a cut
    # rarely leaves a zero run that runs off its block; giving ZRL the all-zeros code makes nearly every cut inside the
    # AC codes of a block end in the eof fix-up (coefficient 63 set to 1).
    zrl_first = HuffTable(fit_lengths([(0xF0, 8)] + [(s, 8) for s in AC_SYMBOLS if s != 0xF0]))
    add("c420_odd", 1, 77, 61, S420)              # partial MCUs at the right and bottom edges
    add("c422", 2, 64, 56, S422)
    add("c444_odd", 3, 41, 37, S444)
    add("grey_odd", 4, 100, 60, GREY, ac_tables=[zrl_first])    # one component: a non-interleaved scan of the coded blocks
    add("c420_rst1", 5, 48, 48, S420, restart=1)
    add("c444_rst3", 6, 56, 48, S444, restart=3, ac_tables=[zrl_first])
    # 16-bit Huffman codes, and two luma blocks of all-ones codes and magnitudes: runs of stuffed FF 00
    r = rng(7)
    tabs = [long_tables(r), long_tables(r)]
    p = smooth_planes(r, 40, 48, S420)
    p[0][0, :2, 1:21] = 2047
    files.append(("c420_long_ff", 40, 48, S420, 0,
                  write_baseline(p, 40, 48, S420, [[6] + [4 + i // 8 for i in range(63)]] * 2,
                                 dc_tables=[t[0] for t in tabs], ac_tables=[t[1] for t in tabs])))
    return files


def sos_end(jpg):
    """Offset of the first scan byte (right after the SOS segment)."""
    pos = jpg.index(b"\xff\xda")
    return pos + 2 + int.from_bytes(jpg[pos + 2:pos + 4], "big")


def exit_name_of(stderr):
    """The ExitCode a run failed with, from the names it printed.  Threads that fail together print their names on one
    line in either order; the coder's own error (e.g. COEFFICIENT_OUT_OF_RANGE) wins over the THREAD_PROTOCOL_ERROR the
    other threads report, so that the record does not depend on thread timing."""
    text = stderr.decode("latin-1")
    names = [n for n in EXIT_CODES if n in text and not any(n != m and n in m and m in text for m in EXIT_CODES)]
    own = [n for n in names if n != "THREAD_PROTOCOL_ERROR"]
    assert len(own) <= 1, names
    return own[0] if own else (names[0] if names else None)


def run_cut(job):
    """Every flag set on one cut -> {flag: (row, lep bytes of a clean run)}."""
    import lepfmt
    jpg, = job
    out = {}
    with tempfile.TemporaryDirectory() as td:
        src, dst, b = os.path.join(td, "cut.jpg"), os.path.join(td, "o.lep"), os.path.join(td, "b.jpg")
        with open(src, "wb") as f:
            f.write(jpg)
        for flag, fl in FLAGS.items():
            for p in (dst, b):
                if os.path.exists(p):
                    os.unlink(p)
            r0 = subprocess.run([LEPTON, "-unjailed", "-skipverify"] + fl + [src, dst], capture_output=True)
            exit_name = exit_name_of(r0.stderr)
            rc = EXIT_CODES[exit_name] if exit_name else r0.returncode
            lep = open(dst, "rb").read() if rc == 0 and os.path.exists(dst) else b""
            assert rc or lep, "the reference wrote nothing and reported no error"
            back = tbcv = tbc = splits = None
            if lep:
                r = subprocess.run([LEPTON, "-unjailed", dst, b], capture_output=True)
                back = int(r.returncode == 0 and os.path.exists(b) and open(b, "rb").read() == jpg)
                lf = lepfmt.parse_container(lep)
                tbcv, tbc = lepfmt.truncation(lf)
                splits = [h.luma_y_start for h in lf.handoffs]
            tpe = int(b"THREAD_PROTOCOL_ERROR" in r0.stderr)
            out[flag] = ([rc, exit_name, md5(lep) if lep else None, back, tbcv, tbc, splits, tpe], lep)
    return out


def mcu_of(dpos, c, ncmp, sampling, mcuh, bch):
    """MCU index of block dpos of component c (interleaved scans)."""
    y, x = divmod(dpos, bch[c])
    return (y // sampling[c][1]) * mcuh + x // sampling[c][0]


def read(rel):
    with open(os.path.join(HERE, rel), "rb") as f:
        return f.read()


def classify(meta, rows, full_planes, leps_t1):
    """-> {class: [group of cuts committed together, ...]}: the cuts of one source that show each case."""
    import lepfmt
    from helpers import oracle_decode_planes
    w, h, sampling, ln, first = meta["width"], meta["height"], meta["sampling"], meta["len"], meta["first_cut"]
    mcuh, mcuv, grid, _ = geometry(w, h, sampling)
    bch = [g[0] for g in grid]
    ncmp = len(sampling)
    full_bc = [g[0] * g[1] for g in grid]
    t1 = rows["t1"]
    ok = [first + i for i, r in enumerate(t1) if r[0] == 0]
    trunc = [c for c in ok if t1[c - first][5] != full_bc]
    v0 = sampling[0][1]
    out = {}
    # the luma bound inside the first MCU row
    fr = [c for c in trunc if t1[c - first][4][0] <= v0]
    out["first_mcu_row"] = [[c] for c in fr[:1] + fr[-1:]]
    # just before, at and after the cut where the luma bound first reaches MCU row 1
    at = next((c for c in trunc if t1[c - first][5][0] > v0 * bch[0]), None)
    out["mcu_row_boundary"] = [[c for c in (at - 1, at, at + 1) if c in ok]] if at else []
    # the luma of an MCU is coded, its chroma not (yet)
    if ncmp == 3:
        out["chroma_inside_mcu"] = [[c] for c in trunc
                                    if min(mcu_of(t1[c - first][5][k] - 1, k, ncmp, sampling, mcuh, bch) for k in (1, 2))
                                    < mcu_of(t1[c - first][5][0] - 1, 0, ncmp, sampling, mcuh, bch)][:1]
    # the rounded-up trunc_bcv holds a block row that lies wholly past trunc_bc
    out["row_past_bound"] = [[c] for c in trunc
                             if any((t1[c - first][4][k] - 1) * bch[k] >= t1[c - first][5][k] for k in range(ncmp))][:1]
    # eof fix-up: a block cut inside its zero run comes back with coefficient 63 set to 1
    fix = []
    for c in trunc:
        planes, _ = oracle_decode_planes(lepfmt.parse_container(leps_t1[c]))
        tbc = t1[c - first][5]
        if any(((planes[k][:tbc[k], ZZ63] == 1) & (full_planes[k][:tbc[k], ZZ63] != 1)).any() for k in range(ncmp)):
            fix.append([c])
            break
    out["eof_fixup"] = fix
    # the cut falls between FF and 00, between FF and Dn; EOI missing; the complete file
    data = read(meta["path"])
    out["inside_ff00"] = [[c] for c in ok if data[c - 1] == 0xFF and data[c] == 0x00 and c < ln - 2][:1]
    out["inside_rst"] = [[c] for c in ok if data[c - 1] == 0xFF and 0xD0 <= data[c] <= 0xD7][:1]
    out["no_eoi"] = [[c for c in (ln - 2, ln - 1) if c in ok]]
    out["complete"] = [[ln]]
    return {k: [g for g in v if g] for k, v in out.items()}


def classify_threads(rows, meta):
    """-> {(class, flag): [[cut]]} from the -minencodethreads records."""
    first = meta["first_cut"]
    out = {}
    for flag in ("t4", "t8"):
        rs = [(first + i, r) for i, r in enumerate(rows[flag]) if r[0] == 0]
        # a thread-segment starts at or past the last coded luma row
        out[("segment_past_rows", flag)] = [[c] for c, r in rs if any(y >= r[4][0] for y in r[6][1:])][-1:]
        # written cleanly, but the reference's own decoder refuses it (or restores other bytes)
        bad = [[c] for c, r in rs if r[3] == 0]
        out[("reference_cannot_decode", flag)] = bad[len(bad) // 2:len(bad) // 2 + 1]
        # several segments, and the reference decodes it
        out[("multi_segment", flag)] = [[c] for c, r in rs if len(r[6]) > 1 and r[3] == 1][-2:-1]
    return out


def select(cands, cap=2):
    """A few groups per class, taken from different sources in turn (the sources rotate with the class), so that the
    committed subset stays small but covers every geometry."""
    names = sorted(cands)
    picks = {}
    classes = sorted({k for n in names for k in cands[n]}, key=str)
    for i, k in enumerate(classes):
        got = 0
        for n in names[i % len(names):] + names[:i % len(names)]:
            if got == cap:
                break
            if cands[n].get(k):
                picks.setdefault(n, []).append((k, cands[n][k][0]))
                got += 1
    return picks


CLASSES = ["first_mcu_row", "mcu_row_boundary", "chroma_inside_mcu", "row_past_bound", "eof_fixup", "inside_ff00",
           "inside_rst", "no_eoi", "complete"] + ["%s_%s" % (k, f) for k in ("segment_past_rows", "reference_cannot_decode",
                                                                           "multi_segment") for f in ("t4", "t8")]


# one character per cut and run in truncated.json: what the reference did
CODES = {"r": "clean .lep that the reference's own decoder restores to the cut",
         "n": "clean .lep that the reference's own decoder refuses or restores to other bytes",
         "c": "COEFFICIENT_OUT_OF_RANGE (6)",
         "t": "COEFFICIENT_OUT_OF_RANGE (6) together with THREAD_PROTOCOL_ERROR (5) from the other threads",
         "u": "UNSUPPORTED_JPEG (42)"}


def code_of(row):
    rc, _, _, back, _, _, _, tpe = row
    code = {(0, 1): "r", (0, 0): "n"}.get((rc, back)) if rc == 0 else {6: "t" if tpe else "c", 42: "u"}.get(rc)
    assert code, row
    return code


def lep_chain(lep_md5s):
    """md5 over the md5s (hex) of the clean .lep files of one source and flag, in cut order."""
    return md5("".join(lep_md5s).encode())


def main():
    import lepfmt
    from helpers import oracle_decode_planes
    os.makedirs(OUTDIR, exist_ok=True)
    for f in os.listdir(OUTDIR):
        if f.endswith(".lep"):
            os.unlink(os.path.join(OUTDIR, f))
    record = {"codes": CODES, "sources": {}, "runs": {}, "leps": {}}
    cands, kept = {}, {}
    with multiprocessing.Pool(os.cpu_count()) as pool:
        for name, w, h, sampling, restart, jpg in corpus():
            path = "truncated/%s.jpg" % name
            with open(os.path.join(HERE, path), "wb") as f:
                f.write(jpg)
            se = sos_end(jpg)
            meta = {"path": path, "jpg_md5": md5(jpg), "len": len(jpg), "sos_end": se, "first_cut": se - 3,
                    "ncmp": len(sampling), "sampling": [list(s) for s in sampling], "width": w, "height": h,
                    "restart": restart}
            cuts = list(range(se - 3, len(jpg) + 1))
            res = pool.map(run_cut, [(jpg[:c],) for c in cuts], chunksize=4)
            rows = {flag: [r[flag][0] for r in res] for flag in FLAGS}
            leps = {flag: {c: r[flag][1] for c, r in zip(cuts, res)} for flag in FLAGS}
            full_planes, _ = oracle_decode_planes(lepfmt.parse_container(leps["t1"][len(jpg)]))
            cands[name] = {(k, "t1"): v for k, v in classify(meta, rows, full_planes, leps["t1"]).items()}
            cands[name].update(classify_threads(rows, meta))
            kept[name] = (rows, leps)
            record["sources"][name] = meta
            record["runs"][name] = {flag: {"codes": "".join(code_of(r) for r in rows[flag]),
                                           "lep_chain": lep_chain([md5(leps[flag][c]) for c in cuts if leps[flag][c]])}
                                    for flag in FLAGS}
            print(name, len(jpg), len(cuts), "cuts", {f: {k: record["runs"][name][f]["codes"].count(k) for k in CODES}
                                                       for f in FLAGS}, flush=True)
    classes = {}
    for name, picks in sorted(select(cands).items()):
        rows, leps = kept[name]
        first = record["sources"][name]["first_cut"]
        for (k, flag), group in picks:
            k = k if flag == "t1" else "%s_%s" % (k, flag)
            for c in group:
                fn = "%s_%d%s.lep" % (name, c, "" if flag == "t1" else "_" + flag)
                if fn not in record["leps"]:
                    lep = leps[flag][c]
                    with open(os.path.join(OUTDIR, fn), "wb") as f:
                        f.write(lep)
                    r = rows[flag][c - first]
                    record["leps"][fn] = {"source": name, "cut": c, "flag": flag, "lep_md5": md5(lep), "classes": [],
                                          "trunc_bcv": r[4], "trunc_bc": r[5], "splits": r[6]}
                record["leps"][fn]["classes"].append(k)
                classes[k] = classes.get(k, 0) + 1
    record["classes"] = classes
    for k in CLASSES:
        assert classes.get(k), ("selection class missing", k)
    total = sum(os.path.getsize(os.path.join(OUTDIR, f)) for f in os.listdir(OUTDIR))
    print(len(record["leps"]), "committed .lep files;", total, "bytes under truncated/;", sorted(classes.items()))
    leps = record.pop("leps")
    text = json.dumps(record, indent=1, sort_keys=True)
    text = text[:-2] + ',\n "leps": {\n' + ",\n".join("  %s: %s" % (json.dumps(fn), json.dumps(leps[fn], sort_keys=True))
                                                   for fn in sorted(leps)) + "\n }\n}\n"
    with open(OUT, "w") as f:
        f.write(text)


if __name__ == "__main__":
    main()
