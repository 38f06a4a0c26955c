"""Hot set of the probability model on bench-like input (CPU only; a tool, not a test).

    python tests/tools_model_hotset.py [n_images]

Takes `n_images` JPEGs of the benchmark's corpus (bench.make_corpus(2, n): 1080p 4:2:0 q85), gets their coefficient
planes from the repository's own front end (HostJpeg.coef_image()) and codes every thread-segment with the C oracle,
counting how often each branch is used.  The counts come from a private build of oracle/lepton_oracle.c made in a
temporary directory: one line is added to `code_bit`, after the branch update, and nothing else changes; every segment
is coded by that build and by the oracle library itself, and the tool stops if their streams differ.

Each oracle branch is then mapped to its 16-bit word in two layouts of the device model (lep_common.cuh): the one before
the exponent chains were split (`old`) and the shipped one (`new`).  Per segment, averaged over all segments, it prints
the decisions, the distinct words touched, the 32-byte sectors touched, and how many of the most used sectors cover
50 / 80 / 90 / 95 / 99 % of the decisions; then the decision share per table, per exponent word k, and of the front
region that the group decode kernel keeps in shared memory.  The row `new, global memory` leaves that region out: it is
what the group kernel's decisions bring through the L2 (its percentages are of the decisions that remain).
"""
import ctypes
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import oracle  # noqa: E402

# ---- oracle Model (oracle/lepton_oracle.c): tables in declaration order, Branch = 3 bytes
ORACLE_TABLES = [
    ("nz7", (2, 26, 6, 32)), ("nze_v", (2, 8, 8, 3, 4)), ("nze_h", (2, 8, 8, 3, 4)), ("resn", (2, 64, 10, 10)),
    ("resdc", (12, 10)), ("thr", (2, 256, 8, 128)), ("exp7", (2, 10, 49, 12, 11)), ("expx", (2, 10, 15, 12, 11)),
    ("expdc", (12, 17, 11)), ("sign", (2, 4, 12)),
]
N_BRANCHES = sum(int(np.prod(s)) for _, s in ORACLE_TABLES)
CODE_BIT = "static inline int code_bit(Codec *c, Branch *b, int bit) {"
UPDATE = "    branch_update(b, bit);\n    c->ndecisions++;\n"


def counting_oracle(tmp):
    """The oracle with a per-branch hit counter (lo_hits, off while NULL), built in `tmp`."""
    src = open(os.path.join(ROOT, "oracle", "lepton_oracle.c")).read()
    head, sep, body = src.partition(CODE_BIT)
    assert sep and src.count(CODE_BIT) == 1 and body.count(UPDATE) >= 1 and body.index(UPDATE) < body.index("\n}\n"), \
        "code_bit of oracle/lepton_oracle.c is not in the expected form"
    body = body.replace(UPDATE, UPDATE + "    if (lo_hits) lo_hits[b - (Branch *)c->model]++;\n", 1)
    path = os.path.join(tmp, "lepton_oracle_hits.c")
    with open(path, "w") as f:
        f.write(head + "uint64_t *lo_hits = 0;\n" + sep + body)
    so = os.path.join(tmp, "liblepton_oracle_hits.so")
    subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-fwrapv", "-Wno-unused-function", "-o", so, path])
    L = ctypes.CDLL(so)
    P3 = ctypes.c_void_p * 3
    L.lo_encode_segment.argtypes = [ctypes.POINTER(oracle.Geometry), P3, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                    ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t), ctypes.POINTER(ctypes.c_uint64)]
    L.lo_encode_segment.restype = ctypes.c_int
    return L


# ---- device model layouts (word index of every oracle branch; -1 where the device allocates no word)
def _grid(shape):
    return np.indices(shape).reshape(len(shape), -1)


def layout(new):
    if new:      # lep_common.cuh as shipped
        SIGN = 0; RESDC = 96; NZ7T = RESDC + 120; EXPH = NZ7T + 160 + 8; EXPDC = EXPH; HOT = EXPDC + 12 * 17 * 4
        EXP7 = HOT; EXPX = EXP7 + 2 * 10 * 49 * 12 * 4; EXPT = EXPX + 2 * 8 * 15 * 12 * 4; NZ7 = EXPT + 2 * (EXPT - EXPH)
        NZE = NZ7 + 2 * 10 * 56; RESN = NZE + 3072; THR = RESN + 20480; TOTAL = THR + 2 * 256 * 8 * 128
        hstride, rdc = 4, 10
    else:        # before the split: exponent rows of 16 words, no front region
        NZ7 = 0; NZE = 3840; RESN = NZE + 3072; RESDC = RESN + 20480; EXP7 = RESDC + 192; EXPX = EXP7 + 2 * 10 * 49 * 12 * 16
        EXPDC = EXPX + 2 * 8 * 15 * 12 * 16; SIGN = EXPDC + 12 * 17 * 16; THR = SIGN + 128; TOTAL = THR + 2 * 256 * 8 * 128
        HOT = 0; hstride, rdc = 16, 16

    def exp_word(head, k):
        if not new:
            return head + k
        return np.where(k < 4, head + k, EXPT + 2 * (head - EXPH) + (k - 4))

    out = []
    for name, shape in ORACLE_TABLES:
        g = _grid(shape)
        w = np.full(g.shape[1], -1, np.int64)
        if name == "nz7":
            ci, b, idx, pre = g
            ok = (b < 10) & (pre < (1 << (5 - idx)))
            tree = ci * 10 + b
            if new:
                top = NZ7T + tree * 8 + 8 - (16 >> np.maximum(idx - 2, 0))
                rear = NZ7 + tree * 56 + 64 - (64 >> np.minimum(idx, 2))
                w = np.where(ok, np.where(idx >= 3, top, rear) + pre, -1)
            else:
                w = np.where(ok, NZ7 + ((tree * 6 + idx) << 5) + pre, -1)
        elif name in ("nze_v", "nze_h"):
            ci, eob, nzb, idx, pre = g
            vert = 1 if name == "nze_v" else 0
            w = NZE + (((((vert * 2 + ci) * 8 + eob) * 8 + nzb) * 3 + idx) << 2) + pre
        elif name == "resn":
            ci, coord, b, i = g
            w = RESN + (((ci * 64 + coord) * 10 + b) << 4) + i
        elif name == "resdc":
            lm, i = g
            w = RESDC + lm * rdc + i
        elif name == "thr":
            ci, ctx, ln, so = g
            w = THR + (((ci * 256 + ctx) * 8 + ln) << 7) + so
        elif name == "exp7":
            ci, b, zz, bsr, k = g
            w = exp_word(EXP7 + (((ci * 10 + b) * 49 + zz) * 12 + bsr) * hstride, k)
        elif name == "expx":
            ci, ne, z, bsr, k = g
            w = np.where(ne < 8, exp_word(EXPX + (((ci * 8 + ne) * 15 + z) * 12 + bsr) * hstride, k), -1)
        elif name == "expdc":
            a, b, k = g
            w = exp_word(EXPDC + (a * 17 + b) * hstride, k)
        elif name == "sign":
            ci, a, b = g
            w = SIGN + (ci * 4 + a) * 12 + b
        out.append(w)
    words = np.concatenate(out)
    assert words.max() < TOTAL
    return words, TOTAL, HOT


def segment_stats(hits, words):
    used = hits > 0
    assert not np.any(used & (words < 0)), "a branch the device model does not allocate was used"
    nd = int(hits.sum())
    sec = np.bincount(words[used] // 16, weights=hits[used].astype(np.float64))
    sec = np.sort(sec[sec > 0])[::-1]
    cum = np.cumsum(sec) / nd
    cover = [int(np.searchsorted(cum, f - 1e-12) + 1) for f in (0.5, 0.8, 0.9, 0.95, 0.99)]
    return nd, int(np.unique(words[used]).size), len(sec), cover


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 2
    import bench
    from lepton_b200 import HostJpeg
    from lepton_b200.codec import lib
    jpegs = bench.make_corpus(2, n)
    old_w, old_total, _ = layout(False)
    new_w, new_total, hot = layout(True)
    assert new_total * 2 == lib().lepb200_model_bytes(), "layout() disagrees with lep_common.cuh"
    g_tab = np.concatenate([np.full(int(np.prod(s)), i) for i, (_, s) in enumerate(ORACLE_TABLES)])
    g_k = np.concatenate([np.indices(s)[-1].ravel() if nm.startswith("exp") else np.full(int(np.prod(s)), -1)
                          for nm, s in ORACLE_TABLES])
    rows = {"old": [], "new": [], "new, global memory": []}
    tab = np.zeros(len(ORACLE_TABLES)); kh = np.zeros(11); front = 0.0; total = 0
    with tempfile.TemporaryDirectory() as tmp:
        L = counting_oracle(tmp)
        hits = np.zeros(N_BRANCHES, np.uint64)
        ptr = ctypes.c_void_p.in_dll(L, "lo_hits")
        for data in jpegs:
            hj = HostJpeg(data)
            img = hj.coef_image()
            g = oracle.make_geometry(img.ncmp, list(img.bch), list(img.bcv), img.mcuv, img.qtables_zigzag,
                                     list(img.trunc_bcv), list(img.trunc_bc))
            planes = [np.ascontiguousarray(p) for p in img.planes]
            starts = list(img.luma_y_start)
            for i, y0 in enumerate(starts):
                last = i == len(starts) - 1
                y1 = img.bcv[0] if last else starts[i + 1]
                rc0, ref, nd0 = oracle.encode_segment(g, planes, y0, y1, last)
                hits[:] = 0
                ptr.value = hits.ctypes.data
                cap = max(1 << 16, sum(p.nbytes for p in planes))
                buf = np.zeros(cap, np.uint8)
                nb = ctypes.c_size_t(0); nd = ctypes.c_uint64(0)
                P3 = ctypes.c_void_p * 3
                rc = L.lo_encode_segment(ctypes.byref(g), P3(*[p.ctypes.data for p in planes]), y0, y1, int(last),
                                         buf.ctypes.data, cap, ctypes.byref(nb), ctypes.byref(nd))
                ptr.value = None
                assert (rc, buf[:nb.value].tobytes(), nd.value) == (rc0, ref, nd0), "the counting build codes other bits"
                h = hits.astype(np.int64)
                assert int(h.sum()) == nd0
                rows["old"].append(segment_stats(h, old_w))
                rows["new"].append(segment_stats(h, new_w))
                rows["new, global memory"].append(segment_stats(np.where(new_w >= hot, h, 0), new_w))
                tab += np.bincount(g_tab, weights=h, minlength=len(ORACLE_TABLES))
                kh += np.bincount(g_k[g_k >= 0], weights=h[g_k >= 0], minlength=11)
                front += float(h[(new_w >= 0) & (new_w < hot)].sum())
                total += nd0
            hj.close()
    nseg = len(rows["old"])
    print("%d images, %d segments; per segment (mean):" % (len(jpegs), nseg))
    print("| | decisions | distinct words | sectors touched | sectors for 50 / 80 / 90 / 95 / 99 % of decisions |")
    print("|---|---|---|---|---|")
    for name in rows:
        r = np.array([[a, b, c] + d for a, b, c, d in rows[name]], np.float64).mean(axis=0)
        print("| %s | %.0f | %.0f | %.0f | %s |" % (name, r[0], r[1], r[2], " / ".join("%.0f" % v for v in r[3:])))
    print("decision share by table: " + ", ".join("%s %.1f %%" % (nm, 100 * t / total) for (nm, _), t in zip(ORACLE_TABLES, tab)))
    ke = kh / kh.sum()
    print("exponent decisions by word k: " + ", ".join("%d: %.2f %%" % (k, 100 * v) for k, v in enumerate(ke)) +
          "; k = 0..3: %.2f %%" % (100 * ke[:4].sum()))
    print("front region (%d words, shared memory in the group decode kernel): %.1f %% of decisions" % (hot, 100 * front / total))


if __name__ == "__main__":
    main()
