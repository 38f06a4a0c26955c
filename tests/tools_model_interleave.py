"""Hot set of the group decode kernel's interleaved model pool on bench-like input (CPU only; a tool, not a test).

    python tests/tools_model_interleave.py [n_images]

Counts the branch uses of every thread-segment of `n_images` JPEGs of the benchmark's corpus with the counting build of
the C oracle of tests/tools_model_hotset.py (same images, same check of the streams), and keeps the words outside the
front region, which the group kernel reads through the L2.  It then lays those words out as the kernel's pool does
(lep_common.cuh, mi_offset): B-byte unit u of model k of a block of K models at unit u * K + k, with K * B = 32, so that
one 32-byte sector holds unit u of all K models.  The segments go into blocks in the library's queue order (largest first,
lep_plan.cuh: a stable sort by block count), K consecutive segments per block, and the sectors a block touches, and those
that cover 50 / 80 / 90 / 95 / 99 % of its decisions, are divided among its segments.  `B = 32, K = 1` is the private
layout (the row `new, global memory` of tools_model_hotset.py).
"""
import ctypes
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import oracle  # noqa: E402
from tools_model_hotset import N_BRANCHES, counting_oracle, layout  # noqa: E402


def block_stats(hits, words, unit_words):
    """sectors touched and sectors for each share of the decisions of a block of segments (their hit arrays `hits`) whose
    models share the sectors of unit_words-word units, per segment"""
    h = np.sum(hits, axis=0)
    used = h > 0
    nd = int(h.sum())
    sec = np.bincount(words[used] // unit_words, weights=h[used].astype(np.float64))
    sec = np.sort(sec[sec > 0])[::-1]
    cum = np.cumsum(sec) / nd
    cover = [int(np.searchsorted(cum, f - 1e-12) + 1) for f in (0.5, 0.8, 0.9, 0.95, 0.99)]
    return [len(sec) / len(hits)] + [c / len(hits) for c in cover]


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 2
    import bench
    from lepton_b200 import HostJpeg
    from lepton_b200.codec import lib
    jpegs = bench.make_corpus(2, n)
    words, total, hot = layout(True)
    assert total * 2 == lib().lepb200_model_bytes(), "layout() disagrees with lep_common.cuh"
    segs = []            # (blocks, hits outside the front region) of every segment, in batch order
    with tempfile.TemporaryDirectory() as tmp:
        L = counting_oracle(tmp)
        hits = np.zeros(N_BRANCHES, np.uint64)
        ptr = ctypes.c_void_p.in_dll(L, "lo_hits")
        P3 = ctypes.c_void_p * 3
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
                rc = L.lo_encode_segment(ctypes.byref(g), P3(*[p.ctypes.data for p in planes]), y0, y1, int(last),
                                         buf.ctypes.data, cap, ctypes.byref(nb), ctypes.byref(nd))
                ptr.value = None
                assert (rc, buf[:nb.value].tobytes(), nd.value) == (rc0, ref, nd0), "the counting build codes other bits"
                h = hits.astype(np.int64)
                blocks = sum(bch * ((y1 - y0) * bcv // img.bcv[0]) for bch, bcv in zip(img.bch, img.bcv))
                segs.append((blocks, np.where(words >= hot, h, 0)))
            hj.close()
    queue = [h for _, h in sorted(segs, key=lambda t: -t[0])]          # stable: largest first, then batch order
    print("%d images, %d segments; global memory, K models interleaved in B-byte units (per segment, mean over the blocks):"
          % (len(jpegs), len(queue)))
    print("| layout | sectors touched | sectors for 50 / 80 / 90 / 95 / 99 % of decisions |")
    print("|---|---|---|")
    for b in (32, 16, 8, 4, 2):
        k = 32 // b
        r = np.array([block_stats(queue[i:i + k], words, b // 2) for i in range(0, len(queue), k)]).mean(axis=0)
        print("| B = %d B, K = %d | %.0f | %s |" % (b, k, r[0], " / ".join("%.0f" % v for v in r[1:])))


if __name__ == "__main__":
    main()
