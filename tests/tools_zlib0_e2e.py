"""Diagnostic (not a test): what zlib0 output costs when restoring .lep files through the file API.

Config 2's corpus (1080p 4:2:0 q85, 32 distinct images replicated to N files) is compressed once, then `decompress` is timed
in two settings on one codec, alternated round by round: zlib0 off; zlib0 on (the Adler-32 of device-encoded scans from
the encode kernel).  The zlib0 output is checked against the plain restore.  Prints one JSON line with the card, its power limit and the times.

    python tests/tools_zlib0_e2e.py [files] [rounds]
"""
import json
import os
import statistics
import subprocess
import sys
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from lepton_b200 import LeptonB200FileCodec  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 2048
rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 5
distinct = bench.make_corpus(2, 32)
jpegs = [distinct[i % 32] for i in range(n)]
tot = sum(len(j) for j in jpegs)
fc = LeptonB200FileCodec(0, host_threads=16)
r = fc.compress(jpegs)
assert all(st == 0 for st, _ in r)
handle = LeptonB200FileCodec.prepare([b for _, b in r])

SETTINGS = {"plain": 0, "zlib0_kernel_adler": 1}


def use(name):
    fc._L.lepb200_codec_set_zlib0(fc._c, SETTINGS[name])


# outputs first: every setting restores every file, and the zlib streams hold the plain JPEGs
use("plain")
plain = fc.decompress(handle)
assert all(st == 0 and out == j for (st, out), j in zip(plain, jpegs))
gpu_recoded = fc.last_gpu_recoded
use("zlib0_kernel_adler")
got = fc.decompress(handle)
for k in range(0, n, 97):
    assert got[k][0] == 0 and zlib.decompress(got[k][1]) == plain[k][1], k
assert fc.last_gpu_recoded == gpu_recoded
times = {k: [] for k in SETTINGS}
for _ in range(rounds):
    for name in SETTINGS:
        use(name)
        fc.decompress(handle, copy=False)               # warm: output buffers at their zlib0 size
        t0 = time.perf_counter()
        fc.decompress(handle, copy=False)
        times[name].append(time.perf_counter() - t0)
fc.close()
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
except (OSError, IndexError):
    card = "unknown"
res = {"files": n, "jpeg_bytes": tot, "rounds": rounds, "gpu_recoded": gpu_recoded, "card": card}
for name, ts in times.items():
    res[name] = {"min_s": round(min(ts), 4), "median_s": round(statistics.median(ts), 4), "MB_per_s_at_median": round(tot / statistics.median(ts) / 1e6, 1),
                 "all_s": [round(t, 4) for t in ts]}
print(json.dumps(res))
