"""Diagnostic (not a test): restore throughput of container version 3 (rANS-coded streams) through the file API, against
the same corpus as version-1 files.

Config 2's corpus (1080p 4:2:0 q85, 32 distinct images replicated to N files): the 32 distinct JPEGs are compressed once
by the reference built with the ANS coder (oracle/_ref/lepton-ans -ans, on the host) and once by this library (version 1);
then `decompress` is timed over N files of each kind, alternated round by round on one codec.  Every restore is checked
against the input JPEGs.  Prints one JSON line with the card, its power limit and the times.

    python tests/tools_ans_e2e.py [files] [rounds]
"""
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from lepton_b200 import LeptonB200FileCodec  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 2048
rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 5
distinct = bench.make_corpus(2, 32)
jpegs = [distinct[i % 32] for i in range(n)]
tot = sum(len(j) for j in jpegs)
ans = []
with tempfile.TemporaryDirectory() as tmp:
    for k, j in enumerate(distinct):
        src, dst = os.path.join(tmp, "%d.jpg" % k), os.path.join(tmp, "%d.lep" % k)
        with open(src, "wb") as f:
            f.write(j)
        subprocess.run([os.path.join(ROOT, "oracle", "_ref", "lepton-ans"), "-unjailed", "-ans", "-skipverify", src, dst],
                       check=True, capture_output=True)
        ans.append(open(dst, "rb").read())
        assert ans[-1][2] == 3
fc = LeptonB200FileCodec(0, host_threads=16)
r = fc.compress(distinct)
assert all(st == 0 for st, _ in r)
handles = {"version1": LeptonB200FileCodec.prepare([r[i % 32][1] for i in range(n)]),
           "version3_rans": LeptonB200FileCodec.prepare([ans[i % 32] for i in range(n)])}
for name, h in handles.items():
    got = fc.decompress(h)
    assert all(st == 0 and out == j for (st, out), j in zip(got, jpegs)), name
times = {k: [] for k in handles}
for _ in range(rounds):
    for name, h in handles.items():
        t0 = time.perf_counter()
        fc.decompress(h, copy=False)
        times[name].append(time.perf_counter() - t0)
fc.close()
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
except (OSError, IndexError):
    card = "unknown"
res = {"files": n, "jpeg_bytes": tot, "rounds": rounds, "lep_bytes_v1": sum(len(r[i % 32][1]) for i in range(n)),
       "lep_bytes_v3": sum(len(ans[i % 32]) for i in range(n)), "card": card}
for name, ts in times.items():
    res[name] = {"min_s": round(min(ts), 4), "median_s": round(statistics.median(ts), 4),
                 "MB_per_s_at_median": round(tot / statistics.median(ts) / 1e6, 1), "all_s": [round(t, 4) for t in ts]}
print(json.dumps(res))
