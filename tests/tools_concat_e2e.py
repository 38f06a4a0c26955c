"""Diagnostic (not a test): restoring N .lep files passed as N buffers against the same N files as ONE concatenated buffer.

The files are the reference's version-2 members committed under tests/golden/concat/ (the default version-1 container has
no EOF marker, so only -brotliheader files can be concatenated), cycled to N.  Both forms go through `decompress` on one
codec, alternated round by round; the concatenated restore must equal the separate restores joined.  Prints one JSON line
with the card, its power limit, the kernel launches of each form and the times.

    python tests/tools_concat_e2e.py [files] [rounds]
"""
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from lepton_b200 import LeptonB200FileCodec  # noqa: E402
from make_concat import member  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 2048
rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 7
NAMES = ["androidcrop", "androidtrail", "colorswap", "narrowrst", "tall_t1", "tall_t4", "tall_t8", "trailingrst2"]
files = [member(NAMES[i % len(NAMES)]) for i in range(n)]
stream = b"".join(files)
fc = LeptonB200FileCodec(0, host_threads=16)
forms = {"separate": LeptonB200FileCodec.prepare(files), "concatenated": LeptonB200FileCodec.prepare([stream])}
sep = fc.decompress(forms["separate"])
assert all(st == 0 for st, _ in sep)
one = fc.decompress(forms["concatenated"])
assert one[0][0] == 0 and one[0][1] == b"".join(b for _, b in sep)
jpeg_bytes = len(one[0][1])
launches = {}
for name, h in forms.items():
    k0 = fc.kernel_launches
    fc.decompress(h, copy=False)
    launches[name] = fc.kernel_launches - k0
times = {k: [] for k in forms}
for _ in range(rounds):
    for name, h in forms.items():
        t0 = time.perf_counter()
        fc.decompress(h, copy=False)
        times[name].append(time.perf_counter() - t0)
fc.close()
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
except (OSError, IndexError):
    card = "unknown"
res = {"files": n, "lep_bytes": len(stream), "jpeg_bytes": jpeg_bytes, "rounds": rounds, "card": card, "kernel_launches": launches}
for name, ts in times.items():
    res[name] = {"min_s": round(min(ts), 4), "median_s": round(statistics.median(ts), 4),
                 "MB_per_s_at_median": round(jpeg_bytes / statistics.median(ts) / 1e6, 1), "all_s": [round(t, 4) for t in ts]}
print(json.dumps(res))
