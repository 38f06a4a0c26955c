"""Encode time with the planes resident in HBM, bool coder against rANS coder (container version 3), on the bench corpus
(synthetic 1920x1080 4:2:0 q=85 baseline JPEGs, bench.py's config 2; `distinct` of them repeated to --images).

For each coder the batch is uploaded once and launched --steps times after --warmup launches; per launch the library's
events give kernel A (lepb200_last_symbolise_ms: from the first kernel A launch to the last) and the whole encode
(lepb200_last_kernel_ms); the entropy pass is their difference (range coder, or the rANS pass).  Prints one JSON line per
coder, with the GPU's name and power limit.  Needs a GPU; there is no CPU path.

    python tests/tools_ans_encode_bench.py --images 2048 --distinct 32 --steps 5 --warmup 1
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=2048)
    ap.add_argument("--distinct", type=int, default=32)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import bench
    from lepton_b200 import HostJpeg, LeptonB200Codec
    from lepton_b200.codec import CODER_ANS, CODER_BOOL
    jpegs = bench.make_corpus(2, args.distinct)
    hjs = [HostJpeg(j) for j in jpegs]
    base = [h.coef_image() for h in hjs]
    imgs = [base[i % len(base)] for i in range(args.images)]
    nseg = sum(im.nseg for im in imgs)
    codec = LeptonB200Codec(0)
    info = gpu_info()
    for name, coder in (("bool", CODER_BOOL), ("ans", CODER_ANS)):
        codec.encode_upload(imgs, coders=[coder] * len(imgs))
        a_ms, tot_ms = [], []
        for step in range(args.warmup + args.steps):
            codec.encode_launch()
            codec.sync()
            if step >= args.warmup:
                tot_ms.append(codec.last_kernel_ms)
                a_ms.append(codec.last_symbolise_ms)
        res = codec.encode_fetch()
        nbytes = sum(len(s.data) for r in res for s in r)
        assert all(s.status == 0 for r in res for s in r)
        ent = [t - a for t, a in zip(tot_ms, a_ms)]
        print(json.dumps(dict(coder=name, images=len(imgs), segments=nseg, decisions=sum(s.ndecisions for r in res for s in r),
                              stream_bytes=nbytes, kernel_a_ms=round(statistics.median(a_ms), 2),
                              entropy_ms=round(statistics.median(ent), 2), entropy_ms_all=[round(x, 2) for x in ent],
                              encode_ms=round(statistics.median(tot_ms), 2), gpu=info)), flush=True)
    codec.close()


if __name__ == "__main__":
    main()
