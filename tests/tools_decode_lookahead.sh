#!/bin/bash
# Group decode kernel with the count trees read ahead vs the build of the parent commit, on an H100: A/B of the bench
# line, byte comparison of the dumped outputs, the GPU tests, smoke(), the decode crossover and the full bench line.
# Build both first:
#   git worktree add /tmp/base HEAD~1 && (cd /tmp/base && python -m lepton_b200.build --variant base)
#   cp /tmp/base/lepton_b200/variants/libbase.so lepton_b200/variants/ && python -c "import __graft_entry__ as g; g.build()"
# then run this script from the repository root:  bash tests/tools_decode_lookahead.sh [OUTPUT_DIR]
# Everything it writes goes under OUTPUT_DIR (default: a new temporary directory).
O=${1:-$(mktemp -d)}
mkdir -p "$O"
echo "== output: $O"
BASE=$PWD/lepton_b200/variants/libbase.so
NEW=$PWD/lepton_b200/liblepton_b200.so
date +%s > $O/t0
el() { echo "$(( $(date +%s) - $(cat $O/t0) )) s"; }
show() {   # value, per-direction kernel time and the clock samples of one bench line
  python -c "
import json, sys
d = json.loads(open(sys.argv[1]).read().strip().splitlines()[-1])
print('%-5s value %.1f MB/s  decode %.1f ms  encode %.1f ms  roundtrip %s  clocks %s' % (sys.argv[2], d['value'], d['decode']['ms_per_step'],
      d['encode']['ms_per_step'], d['roundtrip_pass_rate'], json.dumps(d.get('clocks'))[:300]))" "$1" "$2"
}
lib() { [ "$1" = base ] && echo "$BASE" || echo "$NEW"; }

echo "== card"; nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv
echo "== A/B, alternating ($(el))"
for i in 1 2 3; do
  for v in base new; do
    LEPB200_LIBRARY=$(lib $v) timeout 240 python bench.py --no-e2e --no-cpu-baseline --steps 5 --warmup 3 > $O/ab_${v}_$i.json 2> $O/ab_${v}_$i.err
    show $O/ab_${v}_$i.json $v || tail -3 $O/ab_${v}_$i.err
  done
done
echo "== outputs of both builds ($(el))"
for v in base new; do
  LEPB200_LIBRARY=$(lib $v) timeout 240 python bench.py --no-e2e --no-cpu-baseline --steps 1 --warmup 1 --dump-outputs $O/dump_$v > $O/dump_$v.json 2> $O/dump_$v.err || tail -3 $O/dump_$v.err
done
for f in $O/dump_base/*.npy; do cmp -s "$f" "$O/dump_new/$(basename $f)" && echo "same   $(basename $f)" || echo "DIFFER $(basename $f)"; done
echo "== pytest -m gpu ($(el))"; timeout 600 python -m pytest tests -m gpu -q 2>&1 | tail -4
echo "== smoke ($(el))"; timeout 120 python -c "import __graft_entry__ as g; g.smoke(); print('smoke ok')" 2>&1 | tail -2
echo "== crossover: warp kernel (1) / group kernel (2) ($(el))"
for n in 1024 1536; do
  for m in 1 2; do
    LEPB200_DEC_MODE=$m timeout 180 python bench.py --no-e2e --no-cpu-baseline --images $n --steps 3 --warmup 2 > $O/x_${n}_$m.json 2> $O/x_${n}_$m.err
    python -c "
import json, sys
d = json.loads(open(sys.argv[1]).read().strip().splitlines()[-1])
print('%d segments, mode %s: decode %.1f ms' % (4 * int(sys.argv[2]), sys.argv[3], d['decode']['ms_per_step']))" $O/x_${n}_$m.json $n $m || tail -3 $O/x_${n}_$m.err
  done
done
echo "== full bench line of the new build ($(el))"
timeout 420 python bench.py > $O/full.json 2> $O/full.err; tail -c 3000 $O/full.json; tail -3 $O/full.err
echo "== done ($(el))"
