#!/bin/bash
# occupancy experiment: device-resident value of the bench workload with fewer persistent stage-1 CTAs (SMs left free for the
# kernels of the other streams)
cd "$(dirname "$0")/.."
out=$(mktemp -d)
trap 'rm -rf "$out"' EXIT
for ctas in 0 132 120 104 88; do
    timeout 300 python bench.py --quick --steps 8 --warmup 4 --no-cpu --c3 0 --c4 0 --ft s1_ctas=$ctas > "$out/prio.json" 2> "$out/prio.err"
    python - "$ctas" "$out/prio.json" <<'PY'
import json,sys
try:
    d=json.loads(open(sys.argv[2]).read().strip().splitlines()[-1])
    g={x['group']:round(x['avg_ms']*1e3,1) for x in d['roofline']['by_group']}
    print(sys.argv[1], round(d['value']), g)
except Exception as e:
    print(sys.argv[1], 'failed', e)
PY
done
