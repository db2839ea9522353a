#!/bin/bash
# re-tune of the wgmma tile-conv kernel's A/B knobs (SIGE_TC5_*), each arm timed twice in one run
run() { env $1 timeout 200 python bench.py --steps 100 --warmup 10 --no-cpu-baseline --no-reference-cuda $2 2>/dev/null | python -c "import json,sys; d=json.loads(sys.stdin.read().strip().splitlines()[-1]); print('[$1 $2]', round(d['ms_per_step'],4), round(d['e2e']['ms_per_step'],4), d['roofline'].get('sum_in_graph_us'))"; }
for rep in 1 2; do for arm in "A=0" "SIGE_TC5_DEEP=2" "SIGE_TC5_MIN_TAPS=2" "SIGE_TC5_MIN_TAPS=5" "SIGE_TC5_LATE_TRIGGER=0"; do run "$arm" ""; done; done
for arm in "A=0" "SIGE_TC5_DEEP=2"; do run "$arm" "--edits 8"; run "$arm" "--ratio 0.30"; done
