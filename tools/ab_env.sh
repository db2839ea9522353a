#!/bin/bash
# A/B of environment knobs of the kernels inside ONE run on the GPU (box-to-box variation is ~2 %):
#   bash tools/ab_env.sh "" "SIGE_TC5_PAIR_FIT=1" ...      (each argument = one arm's environment, "" = defaults)
run() { env $1 timeout 200 python bench.py --steps 200 --warmup 20 --no-cpu-baseline --no-reference-cuda $F 2>/dev/null | python -c "import json,sys; d=json.loads(sys.stdin.read().strip().splitlines()[-1]); print('[$1 $F]', round(d['ms_per_step'],4), round(d['e2e']['ms_per_step'],4), d['roofline'].get('sum_in_graph_us'))"; }
for rep in 1 2 3; do for arm in "$@"; do run "$arm"; done; done
