#!/bin/bash
# A/B timing of the working tree against a control build, inside ONE run on the GPU (box-to-box variation is ~2 %, the
# effects being chased are 1-5 %).  Control = a copy of a commit with its own library under _base/ (git-ignored):
#   rm -rf _base && mkdir _base && git archive HEAD | tar -x -C _base && (cd _base && python -m sige_b200.build)
# Usage on the GPU box:  bash tools/ab.sh [ENV=VALUE ...]     (the variables go to the NEW arm only)
run() { env "$@" timeout 200 python bench.py --steps 100 --warmup 10 --no-cpu-baseline $F 2>/dev/null | python -c "import json,sys; d=json.loads(sys.stdin.read().strip().splitlines()[-1]); print('[$* $F]', round(d['ms_per_step'],4), round(d['e2e']['ms_per_step'],4))"; }
for rep in 1 2 3; do
  if [ -d _base ]; then (cd _base && F="" run BASE=1); fi
  F="" run NEW=1 "$@"
done
