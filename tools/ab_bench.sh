#!/usr/bin/env bash
# Interleaved A/B runs of bench.py on ONE box (run-to-run noise between boxes is larger than most kernel effects):
#   tools/ab_bench.sh <out-prefix> <rounds> "ENV_A" "ENV_B" ...
# e.g. tools/ab_bench.sh /tmp/ab 2 "" "PGQ_B200_PULL_SKIP=0"
# writes <out-prefix>_<variant index>_<round>.json (the bench line) and prints pairs/s, ms per step and the
# bottom-up level's average time per variant.
set -euo pipefail
prefix=$1; rounds=$2; shift 2
for r in $(seq 1 "$rounds"); do
  i=0
  for envs in "$@"; do
    env $envs python bench.py --no-extra --steps 20 > "${prefix}_${i}_${r}.json" 2> "${prefix}_${i}_${r}.err" || true
    python - "$i" "$envs" "${prefix}_${i}_${r}.json" <<'PY'
import json, sys
try:
    j = json.loads(open(sys.argv[3]).read().strip().splitlines()[-1])
    d = j["roofline"]["dominant"]
    print(f"variant {sys.argv[1]} [{sys.argv[2] or 'default'}]: {j['value']:.0f} pairs/s, {j['ms_per_step']:.3f} ms/step, "
          f"bottom-up level {d['ms']:.4f} ms x {d['launches_per_step']}/step, clocks {j['clocks'].get('sm_mhz')}")
except Exception as ex:
    print(f"variant {sys.argv[1]} [{sys.argv[2]}]: failed ({ex})")
PY
    i=$((i + 1))
  done
done
