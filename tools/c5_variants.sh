#!/bin/bash
# C5 specialised kernel: resident CTAs / SM the kernel is budgeted for (launch bounds -> registers per thread)
OUT=${OUT:-profile_out}; mkdir -p "$OUT"
for UB in ${@:-2 3 4}; do
  CERBOS_B200_SPEC_UC_BLOCKS=$UB python bench.py --workload C5 --steps 5 --warmup 3 --no-e2e --no-cpu --no-secondary > $OUT/c5_ub$UB.json 2> $OUT/c5_ub$UB.err
  python - <<PY
import json
d = json.load(open("$OUT/c5_ub$UB.json"))
print("UC_BLOCKS=$UB value %.3e kernel_ms %.4f frac %.3f grid %d verified %s" % (d["value"], d["roofline"]["kernel_ms_mean"], d["roofline"]["frac"], d["config"]["kernel"]["grid"], d["verified_vs_oracle"]))
PY
done
