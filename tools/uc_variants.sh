#!/bin/bash
# Times the C3 check kernel under experiment switches of the run-time specialised build (one bench.py run per variant;
# kernel_ms_mean = CUDA events around the check kernel alone).  Usage (needs a GPU): tools/uc_variants.sh [requests]
OUT=${OUT:-profile_out}; mkdir -p "$OUT"
N=${1:-4194304}
out=$OUT/uc_variants.txt
: > "$out"
run() {
    name=$1; shift
    line=$(env "$@" python bench.py --requests $N --steps 5 --warmup 3 --no-cpu --no-e2e --no-secondary --no-verify 2>$OUT/uc_variant_$name.err | tail -1)
    echo "$name $(echo "$line" | python -c 'import sys,json; d=json.load(sys.stdin); r=d["roofline"]; print(r["kernel_ms_mean"], r["frac"], d["config"]["kernel"]["grid"])' 2>&1)" | tee -a $out
}
run default X=1
run keys64 CERBOS_B200_SPEC_DEFS=-DCB_LIST_KEYS64
run blocks3 CERBOS_B200_SPEC_UC_BLOCKS=3
run blocks5 CERBOS_B200_SPEC_UC_BLOCKS=5
run blocks6 CERBOS_B200_SPEC_UC_BLOCKS=6
