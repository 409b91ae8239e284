#!/bin/bash
# Times the C3 check kernel under experiment switches of the run-time specialised build (one bench.py run per variant;
# kernel_ms_mean = CUDA events around the check kernel alone).  Usage (needs a GPU): tools/uc_variants.sh [requests]
# The stub_* variants replace one phase of cb::eval_request_uc by a trivial stand-in whose result is still stored
# (cb_core.h: CB_UC_STUB_*; their decisions are wrong, hence --no-verify): default minus stub = that phase's share.
# stub_lists drops the list loads and compares, stub_list_probes only the compares (list_probe, list_mask).
# stub_fallback keeps only the typed branch of a table that has one (the path a request of well-typed attributes runs).
# no_list_pf drops the prefetch of the next chunk's list headers (cb_kernels.h: check_uc_body; results unchanged).
OUT=${OUT:-profile_out}; mkdir -p "$OUT"
N=${1:-16777216}
out=$OUT/uc_variants.txt
: > "$out"
run() {
    name=$1; shift
    line=$(env "$@" python bench.py --requests $N --steps 5 --warmup 3 --no-cpu --no-e2e --no-secondary --no-verify 2>$OUT/uc_variant_$name.err | tail -1)
    echo "$name $(echo "$line" | python -c 'import sys,json; d=json.load(sys.stdin); r=d["roofline"]; print(r["kernel_ms_mean"], r["frac"], d["config"]["kernel"]["grid"])' 2>&1)" | tee -a $out
}
run default X=1
run stub_walk CERBOS_B200_SPEC_DEFS=-DCB_UC_STUB_WALK
run stub_lists CERBOS_B200_SPEC_DEFS=-DCB_UC_STUB_LISTS
run stub_list_probes CERBOS_B200_SPEC_DEFS=-DCB_UC_STUB_LIST_PROBES
run stub_strpred CERBOS_B200_SPEC_DEFS=-DCB_UC_STUB_STRPRED
run stub_fallback CERBOS_B200_SPEC_DEFS=-DCB_UC_STUB_FALLBACK
run stub_terms CERBOS_B200_SPEC_DEFS=-DCB_UC_STUB_TERMS
run no_list_pf CERBOS_B200_SPEC_DEFS=-DCB_UC_NO_LIST_PF
run keys64 CERBOS_B200_SPEC_DEFS=-DCB_LIST_KEYS64
run blocks3 CERBOS_B200_SPEC_UC_BLOCKS=3
run blocks4 CERBOS_B200_SPEC_UC_BLOCKS=4
run blocks5 CERBOS_B200_SPEC_UC_BLOCKS=5
