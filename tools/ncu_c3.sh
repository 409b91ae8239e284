#!/bin/bash
# ncu --set full capture of one cb_spec_uc launch on C3 (2^22 requests) + summaries under $OUT (default profile_out/).
OUT=${OUT:-profile_out}; mkdir -p "$OUT"
export CERBOS_B200_SPEC_DUMP=$OUT/spec_uc.cu
export CERBOS_B200_CACHE_DIR=$OUT/cache
rm -rf $OUT/cache; mkdir -p $OUT/cache
ncu --set full --import-source on --clock-control none -k regex:cb_spec_uc -s 3 -c 1 -o $OUT/c3_uc -f \
    python bench.py --workload C3 --requests 4194304 --steps 1 --warmup 3 --no-e2e --no-cpu --no-verify --no-secondary > $OUT/ncu_c3.log 2>&1
python tools/ncu_summary.py $OUT/c3_uc.ncu-rep > $OUT/c3_uc_ncu_full.json 2>>$OUT/ncu_c3.log
python tools/ncu_spec_lines.py $OUT/c3_uc.ncu-rep $(ls $OUT/cache/*.cubin | head -1) $OUT/spec_uc.cu 70 > $OUT/c3_uc_lines.txt 2>>$OUT/ncu_c3.log
tail -3 $OUT/ncu_c3.log
