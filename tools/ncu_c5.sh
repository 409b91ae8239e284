#!/bin/bash
# ncu --set full capture of one cb_spec_uc_global launch on C5 (2^18 requests) + summaries under $OUT (default profile_out/).
OUT=${OUT:-profile_out}; mkdir -p "$OUT"
N=${1:-262144}
export CERBOS_B200_SPEC_DUMP=$OUT/spec_c5.cu
export CERBOS_B200_CACHE_DIR=$OUT/cache_c5
rm -rf $OUT/cache_c5; mkdir -p $OUT/cache_c5
ncu --set full --import-source on --clock-control none -k regex:cb_spec_uc -s 5 -c 1 -o $OUT/c5_uc -f \
    python bench.py --workload C5 --requests $N --steps 1 --warmup 3 --batches-per-step 1 --no-e2e --no-cpu --no-verify --no-secondary > $OUT/ncu_c5.log 2>&1
python tools/ncu_summary.py $OUT/c5_uc.ncu-rep > $OUT/c5_uc_ncu_full.json 2>>$OUT/ncu_c5.log
python tools/ncu_spec_lines.py $OUT/c5_uc.ncu-rep $(ls $OUT/cache_c5/*.cubin | head -1) $OUT/spec_c5.cu 80 > $OUT/c5_uc_lines.txt 2>>$OUT/ncu_c5.log
tail -3 $OUT/ncu_c5.log; head -c 400 $OUT/c5_uc_ncu_full.json
