#!/bin/bash
# Nsight Compute evidence for profiles/ (one GPU, ncu on PATH).
#   1. kernel launch list of one bench step (time shares)
#   2. full capture of one steady-state 8-frame launch of the single-sequence persistent decode kernel
#   3. full capture of one launch of the batched decode kernel (32 slots)
#   4. full captures of the wgmma GEMM launches of one codec window decode (T=33)
# The CSV exports and the decode kernel's .ncu-rep go to $OUT (default prof_out/).
# usage: tools/profile_box.sh r2   -> $OUT/{launches,prof_decode,prof_batch,prof_gemm}_<tag>*
R=${1:-r2}
OUT=${OUT:-prof_out}
mkdir -p "$OUT"
B="python bench.py --steps 1 --warmup 1 --no-cpu-baseline --no-gpu-reference --no-stateful"
ncu --metrics gpu__time_duration.sum --clock-control none -s 600 -c 6000 --csv --log-file "$OUT/launches_$R.csv" \
    $B --batch 0 > "$OUT/ncu_launch_$R.log" 2>&1
ncu --set full --clock-control none --import-source on -k regex:fq3_decode_kernel -s 3 -c 1 -f -o "$OUT/prof_decode_$R" \
    $B --batch 0 > "$OUT/ncu_full_$R.log" 2>&1
ncu -i "$OUT/prof_decode_$R.ncu-rep" --page raw --csv > "$OUT/prof_decode_${R}_raw.csv" 2>/dev/null
ncu --set full --clock-control none -k regex:fq3_decode_batch_kernel -s 2 -c 1 -f -o /tmp/prof_batch_$R \
    python tools/batch_bench.py --batches 32 --frames 16 > "$OUT/ncu_batch_$R.log" 2>&1
ncu -i /tmp/prof_batch_$R.ncu-rep --page raw --csv > "$OUT/prof_batch_${R}_raw.csv" 2>/dev/null
ncu --set full --clock-control none -k regex:conv_gemm_tc_kernel -s 200 -c 24 -f -o /tmp/prof_gemm_$R \
    python tools/codec_bench3.py --cases 1x33 > "$OUT/ncu_gemm_$R.log" 2>&1
ncu -i /tmp/prof_gemm_$R.ncu-rep --page raw --csv > "$OUT/prof_gemm_${R}_raw.csv" 2>/dev/null
du -sh "$OUT"; ls -la "$OUT" | grep -E "prof_|launches_" | awk '{print $5, $9}'
