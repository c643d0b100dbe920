#!/bin/bash
# compute-sanitizer racecheck / synccheck / memcheck over every hand-written kernel
# family on the tiny geometry (tools/sanitize_target.py).  usage: tools/sanitize_box.sh r2 [per-run timeout s]
#   -> $OUT/sanitizer_<tag>_<tool>_<part>.log (OUT defaults to prof_out) + a one-line summary per run on stdout
R=${1:-r2}
TMO=${2:-300}
OUT=${OUT:-prof_out}
mkdir -p "$OUT"
run() {
  timeout $TMO compute-sanitizer --tool $1 --print-limit 20 python tools/sanitize_target.py $2 \
    > "$OUT/sanitizer_${R}_$1_$2.log" 2>&1
  echo "$1 $2 exit=$? : $(grep -E 'ERROR SUMMARY|RACECHECK SUMMARY|OK ' "$OUT/sanitizer_${R}_$1_$2.log" | tr '\n' ' ')"
}
for part in fused split batch; do run racecheck $part; run synccheck $part; done
for part in fused split batch codec prefill; do run memcheck $part; done
for part in codec prefill; do run racecheck $part; run synccheck $part; done
