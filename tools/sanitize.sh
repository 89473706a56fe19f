#!/bin/bash
# compute-sanitizer memcheck + racecheck over small decodes of every resampler path and a small PNG encode; logs under $OUT (default tool_out/).
OUT=${OUT:-tool_out}
mkdir -p "$OUT"
CS=/usr/local/cuda/bin/compute-sanitizer
timeout 900 $CS --tool memcheck --print-limit 20 python tools/sanitize_decode.py > $OUT/sanitizer_memcheck.log 2>&1
echo "memcheck rc=$?" >> $OUT/sanitizer_memcheck.log
timeout 900 $CS --tool racecheck --print-limit 20 python tools/sanitize_decode.py 2 > $OUT/sanitizer_racecheck.log 2>&1
echo "racecheck rc=$?" >> $OUT/sanitizer_racecheck.log
tail -4 $OUT/sanitizer_memcheck.log $OUT/sanitizer_racecheck.log
