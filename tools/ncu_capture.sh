#!/bin/bash
# Profile capture with Nsight Compute; output under $OUT (default tool_out/).  Numbers printed by runs under ncu are never bench values.
#   tools/ncu_capture.sh <tag> [kernel-regex]
TAG=${1:-r02}
KRE=${2:-'k_polyphase_ut|k_lowpass_records|k_resolve_roots|k_pick_cluster|k_pick_links|k_gather_rows_lp'}
OUT=${OUT:-tool_out}
mkdir -p "$OUT"
# (1) launch list: per-launch durations of three decodes
timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none -c 60 --csv --log-file $OUT/${TAG}_launches.csv \
    python tools/one_decode.py > $OUT/ncu_${TAG}.log 2>&1
# (2) one full capture of each kernel of the last decode
timeout 900 ncu --set full --clock-control none --import-source on -k "regex:${KRE}" --launch-skip 10 --launch-count 5 \
    -o $OUT/${TAG}_full -f python tools/one_decode.py >> $OUT/ncu_${TAG}.log 2>&1
ls -la $OUT/*.ncu-rep | tail -3
# (3) DRAM traffic in application order: caches are NOT flushed between kernels and the two counters fit one pass (no replay),
#     so e -- written by the resampler, read by the record and gather kernels -- is served from L2 as in a real decode
timeout 300 ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum --cache-control none --clock-control none \
    -k "regex:${KRE}" --launch-skip 10 --launch-count 5 --csv --log-file $OUT/${TAG}_dram_warm.csv \
    python tools/one_decode.py >> $OUT/ncu_${TAG}.log 2>&1
tail -12 $OUT/${TAG}_dram_warm.csv
