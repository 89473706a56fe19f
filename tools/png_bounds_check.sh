#!/bin/bash
# The PNG encoder's GPU tests and the PNG cases of tools/sanitize_decode.py against a build in which every global and
# shared index of kernels_png.cuh is checked against its buffer (-DAPTB200_PNG_CHECK): a violation makes the encode fail
# with APT_ERR_CUDA instead of faulting.  Logs under $OUT (default tool_out/).
OUT=${OUT:-tool_out}
mkdir -p "$OUT"
LIB=${PNG_CHECK_LIB:-noaa-apt_b200/build/libaptb200_pngcheck.so}
if [ ! -f "$LIB" ]; then
    mkdir -p "$(dirname "$LIB")"
    python -c "import sys; sys.path.insert(0, 'noaa-apt_b200'); import build; build.build_library(out='$LIB', extra_flags=['-DAPTB200_PNG_CHECK'])" || exit 1
fi
APTB200_LIB=$LIB python -m pytest -m gpu tests/test_gpu_png.py tests/test_gpu_batch_png.py -q -p no:cacheprovider > $OUT/png_bounds_check.log 2>&1
echo "tests rc=$?" >> $OUT/png_bounds_check.log
APTB200_LIB=$LIB python tools/sanitize_decode.py 1 >> $OUT/png_bounds_check.log 2>&1
echo "sanitize_decode rc=$?" >> $OUT/png_bounds_check.log
tail -6 $OUT/png_bounds_check.log
