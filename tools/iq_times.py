"""Times of the I/Q stage (DESIGN.md §10).  Prints one JSON line and writes $OUT/iq_times.json (default tool_out/).
    python tools/iq_times.py [--seconds-cu8 900] [--seconds-cs16 300] [--seconds-cf32 150]
  - k_fm_demod device time (torch.profiler, summed over the chunk launches of one apt_fm_demod) for a 2.4 Msps pass in
    each format, with its share of the data-sheet bound that binds it (bytes b*n + 4*n/D, flops 4*N*n/D + 6*n);
  - apt_decode_iq wall time of the cu8 pass from pageable host memory;
  - the I/Q stream (Stream.for_iq): seconds of signal per wall second in 0.5 s pushes."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

import noaa_apt_b200 as na
from noaa_apt_b200 import synth

# H100 SXM5 data sheet: FP32 (non-tensor) and HBM3 bandwidth
PEAK_FLOPS = 67e12
PEAK_BYTES = 3.35e12

ap = argparse.ArgumentParser()
ap.add_argument("--seconds-cu8", type=float, default=900)
ap.add_argument("--seconds-cs16", type=float, default=300)
ap.add_argument("--seconds-cf32", type=float, default=150)
args = ap.parse_args()

res = {}
try:
    res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as e:                                              # noqa: BLE001
    res["gpu"] = f"unknown ({e})"

fs = 2_400_000
s = na.iq.IqSettings(fs, offset_hz=37_000)
D = s.decimation
from oracle import design, freq_hz, FILTER_LOWPASS   # noqa: E402  tap count only
N = design(FILTER_LOWPASS, freq_hz(s.cutout, fs), s.atten, freq_hz(s.delta_freq, fs)).size
res["settings"] = {"iq_rate": fs, "audio_rate": s.audio_rate, "D": D, "taps": N, "offset_hz": s.offset_hz}
one_s = {fmt: synth.apt_iq(fs, 1.0, seed=1, offset_hz=s.offset_hz, fmt=fmt) for fmt in ("cu8", "cs16", "cf32")}


def kernel_ms(x):
    na.iq.fm_demod(x[: x.size // 50], s)                     # warm-up: tables, attributes
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        na.iq.fm_demod(x, s)
    us = [ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
          for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA and "k_fm_demod" in ev.name]
    return float(np.sum(us)) / 1e3, len(us)


res["k_fm_demod"] = {}
for fmt, secs, b in (("cu8", args.seconds_cu8, 2), ("cs16", args.seconds_cs16, 4), ("cf32", args.seconds_cf32, 8)):
    x = np.tile(one_s[fmt], int(secs))
    n = int(secs) * fs
    ms, launches = kernel_ms(x)
    flops = 4.0 * N * n / D + 6.0 * n
    byts = b * n + 4.0 * n / D
    t_flop, t_byte = flops / PEAK_FLOPS * 1e3, byts / PEAK_BYTES * 1e3
    res["k_fm_demod"][fmt] = {"seconds": int(secs), "kernel_ms": ms, "launches": launches, "flops": flops, "bytes": byts,
                              "bound_ms": max(t_flop, t_byte), "bound": "fp32" if t_flop >= t_byte else "hbm",
                              "share_of_bound": max(t_flop, t_byte) / ms, "tflops": flops / ms / 1e9}
    if fmt == "cu8":
        na.iq.decode_iq(x[: 2 * fs * 20], s)                   # parks a decoder; the timed call allocates what it needs
        t0 = time.perf_counter()
        rows = na.iq.decode_iq(x, s)
        res["decode_iq_cu8_wall_s"] = {"seconds": int(secs), "wall_s": time.perf_counter() - t0, "rows": rows.size // 2080,
                                       "host_gb": x.nbytes / 1e9}
    del x

# ---- the I/Q stream: seconds of signal per wall second in 0.5 s pushes (cu8, 2.4 Msps, 120 s)
x = np.tile(one_s["cu8"], 120)
k = fs // 2
with na.Stream.for_iq(s, max_push=k) as st:
    t0 = time.perf_counter()
    for t in range(0, x.size // 2, k):
        st.push(x[2 * t: 2 * (t + k)])
    st.finish()
    wall = time.perf_counter() - t0
res["stream_cu8_0.5s_pushes"] = {"seconds": 120, "wall_s": wall, "signal_s_per_wall_s": 120 / wall}

print(json.dumps(res))
out_dir = os.environ.get("OUT") or os.path.join(ROOT, "tool_out")
os.makedirs(out_dir, exist_ok=True)
with open(os.path.join(out_dir, "iq_times.json"), "w") as f:
    json.dump(res, f, indent=1)
