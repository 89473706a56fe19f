"""Times of the carrier search (DESIGN.md §10, "Finding carriers").  Prints one JSON line and writes
$OUT/iq_search_times.json (default tool_out/).
    python tools/iq_search_times.py [--seconds 900] [--block 4] [--repeats 5]
On a 2.4 Msps cu8 pass holding three APT carriers (a --block seconds synthetic recording of apt_iq_multi, tiled):
  - the spectrum kernels' device time (torch.profiler) for nfft 16384 and 2048 segments, with its share of the data-sheet
    bound (flops 5 N log2 N per segment, bytes of the segments read);
  - apt_iq_find_carriers wall time from pageable host memory;
  - apt_decode_iq_auto wall time against three apt_decode_iq calls at the offsets it found."""
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
ap.add_argument("--seconds", type=int, default=900)
ap.add_argument("--block", type=float, default=4.0)
ap.add_argument("--repeats", type=int, default=5)
args = ap.parse_args()

res = {}
try:
    res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as e:                                              # noqa: BLE001
    res["gpu"] = f"unknown ({e})"

fs = 2_400_000
carriers = [(37_000, 1, 0.0, None, 20.0), (-300_000, 2, 0.0, None, 20.0), (412_500, 3, 0.0, None, 20.0)]
block = synth.apt_iq_multi(fs, args.block, carriers=carriers, fmt="cu8", noise_rel=0.03)
x = np.tile(block, int(np.ceil(args.seconds / args.block)))[: 2 * fs * args.seconds]
n = x.size // 2
res["pass"] = {"seconds": args.seconds, "iq_rate": fs, "format": "cu8", "host_gb": x.nbytes / 1e9,
               "carriers_hz": [c[0] for c in carriers]}


def median_wall(fn, k):
    ts = []
    for _ in range(k):
        t0 = time.perf_counter()
        out = fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), out


# ---- the spectrum kernels
nfft, K = 16384, 2048
na.iq.spectrum(x, fs, nfft=nfft, max_segments=K)                     # warm-up: workspace, stager, attributes
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    na.iq.spectrum(x, fs, nfft=nfft, max_segments=K)
ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "k_spectrum" in e.name]
us = {name: float(np.sum([(e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total)
                          for e in ev if name in e.name and ("finish" in e.name) == ("finish" in name)]))
      for name in ("k_spectrum<", "k_spectrum_finish")}
ms = (us["k_spectrum<"] + us["k_spectrum_finish"]) / 1e3
flops = 5.0 * nfft * np.log2(nfft) * K
byts = 2.0 * nfft * K + 2 * 4.0 * 256 * nfft + 4.0 * 256 * nfft      # segments; the slots' sums read and written, then read
t_flop, t_byte = flops / PEAK_FLOPS * 1e3, byts / PEAK_BYTES * 1e3
res["spectrum_kernels"] = {"nfft": nfft, "segments": K, "k_spectrum_ms": us["k_spectrum<"] / 1e3,
                           "k_spectrum_finish_ms": us["k_spectrum_finish"] / 1e3, "total_ms": ms,
                           "launches": len(ev), "flops": flops, "bytes": byts, "bound_ms": max(t_flop, t_byte),
                           "bound": "fp32" if t_flop >= t_byte else "hbm", "share_of_bound": max(t_flop, t_byte) / ms}
wall, _ = median_wall(lambda: na.iq.spectrum(x, fs, nfft=nfft, max_segments=K), args.repeats)
res["spectrum_wall_s"] = wall

# ---- find_carriers from pageable memory
wall, found = median_wall(lambda: na.iq.find_carriers(x, fs), args.repeats)
res["find_carriers"] = {"wall_s": wall, "found": [(c.offset_hz, round(c.snr_db, 2), round(c.apt_score, 3), c.is_apt)
                                                  for c in found]}

# ---- decode_iq_auto against three decode_iq calls, alternated
s = na.iq.IqSettings(fs)
na.iq.decode_iq_auto(x[: 2 * fs * 20], fs)                          # parks decoders
offsets = [c.offset_hz for c in found if c.is_apt]
t_auto, t_three = [], []
for _ in range(3):
    t0 = time.perf_counter()
    cars, rows = na.iq.decode_iq_auto(x, fs)
    t_auto.append(time.perf_counter() - t0)
    t0 = time.perf_counter()
    singles = [na.iq.decode_iq(x, na.iq.IqSettings(fs, offset_hz=o)) for o in offsets]
    t_three.append(time.perf_counter() - t0)
res["decode_iq_auto"] = {"wall_s": float(np.median(t_auto)), "channels": len(cars),
                         "rows": [int(r.size // 2080) if r is not None else None for r in rows]}
res["three_decode_iq"] = {"wall_s": float(np.median(t_three)), "rows": [int(r.size // 2080) for r in singles]}
res["equal_rows"] = all(r is not None and np.array_equal(r, sgl) for r, sgl in
                        zip(rows, [singles[offsets.index(c.offset_hz)] for c in cars]))

print(json.dumps(res))
out_dir = os.environ.get("OUT") or os.path.join(ROOT, "tool_out")
os.makedirs(out_dir, exist_ok=True)
with open(os.path.join(out_dir, "iq_search_times.json"), "w") as f:
    json.dump(res, f, indent=1)
