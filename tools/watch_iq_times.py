"""Times of the I/Q watcher (DESIGN.md §14).  Prints one JSON line and writes $OUT/watch_iq_times.json (default tool_out/);
the card's name, power limit and maximum SM clock are part of every number.
    python tools/watch_iq_times.py [--rate 2400000] [--seconds 900] [--profile]
  (a) idle push latency, median and p90, for 0.5 s cu8 pushes of receiver noise on the three NOAA channels of a
      137.5 MHz centre (-400, +120 and +412.5 kHz);
  (b) a cu8 feed of --seconds at --rate with a pass on every channel, the first two overlapping, pushed in 0.5 s pieces
      with grey MinMax PNG output: wall time, seconds of feed per second, the latency of each push that fires an LOS, the
      device bytes, and every PNG compared with the recording path on that channel's fm_demod audio;
  (c) with --profile, in a run of its own: the FM kernel time of one 0.5 s step, one launch for the three channels
      against three one-channel launches, from torch.profiler over 50 steps each."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

import noaa_apt_b200 as na
from noaa_apt_b200 import image, synth

ap = argparse.ArgumentParser()
ap.add_argument("--rate", type=int, default=2_400_000)
ap.add_argument("--seconds", type=float, default=900.0)
ap.add_argument("--profile", action="store_true")
args = ap.parse_args()

NOAA = [-400_000, 120_000, 412_500]
res = {}
try:
    res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as e:                                              # noqa: BLE001
    res["gpu"] = f"unknown ({e})"
rate, half = args.rate, args.rate // 2
s = na.iq.IqSettings(rate)

if args.profile:
    import torch
    from torch.profiler import ProfilerActivity, profile
    x = synth.apt_iq_multi(rate, 0.5, carriers=tuple((o, 3 + k, 0.0, None, 60.0) for k, o in enumerate(NOAA)), fmt="cu8")
    singles = [na.iq.IqSettings(rate, offset_hz=o) for o in NOAA]
    for _ in range(3):                                              # warm-up
        na.iq.fm_demod_channels(x, s, NOAA)
        for q in singles:
            na.iq.fm_demod(x, q)

    def kernel_us(fn):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(50):
                fn()
            torch.cuda.synchronize()
        return {ev.key: ev.device_time_total / 50.0 for ev in prof.key_averages() if "fm_demod" in ev.key}

    # apt_fm_demod runs the multi-channel kernel with one channel, so each side is profiled in a session of its own
    one = kernel_us(lambda: na.iq.fm_demod_channels(x, s, NOAA))
    three = kernel_us(lambda: [na.iq.fm_demod(x, q) for q in singles])
    res["fm_kernel_us_per_half_second_step"] = {"one_launch_three_channels": sum(one.values()),
                                                 "three_launches_one_channel_each": sum(three.values()),
                                                 "kernels": [list(one), list(three)]}
else:
    # (a) idle pushes
    rng = np.random.default_rng(1)
    noise = np.clip(np.rint(rng.normal(127.5, 3.0, 2 * 40 * rate)), 0, 255).astype(np.uint8)
    with na.IqWatch(s, NOAA, image_out="png", max_push=half) as w:
        w.push(noise[: 2 * half])                                   # warm-up
        lat = []
        for a in range(half, noise.size // 2 - half + 1, half):
            t0 = time.perf_counter()
            w.push(noise[2 * a:2 * (a + half)])
            lat.append(time.perf_counter() - t0)
    res["idle_push_half_s"] = {"median_ms": 1e3 * float(np.median(lat)), "p90_ms": 1e3 * float(np.percentile(lat, 90))}

    # (b) the pass feed
    T = args.seconds
    passes = [(NOAA[0], 11, 0.05 * T, 0.45 * T), (NOAA[1], 12, 0.30 * T, 0.70 * T), (NOAA[2], 13, 0.75 * T, 0.97 * T)]
    t0 = time.perf_counter()
    x = synth.apt_iq_passes(rate, T, passes, fmt="cu8", fade_s=min(10.0, 0.02 * T), chunk=1 << 23)
    res["generate_s"] = time.perf_counter() - t0
    search = dict(min_length_s=min(60.0, 0.1 * T), max_gap_s=min(30.0, 0.03 * T))
    n = x.size // 2
    with na.IqWatch(s, NOAA, image_out="png", contrast=image.MINMAX, max_push=half, max_rows=4000,
                    search=search) as w:
        bytes0 = w.device_bytes
        los, los_ms = [], []
        t0 = time.perf_counter()
        for a in range(0, n, half):
            t1 = time.perf_counter()
            _q, evs = w.push(x[2 * a:2 * min(n, a + half)])
            dt = time.perf_counter() - t1
            got = [(c, e) for c, e in evs if e.kind == "los"]
            if got:
                los += got
                los_ms.append(1e3 * dt)
        _q, evs = w.finish()
        los += [(c, e) for c, e in evs if e.kind == "los"]
        wall = time.perf_counter() - t0
        assert w.device_bytes == bytes0
    same, found_all = [], 0
    for c, off in enumerate(NOAA):
        a_c = na.iq.fm_demod(x, na.iq.IqSettings(rate, offset_hz=off))
        with na.Recording(a_c, s.audio_rate) as rec:
            found = rec.find_passes(**search)
            want, _inf, _sts = rec.decode_png(found, contrast=image.MINMAX)
        mine = [e for ch, e in los if ch == c]
        found_all += len(found)
        same.append([e.pass_ for e in mine] == found and all(e.data == d for e, d in zip(mine, want)))
    res["feed"] = {"rate": rate, "seconds": T, "wall_s": wall, "feed_s_per_wall_s": T / wall, "los_push_ms": los_ms,
                   "device_bytes": bytes0, "passes": len(los), "passes_offline": found_all,
                   "pngs_equal_recording_path": all(same)}

line = json.dumps(res, default=str)
print(line)
out = os.environ.get("OUT", os.path.join(ROOT, "tool_out"))
os.makedirs(out, exist_ok=True)
with open(os.path.join(out, "watch_iq_times_profile.json" if args.profile else "watch_iq_times.json"), "w") as f:
    f.write(line + "\n")
