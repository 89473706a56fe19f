"""Times of the streaming decoder (apt_stream, DESIGN.md §9).  Writes $OUT/stream_times.json (default tool_out/).
    python tools/stream_times.py
  - per-push latency (host clock around push) for 0.1 s, 0.5 s and 5 s pushes at 48 kHz and 11 025 Hz (max_push = 1 s);
  - device time per kernel of the steps of a 48 kHz stream in 1 s pushes (torch.profiler);
  - wall time to stream 48 kHz x 900 s in 1 s pushes, against one apt_decode of the same recording;
  - 64 concurrent streams on one GPU, one per thread, 48 kHz x 120 s each in 1 s pushes."""
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import noaa_apt_b200 as na
from noaa_apt_b200 import synth

res = {}
try:
    res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as e:                                              # noqa: BLE001
    res["gpu"] = f"unknown ({e})"
print(res["gpu"])


def pct(v):
    v = np.asarray(v)
    return {"median": float(np.median(v)), "p90": float(np.percentile(v, 90)), "max": float(v.max()), "n": int(v.size)}


# ---- per-push latency
res["push_latency_ms"] = {}
for rate in (48000, 11025):
    x = synth.apt_pcm16(rate, 120, seed=1).astype(np.float32)
    for secs in (0.1, 0.5, 5.0):
        k = int(rate * secs)
        with na.Stream(rate, max_push=rate) as s:
            lat = []
            for t in range(0, x.size - k + 1, k):
                t0 = time.perf_counter()
                s.push(x[t:t + k])
                lat.append((time.perf_counter() - t0) * 1e3)
            s.finish()
        res["push_latency_ms"][f"{rate}_{secs}s"] = pct(lat[1:])
        print("push", rate, secs, {a: round(b, 3) for a, b in pct(lat[1:]).items()})

# ---- device time per kernel, 48 kHz in 1 s pushes
from torch.profiler import ProfilerActivity, profile
x = synth.apt_pcm16(48000, 60, seed=2).astype(np.float32)
with na.Stream(48000, max_push=48000) as s:
    for t in range(0, 48000 * 5, 48000):
        s.push(x[t:t + 48000])
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        steps = 0
        for t in range(48000 * 5, x.size, 48000):
            s.push(x[t:t + 48000])
            steps += 1
acc = {}
for ev in prof.events():
    if ev.device_type == torch.autograd.DeviceType.CUDA:
        short = ev.name.split("(")[0].split("::")[-1].split("<")[0]
        acc.setdefault(short, []).append(ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total)
res["kernel_us_per_step_48k_1s"] = {k: {"median": float(np.median(v)), "per_step_total": float(np.sum(v)) / steps}
                                    for k, v in acc.items()}
for k, v in res["kernel_us_per_step_48k_1s"].items():
    print("kernel", k, round(v["median"], 2), "us")

# ---- 48 kHz x 900 s: stream in 1 s pushes vs one apt_decode
pcm = synth.apt_pcm16(48000, 900, seed=0)
x = pcm.astype(np.float32)
na.decode(None, na.Settings(), x, 48000, True)
t0 = time.perf_counter()
na.decode(None, na.Settings(), x, 48000, True)
one = time.perf_counter() - t0
with na.Stream(48000, max_push=48000) as s:
    t0 = time.perf_counter()
    for t in range(0, x.size, 48000):
        s.push(x[t:t + 48000])
    s.finish()
    streamed = time.perf_counter() - t0
res["900s_48k_s"] = {"stream_1s_pushes": streamed, "apt_decode": one}
print("900 s:", res["900s_48k_s"])

# ---- 64 concurrent streams, one per thread
N, SECS = 64, 120
xs = [synth.apt_pcm16(48000, SECS, seed=10 + i).astype(np.float32) for i in range(4)]
lat = [[] for _ in range(N)]
barrier = threading.Barrier(N)


def work(i):
    x = xs[i % 4]
    with na.Stream(48000, max_push=48000) as s:
        barrier.wait()
        for t in range(0, x.size, 48000):
            t0 = time.perf_counter()
            s.push(x[t:t + 48000])
            lat[i].append((time.perf_counter() - t0) * 1e3)
        s.finish()


th = [threading.Thread(target=work, args=(i,)) for i in range(N)]
t0 = time.perf_counter()
for t in th:
    t.start()
for t in th:
    t.join()
wall = time.perf_counter() - t0
res["concurrent_64x120s_48k"] = {"wall_s": wall, "audio_s_per_wall_s": N * SECS / wall,
                                 "push_ms": pct([v for lv in lat for v in lv])}
print("64 streams:", res["concurrent_64x120s_48k"])

out_dir = os.environ.get("OUT") or os.path.join(ROOT, "tool_out")
os.makedirs(out_dir, exist_ok=True)
with open(os.path.join(out_dir, "stream_times.json"), "w") as f:
    json.dump(res, f, indent=1)
