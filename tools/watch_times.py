"""Times of the watcher (DESIGN.md §13).  Prints one JSON line and writes $OUT/watch_times.json (default tool_out/); the
card's name, power limit and maximum SM clock are part of every number.
    python tools/watch_times.py [--rate 96000] [--hours 10] [--passes 8] [--watchers 64]
  (a) idle push latency, median and p90, for 1 s pushes of receiver noise at 48 and 96 kHz;
  (b) a PCM16 feed of --hours at --rate holding --passes synthetic passes (the layout of tools/pass_times.py), in 1 s
      pushes, once with grey MinMax PNG output and once with RGBA telemetry + false colour + rotation pixels: total wall
      time, the latency of each push that fires an LOS, the watcher's device bytes, and each pass's bytes compared with
      the recording path's (apt_recording_decode of the same range);
  (c) --watchers watchers on one device, one thread each, fed 1 s pushes of the first --watch-seconds of the feed:
      seconds of audio per second of wall time, all watchers together."""
import argparse
import concurrent.futures as cf
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

import noaa_apt_b200 as na
from noaa_apt_b200 import image, synth

ap = argparse.ArgumentParser()
ap.add_argument("--rate", type=int, default=96000)
ap.add_argument("--hours", type=float, default=10.0)
ap.add_argument("--passes", type=int, default=8)
ap.add_argument("--watchers", type=int, default=64)
ap.add_argument("--watch-seconds", type=float, default=1800.0)
args = ap.parse_args()

res = {}
try:
    res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as e:                                              # noqa: BLE001
    res["gpu"] = f"unknown ({e})"

# (a) idle pushes
idle = {}
for rate in (48000, 96000):
    noise = (np.random.default_rng(1).normal(0, 2000, 60 * rate)).astype(np.int16)
    with na.Watch(rate) as w:
        w.push(noise[:rate])                                        # warm-up
        lat = []
        for k in range(1, 60):
            t0 = time.perf_counter()
            w.push(noise[k * rate:(k + 1) * rate])
            lat.append(time.perf_counter() - t0)
    idle[str(rate)] = {"median_ms": 1e3 * float(np.median(lat)), "p90_ms": 1e3 * float(np.percentile(lat, 90))}
res["idle_push_1s"] = idle

# (b) the long feed
rate, total_s = args.rate, args.hours * 3600.0
lengths = [720.0 + 180.0 * k / max(args.passes - 1, 1) for k in range(args.passes)]     # 12 .. 15 min
gap = (total_s - sum(lengths)) / (args.passes + 1)
layout = []
for k, length in enumerate(lengths):
    layout.append(("noise" if k % 2 == 0 else "silence", gap))
    layout.append(("pass", length, 11 + k))
layout.append(("noise", gap))
n = synth.apt_passes_len(rate, layout)
pcm = np.empty(n, dtype=np.int16)
step = 1 << 24
with cf.ThreadPoolExecutor(16) as ex:
    list(ex.map(lambda a: pcm.__setitem__(slice(a, min(n, a + step)),
                                         synth.apt_passes(rate, layout, seed=1, start=a, n_samples=min(n, a + step) - a)),
                range(0, n, step)))
pal = np.random.default_rng(3).integers(0, 256, (256, 256, 3), dtype=np.uint8)
outputs = {"grey_png": dict(image_out="png", contrast=image.MINMAX),
           "rgba_telemetry_false_colour_rotated": dict(image_out="image", contrast=image.TELEMETRY, palette=pal, rotate=True,
                                                       rgba=True)}
feed = {}
with na.Recording(pcm, rate) as rec:
    found = rec.find_passes()
    for name, kw in outputs.items():
        with na.Watch(rate, max_rows=2000, **kw) as w:
            bytes0 = w.device_bytes
            los, los_ms = [], []
            t0 = time.perf_counter()
            for a in range(0, n, rate):
                t1 = time.perf_counter()
                _q, evs = w.push(pcm[a:a + rate])
                dt = time.perf_counter() - t1
                got = [e for e in evs if e.kind == "los"]
                if got:
                    los += got
                    los_ms.append(1e3 * dt)
            _q, evs = w.finish()
            los += [e for e in evs if e.kind == "los"]
            wall = time.perf_counter() - t0
            assert w.device_bytes == bytes0
        if kw["image_out"] == "png":
            want, _inf, _sts = rec.decode_png(found, contrast=image.MINMAX)
            same = [e.data == d for e, d in zip(los, want)]
        else:
            want, _inf, _sts = rec.decode_image(found, contrast=image.TELEMETRY, palette=pal, rotate=True, rgba=True)
            same = [e.data is not None and d is not None and np.array_equal(e.data, d) for e, d in zip(los, want)]
        feed[name] = {"wall_s": wall, "audio_s_per_wall_s": n / rate / wall, "los_push_ms": los_ms,
                      "device_bytes": bytes0, "passes": len(los), "passes_offline": len(found),
                      "same_passes": [e.pass_ for e in los] == found, "same_bytes": all(same) and len(same) == len(found)}
res["feed"] = {"rate": rate, "hours": args.hours, **feed}

# (c) many watchers on one device
m = min(n, int(args.watch_seconds * rate))
start = threading.Barrier(args.watchers)


def watch_one(_):
    with na.Watch(rate, image_out="png") as w:
        start.wait()
        for a in range(0, m, rate):
            w.push(pcm[a:min(m, a + rate)])
        w.finish()


t0 = time.perf_counter()
with cf.ThreadPoolExecutor(args.watchers) as ex:
    list(ex.map(watch_one, range(args.watchers)))
wall = time.perf_counter() - t0
res["many_watchers"] = {"watchers": args.watchers, "seconds_each": m / rate, "wall_s": wall,
                        "audio_s_per_wall_s": args.watchers * m / rate / wall}

line = json.dumps(res, default=str)
print(line)
out = os.environ.get("OUT", os.path.join(ROOT, "tool_out"))
os.makedirs(out, exist_ok=True)
with open(os.path.join(out, "watch_times.json"), "w") as f:
    f.write(line + "\n")
