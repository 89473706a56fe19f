"""Times of the pass search (DESIGN.md §12) on a long recording.  Prints one JSON line and writes $OUT/pass_times.json
(default tool_out/).
    python tools/pass_times.py [--rate 96000] [--hours 10] [--passes 8]
On a PCM16 recording of --hours at --rate holding --passes synthetic passes of 12 to 15 minutes between stretches of
receiver noise and silence (synth.apt_passes, generated chunk by chunk):
  - apt_recording_create (the one upload, from pageable memory);
  - apt_recording_quality wall time, and the device time of k_pass_quality and of the first stage (torch.profiler, a run
    of its own) with k_pass_quality's bytes (two rows of 4-byte samples read per window) over time against 3.35 TB/s;
  - the pass rule (apt_find_passes_quality) on the host;
  - apt_recording_decode of every found pass to PNG, against one apt_decode_png per host slice and one apt_decode_png of
    the whole recording; the PNG bytes of the two per-pass paths are compared."""
import argparse
import concurrent.futures as cf
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
from noaa_apt_b200 import image, synth

PEAK_BYTES = 3.35e12   # H100 SXM5 data sheet, HBM3

ap = argparse.ArgumentParser()
ap.add_argument("--rate", type=int, default=96000)
ap.add_argument("--hours", type=float, default=10.0)
ap.add_argument("--passes", type=int, default=8)
args = ap.parse_args()

res = {}
try:
    res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as e:                                              # noqa: BLE001
    res["gpu"] = f"unknown ({e})"

rate, total_s = args.rate, args.hours * 3600.0
lengths = [720.0 + 180.0 * k / max(args.passes - 1, 1) for k in range(args.passes)]     # 12 .. 15 min
gap = (total_s - sum(lengths)) / (args.passes + 1)
layout = []
for k, length in enumerate(lengths):
    layout.append(("noise" if k % 2 == 0 else "silence", gap))
    layout.append(("pass", length, 11 + k))
layout.append(("noise", gap))
n = synth.apt_passes_len(rate, layout)
t0 = time.perf_counter()
pcm = np.empty(n, dtype=np.int16)
step = 1 << 24


def fill(a):
    pcm[a:min(n, a + step)] = synth.apt_passes(rate, layout, seed=1, start=a, n_samples=min(n, a + step) - a)


with cf.ThreadPoolExecutor(max(os.cpu_count() or 1, 1)) as ex:
    list(ex.map(fill, range(0, n, step)))
res["recording"] = {"rate": rate, "hours": args.hours, "samples": n, "format": "pcm16", "host_gb": pcm.nbytes / 1e9,
                    "passes_min": [round(x / 60, 2) for x in lengths], "generate_s": time.perf_counter() - t0}
truth = synth.apt_passes_truth(rate, layout)


def wall(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


torch.cuda.init()
t_create, rec = wall(lambda: na.Recording(pcm, rate))
info = rec.info()
res["create_s"] = t_create
res["upload_gb_per_s"] = pcm.nbytes / t_create / 1e9
res["device_bytes"] = info["device_bytes"]
rec.quality()                                                           # warm: module load
t_q = [wall(rec.quality)[0] for _ in range(3)]
q = rec.quality()
res["quality_s"] = float(np.median(t_q))
res["windows"] = int(q.size)

with profile(activities=[ProfilerActivity.CUDA]) as prof:
    rec.quality()
    torch.cuda.synchronize()
kern = {}
for ev in prof.events():
    if ev.device_type.name == "CUDA":
        key = "k_pass_quality" if "k_pass_quality" in ev.name else ("pcm16_to_f32" if "pcm16" in ev.name else "first_stage")
        kern[key] = kern.get(key, 0.0) + ev.device_time_total / 1e3   # ms
res["kernel_ms"] = kern
row = info["row_samples"]
qbytes = q.size * (2 * row * 4 + 4)
if kern.get("k_pass_quality"):
    res["k_pass_quality_gb_per_s"] = qbytes / (kern["k_pass_quality"] / 1e3) / 1e9
    res["k_pass_quality_share_of_hbm"] = res["k_pass_quality_gb_per_s"] * 1e9 / PEAK_BYTES

t_find, found = wall(lambda: na.find_passes_quality(q, n, rate))
res["find_passes_s"] = t_find
res["passes"] = [[p.start, p.end, round(p.mean_quality, 3), round(p.peak_quality, 3)] for p in found]
res["boundary_error_s"] = [max(abs(p.start - a), abs(p.end - b)) / rate for p, (a, b) in zip(found, truth)] \
    if len(found) == len(truth) else None

rec.decode_png(found[:1], contrast=image.MINMAX)                       # warm
t_dec, (pngs, _infos, sts) = wall(lambda: rec.decode_png(found, contrast=image.MINMAX))
res["decode_png_all_passes_s"] = t_dec
res["statuses"] = sts
rec.close()

t_host = 0.0
same = True
for p, got in zip(found, pngs):
    dt, (want, _) = wall(lambda: image.decode_png(None, None, pcm[p.start:p.end], rate, contrast=image.MINMAX))
    t_host += dt
    same = same and want == got
res["host_slices_decode_png_s"] = t_host
res["png_bytes_equal"] = same
t_whole, _ = wall(lambda: image.decode_png(None, None, pcm, rate, contrast=image.MINMAX))
res["whole_recording_decode_png_s"] = t_whole

line = json.dumps(res)
print(line)
out = os.environ.get("OUT", os.path.join(ROOT, "tool_out"))
os.makedirs(out, exist_ok=True)
with open(os.path.join(out, "pass_times.json"), "w") as f:
    f.write(line + "\n")
