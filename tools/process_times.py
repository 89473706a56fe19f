"""Device times of the process stage (kernels_post.cuh): per kernel for one 48 kHz x 900 s decode (decoder profiling
events) and for a 72 000-row image (image.process under torch.profiler), k_post_stats + k_quantize_i16 of
wav.quantize_i16 on signals of those two lengths, plus the end-to-end apt_decode_image (RGBA) against
apt_decode_image_u8 on the same recording.  Writes $OUT/process_times.json (default tool_out/).
    python tools/process_times.py [reps]"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import noaa_apt_b200 as na
from noaa_apt_b200 import image, synth, wav
from torch.profiler import ProfilerActivity, profile

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 7
res = {}
try:
    res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as e:                                              # noqa: BLE001
    res["gpu"] = f"unknown ({e})"
print(res["gpu"])
pal = np.load(os.path.join(ROOT, "tests", "golden", "palettes.npz"))["noaa-apt-daylight"]
TUNE = (0.4, -0.3, -0.6, 0.8)
MODES = {
    "minmax_grey": dict(contrast=image.MINMAX),
    "percent_grey": dict(contrast=image.PERCENT),
    "histogram_grey_rotate": dict(contrast=image.HISTOGRAM, rotate=True),
    "histogram_rgba": dict(contrast=image.HISTOGRAM, rgba=True),
    "telemetry_palette_rotate_rgba": dict(contrast=image.TELEMETRY, rotate=True, palette=pal, tune=TUNE),
}
med = lambda v: float(np.median(v))                                 # noqa: E731

# ---- 48 kHz x 900 s through the decoder, profiling events on its stream
pcm = synth.apt_pcm16(48000, 900, seed=0)
dec = na.Decoder(48000, na.Settings(), max_samples=pcm.size)
res["decode_48k"] = {}
for name, kw in MODES.items():
    dec.set_process_mode(**kw)
    dec.decode(pcm, True)
    dec.set_profiling(True)
    acc = {}
    for _ in range(reps):
        img = dec.decode(pcm, True)
        for k, ms in dec.kernel_times_ms():
            if k.startswith("post_"):
                acc.setdefault(k, []).append(ms * 1e3)
    dec.set_profiling(False)
    res["decode_48k"][name] = {"rows": int(img.shape[0]), "us": {k: med(v) for k, v in acc.items()}}
    print("48k", name, img.shape[0], {k: round(med(v), 1) for k, v in acc.items()})
# (image mode is process mode with default settings: it launches the minmax_grey kernels above, under the same slot names)
dec.close()

# ---- end to end: apt_decode_image (RGBA, palette, rotation, telemetry) vs apt_decode_image_u8, same recording
e2e = {"decode_image_u8_telemetry": [], "decode_image_rgba_telemetry_palette_rotate": [], "decode_image_grey_histogram": []}
for _ in range(2):
    image.decode_image_u8(None, na.Settings(), pcm, 48000, True, image.TELEMETRY)
    image.decode_image(None, na.Settings(), pcm, 48000, True, **MODES["telemetry_palette_rotate_rgba"])
for _ in range(reps):
    t = time.perf_counter()
    image.decode_image_u8(None, na.Settings(), pcm, 48000, True, image.TELEMETRY)
    e2e["decode_image_u8_telemetry"].append((time.perf_counter() - t) * 1e3)
    t = time.perf_counter()
    image.decode_image(None, na.Settings(), pcm, 48000, True, **MODES["telemetry_palette_rotate_rgba"])
    e2e["decode_image_rgba_telemetry_palette_rotate"].append((time.perf_counter() - t) * 1e3)
    t = time.perf_counter()
    image.decode_image(None, na.Settings(), pcm, 48000, True, **MODES["histogram_grey_rotate"])
    e2e["decode_image_grey_histogram"].append((time.perf_counter() - t) * 1e3)
res["end_to_end_48k_ms"] = {k: {"median": med(v), "min": float(min(v)), "max": float(max(v))} for k, v in e2e.items()}
print("e2e ms", {k: round(med(v), 2) for k, v in e2e.items()})

def kernel_us(call, names, runs=3):
    """median device time (us) per kernel whose name contains one of `names` over `runs` calls, after one warm-up call"""
    call()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(runs):
            call()
    acc = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and any(n in ev.name for n in names):
            short = ev.name.split("(")[0].split("::")[-1].split("<")[0]
            acc.setdefault(short, []).append(ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total)
    return {k: med(v) for k, v in acc.items()}


# ---- 72 000 rows (a 10-hour pass) through apt_process, kernel times from torch.profiler
r = np.random.default_rng(1)
rows = (r.random((72000, 2080), dtype=np.float32) * np.float32(0.8) + np.float32(0.1))
rows[:, :39] = 1.0
rows[:, 1040:1079] = 0.0
res["rows_72000"] = {}
for name, kw in MODES.items():
    if kw["contrast"] == image.TELEMETRY:
        kw = dict(kw, contrast=image.MINMAX)                        # a random image has no telemetry frame
    res["rows_72000"][name] = kernel_us(lambda: image.process(rows, **kw), ("k_post",))
    print("72k", name, {k: round(v, 1) for k, v in res["rows_72000"][name].items()})

# ---- wav.quantize_i16 (the resample tool's 16-bit writer) on signals of 48 kHz x 900 s and of 72 000 rows
res["quantize_i16"] = {}
for name, x in (("48k_900s", np.asarray(pcm, dtype=np.float32)), ("rows_72000", rows.ravel())):
    res["quantize_i16"][name] = kernel_us(lambda: wav.quantize_i16(x), ("k_post_stats", "k_quantize_i16"))
    print("quantize", name, {k: round(v, 1) for k, v in res["quantize_i16"][name].items()})

out_dir = os.environ.get("OUT") or os.path.join(ROOT, "tool_out")
os.makedirs(out_dir, exist_ok=True)
with open(os.path.join(out_dir, "process_times.json"), "w") as f:
    json.dump(res, f, indent=1)
