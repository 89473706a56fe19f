"""Device times of the PNG encoder (kernels_png.cuh): per kernel under torch.profiler for grey and RGBA images of 1 800
and 72 000 rows (the reference's example image tiled), and end to end apt_decode_png against apt_decode_image + Pillow
(zlib level 6) on one 48 kHz x 900 s recording.  Writes $OUT/png_times.json (default tool_out/).
    python tools/png_times.py [reps]"""
import io
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from PIL import Image
from torch.profiler import ProfilerActivity, profile

import noaa_apt_b200 as na
from noaa_apt_b200 import image, synth

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
res = {}
try:
    res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as e:                                              # noqa: BLE001
    res["gpu"] = f"unknown ({e})"
print(res["gpu"])
med = lambda v: float(np.median(v))                                 # noqa: E731
grey0 = np.load(os.path.join(ROOT, "tests", "golden", "argentina_excerpt.npz"))["grey"]


def tiled(rows):
    g = np.tile(grey0, (-(-rows // grey0.shape[0]), 1))[:rows].copy()
    g[::97] ^= 0x5A
    return g


def rgba_of(g):
    out = np.empty(g.shape + (4,), dtype=np.uint8)
    out[..., :3] = g[..., None]
    out[..., 3] = 255
    return out


res["kernels_us"] = {}
for rows in (1800, 72000):
    g = tiled(rows)
    for name, img in (("grey", g), ("rgba", rgba_of(g))):
        png = image.encode_png(img)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                image.encode_png(img)
        acc = {}
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA and ("k_png" in ev.name or "Memset" in ev.name):
                short = ev.name.split("(")[0].split("::")[-1].split("<")[0]
                acc.setdefault(short, []).append(ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total)
        per = {k: sum(v) / reps for k, v in acc.items()}
        key = f"{name}_{rows}"
        res["kernels_us"][key] = {"bytes_raw": int(img.size), "bytes_png": len(png), "us": per, "total_us": sum(per.values())}
        print(key, len(png), round(sum(per.values()), 1), {k: round(v, 1) for k, v in per.items()})

# ---- end to end on one recording: decode + process + PNG on the device vs decode + process + Pillow on the CPU
pcm = synth.apt_pcm16(48000, 900, seed=0)
pal = np.load(os.path.join(ROOT, "tests", "golden", "palettes.npz"))["noaa-apt-daylight"]
MODES = {"grey_minmax": dict(contrast=image.MINMAX),
         "rgba_palette_rotate": dict(contrast=image.MINMAX, rotate=True, palette=pal, tune=(0.4, -0.3, -0.6, 0.8))}
res["end_to_end_48k_ms"] = {}
for name, kw in MODES.items():
    for _ in range(2):
        image.decode_png(None, na.Settings(), pcm, 48000, True, **kw)
    a, b, c = [], [], []
    for _ in range(reps):
        t = time.perf_counter()
        png, _ = image.decode_png(None, na.Settings(), pcm, 48000, True, **kw)
        a.append((time.perf_counter() - t) * 1e3)
        t = time.perf_counter()
        img, _ = image.decode_image(None, na.Settings(), pcm, 48000, True, **kw)
        b.append((time.perf_counter() - t) * 1e3)
        buf = io.BytesIO()
        Image.fromarray(img).save(buf, format="PNG")
        c.append((time.perf_counter() - t) * 1e3)
    res["end_to_end_48k_ms"][name] = {"decode_png": med(a), "decode_image": med(b), "decode_image_plus_pillow": med(c),
                                      "png_bytes": len(png), "pillow_bytes": len(buf.getvalue()), "rows": int(img.shape[0])}
    print("e2e", name, res["end_to_end_48k_ms"][name])

out_dir = os.environ.get("OUT") or os.path.join(ROOT, "tool_out")
os.makedirs(out_dir, exist_ok=True)
with open(os.path.join(out_dir, "png_times.json"), "w") as f:
    json.dump(res, f, indent=1)
