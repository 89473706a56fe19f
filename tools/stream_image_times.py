"""Loss-of-signal latency of the streaming decoder's image output (DESIGN.md §9).  Writes $OUT/stream_image_times.json
(default tool_out/).
    python tools/stream_image_times.py [repeats]
48 kHz x 900 s streamed in 1 s pushes; host clock around the synchronous last call, median of `repeats` (default 7) passes
after one warm-up pass, for grey MinMax and RGBA Telemetry + false colour + rotation:
  (a) finish()
  (b) finish_image() as pixels
  (c) finish_image() as PNG
  (d) finish() + image.process(all rows) + image.encode_png (the route without image output: the rows are on the host)
and the push latency (median / p90 over every 1 s push of the timed passes) with image output off and on."""
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

REPEATS = int(sys.argv[1]) if len(sys.argv) > 1 else 7
RATE = 48000

res = {}
try:
    res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as e:                                              # noqa: BLE001
    res["gpu"] = f"unknown ({e})"
print(res["gpu"], flush=True)
if na.device_count() < 1:
    raise SystemExit("stream_image_times.py measures on the GPU; no CUDA device found")

x = synth.apt_pcm16(RATE, 900, seed=0).astype(np.float32)
palette = np.load(os.path.join(ROOT, "tests", "golden", "palettes.npz"))["noaa-apt-daylight"]
SETTINGS = {"grey_minmax": dict(contrast=image.MINMAX),
            "rgba_telemetry_palette_rotate": dict(contrast=image.TELEMETRY, rotate=True, palette=palette, rgba=True)}


def pct(v):
    v = np.asarray(v)
    return {"median": float(np.median(v)), "p90": float(np.percentile(v, 90)), "n": int(v.size)}


def one_pass(strm, end, push_ms):
    """Pushes the recording in 1 s pushes, then times `end(strm, rows)` (rows: those the pushes returned)."""
    strm.reset()
    rows = []
    for t in range(0, x.size, RATE):
        t0 = time.perf_counter()
        rows.append(strm.push(x[t:t + RATE]))
        push_ms.append((time.perf_counter() - t0) * 1e3)
    t0 = time.perf_counter()
    out = end(strm, rows)
    return (time.perf_counter() - t0) * 1e3, out


def finish_then_host_route(kw):
    def end(strm, rows):
        rows.append(strm.finish())
        img, _ = image.process(np.concatenate([r.ravel() for r in rows]), **kw)
        return image.encode_png(img)
    return end


def measure(strm, end, push_ms):
    one_pass(strm, end, [])                                          # warm-up
    times, out = [], None
    for _ in range(REPEATS):
        ms, out = one_pass(strm, end, push_ms)
        times.append(ms)
    return pct(times), out


res["los_latency_ms"], res["push_latency_ms"], res["device_bytes"] = {}, {}, {}
with na.Stream(RATE, na.Settings(), max_push=RATE) as strm:
    res["device_bytes"]["stream"] = strm.info()["device_bytes"]
    for name, kw in SETTINGS.items():
        r = res["los_latency_ms"][name] = {}
        strm.reset()
        strm.set_process_mode(None)
        push_off = []
        r["a_finish"], _ = measure(strm, lambda s, rows: s.finish(), push_off)
        r["d_finish_process_encode_png"], png_d = measure(strm, finish_then_host_route(kw), [])
        strm.reset()
        strm.set_process_mode(max_rows=2400, **kw)
        res["device_bytes"][name + "_pixels"] = strm.info()["device_bytes"]
        push_on = []
        r["b_finish_image_pixels"], _ = measure(strm, lambda s, rows: s.finish_image(), push_on)
        strm.reset()
        strm.set_png_mode()
        res["device_bytes"][name + "_png"] = strm.info()["device_bytes"]
        r["c_finish_image_png"], (_, png_c, _) = measure(strm, lambda s, rows: s.finish_image(), [])
        assert png_c == png_d, name                                 # the same file either way
        res["push_latency_ms"][name] = {"image_output_off": pct(push_off), "image_output_on": pct(push_on)}
        print(name, {k: round(v["median"], 2) for k, v in r.items()}, "ms;",
              "push off/on median", round(pct(push_off)["median"], 3), round(pct(push_on)["median"], 3),
              "p90", round(pct(push_off)["p90"], 3), round(pct(push_on)["p90"], 3), flush=True)
print("device bytes", res["device_bytes"])

out_dir = os.environ.get("OUT") or os.path.join(ROOT, "tool_out")
os.makedirs(out_dir, exist_ok=True)
with open(os.path.join(out_dir, "stream_image_times.json"), "w") as f:
    json.dump(res, f, indent=1)
