"""Times of batch PNG output (apt_decode_batch_image) and of the batched PNG encoder.  Writes $OUT/batch_png_times.json
(default tool_out/).
    python tools/batch_png_times.py [--reps N] [--parent TREE] [--seconds S] [--count B] [--sections 123]

1. The bench's workload ending in PNG: 64 recordings of 48 kHz x 900 s on one GPU (4 distinct recordings, each passed
   16 times, pageable f32), grey MinMax and RGBA false colour + rotation.  apt_decode_batch_image against
   (a) apt_decode_png per recording, (b) apt_decode_batch rows then apt_process + apt_png_encode per recording,
   (c) 4 decoders in PNG mode driven round-robin; and pixel mode against apt_decode_batch rows.
2. Kernel level: torch.profiler time per kernel of one batched encode (apt_png_encode_batch) of G = 1, 4, 16, 64 grey
   and RGBA images of 1 800 rows, against G single encodes.
3. One image: tools/png_times.py of this tree and of another built tree (--parent, e.g. the parent commit's), alternated,
   in this call."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--parent", default=None, help="another built tree whose tools/png_times.py runs against this one")
ap.add_argument("--seconds", type=int, default=900)
ap.add_argument("--count", type=int, default=64)
ap.add_argument("--sections", default="123")
ap.add_argument("--runs", type=int, default=3, help="alternated runs of each tree in section 3")
args_ = ap.parse_args()
reps = args_.reps
out_dir = os.path.abspath(os.environ.get("OUT") or os.path.join(ROOT, "tool_out"))
os.makedirs(out_dir, exist_ok=True)


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                          # noqa: BLE001
        return f"unknown ({e})"


def stats(v):
    v = np.asarray(v, dtype=np.float64)
    return {"median": float(np.median(v)), "min": float(v.min()), "max": float(v.max()), "n": int(v.size)}


def png_times_run(tree, tag):
    env = dict(os.environ, OUT=os.path.join(out_dir, f"png_times_{tag}"))
    subprocess.run([sys.executable, os.path.join(tree, "tools", "png_times.py"), str(reps)], env=env, capture_output=True,
                   text=True, timeout=1800, cwd=tree)
    with open(os.path.join(env["OUT"], "png_times.json")) as f:
        return json.load(f)


res = {"gpu": gpu_name()}
print(res["gpu"], flush=True)

# ---- 3 first (subprocesses, before this process holds device memory): one image, this build against the parent
if "3" in args_.sections and args_.parent:
    runs = {"new": [], "parent": []}
    for _ in range(args_.runs):
        runs["parent"].append(png_times_run(os.path.abspath(args_.parent), "parent"))
        runs["new"].append(png_times_run(ROOT, "new"))
    one = {}
    for tag, rs in runs.items():
        for key in rs[0]["kernels_us"]:
            one.setdefault(key, {})[tag] = [r["kernels_us"][key]["total_us"] for r in rs]
        for key in rs[0]["end_to_end_48k_ms"]:
            one.setdefault("decode_png_" + key, {})[tag] = [r["end_to_end_48k_ms"][key]["decode_png"] for r in rs]
    res["single_image"] = one
    print("single image", json.dumps(one), flush=True)

import torch                                                        # noqa: E402
from torch.profiler import ProfilerActivity, profile                # noqa: E402

import noaa_apt_b200 as na                                          # noqa: E402
from noaa_apt_b200 import _lib, image, synth                        # noqa: E402

lib = _lib.load()
pal = np.load(os.path.join(ROOT, "tests", "golden", "palettes.npz"))["noaa-apt-daylight"]
MODES = {"grey_minmax": dict(contrast=image.MINMAX),
         "rgba_palette_rotate": dict(contrast=image.MINMAX, rotate=True, palette=pal, rgba=True)}

# ---- 2. kernel level
grey0 = np.load(os.path.join(ROOT, "tests", "golden", "argentina_excerpt.npz"))["grey"]


def tiled(rows, k):
    g = np.tile(grey0, (-(-rows // grey0.shape[0]), 1))[:rows].copy()
    g[k::97] ^= 0x5A
    return g


def rgba_of(g):
    out = np.empty(g.shape + (4,), dtype=np.uint8)
    out[..., :3] = g[..., None]
    out[..., 3] = 255
    return out


def encode_batch(imgs, ps):
    n = len(imgs)
    h, w = imgs[0].shape[:2]
    ch = 1 if imgs[0].ndim == 2 else imgs[0].shape[2]
    bound = image.png_bound(w, h, ch)
    outs = [np.empty(bound, np.uint8) for _ in imgs]
    rc = lib.apt_png_encode_batch((C.c_void_p * n)(*[x.ctypes.data for x in imgs]), (C.c_uint32 * n)(*([h] * n)), n, w, ch,
                                  C.byref(ps), (C.c_void_p * n)(*[o.ctypes.data for o in outs]),
                                  (C.c_uint64 * n)(*([bound] * n)), (C.c_uint64 * n)())
    assert rc == 0, rc


def kernel_us(fn):
    fn()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
    acc = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and "k_png" in ev.name:
            short = ev.name.split("(")[0].split("::")[-1].split("<")[0]
            acc[short] = acc.get(short, 0.0) + (ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total)
    return {k: v / reps for k, v in acc.items()}


ps = image.png_settings()
res["kernels_us"] = {}
for kind in ("grey", "rgba") if "2" in args_.sections else ():
    base = [tiled(1800, k) for k in range(64)]
    imgs = base if kind == "grey" else [rgba_of(g) for g in base]
    for G in (1, 4, 16, 64):
        batched = kernel_us(lambda: encode_batch(imgs[:G], ps))
        single = kernel_us(lambda: [image.encode_png(x) for x in imgs[:G]])
        res["kernels_us"][f"{kind}_G{G}"] = {"batched": batched, "batched_total": sum(batched.values()),
                                             "singles": single, "singles_total": sum(single.values())}
        print(kind, G, round(sum(batched.values()), 1), round(sum(single.values()), 1), flush=True)
    del imgs, base

# ---- 1. the bench's workload ending in PNG
rate, B = 48000, args_.count
distinct = [synth.apt_pcm16(rate, args_.seconds, seed=k).astype(np.float32) for k in range(4)]
sigs = [distinct[i % 4] for i in range(B)]
s = na.Settings().to_c()
bound_rows = na.decode_len_bound(sigs[0].size, rate) // 2080


def batch_image(kw, png):
    ps_c, bpp, pal_keep = image.process_settings(**kw)
    cap = image.png_bound(2080, bound_rows, bpp) if png else bound_rows * 2080 * bpp
    outs = [np.empty(cap, np.uint8) for _ in range(B)]
    pngs = image.png_settings()
    args = ((C.c_void_p * B)(*[x.ctypes.data for x in sigs]), _lib.F32, (C.c_uint64 * B)(*[x.size for x in sigs]), B, rate,
            C.byref(s), 1, C.byref(ps_c), C.byref(pngs) if png else None, (C.c_void_p * B)(*[o.ctypes.data for o in outs]),
            (C.c_uint64 * B)(*([cap] * B)), (C.c_uint64 * B)(), (_lib.CImageInfo * B)(), (C.c_int * B)(), (C.c_int * 1)(0), 1, 4)

    keep = (outs, pal_keep, ps_c, pngs)   # the library writes into outs and reads the palette: alive while run is

    def run():
        assert lib.apt_decode_batch_image(*args) == 0, len(keep)
    return run


def batch_rows():
    cap = bound_rows * 2080
    outs = [np.empty(cap, np.float32) for _ in range(B)]
    args = ((C.c_void_p * B)(*[x.ctypes.data for x in sigs]), _lib.F32, (C.c_uint64 * B)(*[x.size for x in sigs]), B, rate,
            C.byref(s), 1, (C.c_void_p * B)(*[o.ctypes.data for o in outs]), (C.c_uint64 * B)(*([cap] * B)),
            (C.c_uint64 * B)(), (C.c_int * B)(), (C.c_int * 1)(0), 1, 4)

    def run():
        assert lib.apt_decode_batch(*args) == 0
        return outs, args[9]
    return run


def seq_decode_png(kw):
    def run():
        for x in sigs:
            image.decode_png(None, na.Settings(), x, rate, True, **kw)
    return run


def rows_then_encode(kw):
    rows = batch_rows()

    def run():
        outs, nouts = rows()
        for i in range(B):
            img, _ = image.process(outs[i][: nouts[i]], **kw)
            image.encode_png(img)
    return run


def png_mode_round_robin(kw, ndec=4):
    ps_c, bpp, _p = image.process_settings(**kw)
    pngs = image.png_settings()
    cap = image.png_bound(2080, bound_rows, bpp)
    decs = []
    for _ in range(ndec):
        d = C.c_void_p()
        assert lib.apt_decoder_create(0, rate, C.byref(s), sigs[0].size, C.byref(d)) == 0
        assert lib.apt_decoder_set_process_mode(d, C.byref(ps_c)) == 0
        assert lib.apt_decoder_set_png_mode(d, C.byref(pngs)) == 0
        decs.append(d)
    outs = [np.empty(cap, np.uint8) for _ in range(ndec)]
    n = C.c_uint64(0)

    def run():
        busy = [False] * ndec
        for i, x in enumerate(sigs):
            k = i % ndec
            if busy[k]:
                assert lib.apt_decoder_wait(decs[k], C.byref(n)) == 0
            assert lib.apt_decoder_submit_host(decs[k], x.ctypes.data, _lib.F32, x.size, 1, outs[k].ctypes.data, cap) == 0
            busy[k] = True
        for k in range(ndec):
            if busy[k]:
                assert lib.apt_decoder_wait(decs[k], C.byref(n)) == 0
    run._decs = decs
    return run


def timed(fns):
    """fns: name -> callable; alternated, `reps` rounds after one warm-up each."""
    for fn in fns.values():
        fn()
    t = {k: [] for k in fns}
    for _ in range(reps):
        for k, fn in fns.items():
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            t[k].append((time.perf_counter() - t0) * 1e3)
    return {k: stats(v) for k, v in t.items()}


key = f"batch_{B}x{args_.seconds}s_ms"
res[key] = {}
for name, kw in MODES.items() if "1" in args_.sections else ():
    rr = png_mode_round_robin(kw)
    fns = {"decode_batch_image_png": batch_image(kw, True), "a_decode_png_sequence": seq_decode_png(kw),
           "b_batch_rows_process_encode": rows_then_encode(kw), "c_png_mode_round_robin": rr,
           "decode_batch_image_pixels": batch_image(kw, False), "decode_batch_rows": batch_rows()}
    res[key][name] = timed(fns)
    for d in rr._decs:
        lib.apt_decoder_destroy(d)
    print(name, {k: round(v["median"], 1) for k, v in res[key][name].items()}, flush=True)
    with open(os.path.join(out_dir, "batch_png_times.json"), "w") as f:
        json.dump(res, f, indent=1)

res["gpu_after"] = gpu_name()
with open(os.path.join(out_dir, "batch_png_times.json"), "w") as f:
    json.dump(res, f, indent=1)
print("done", flush=True)
