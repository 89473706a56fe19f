"""Tracked sync timing: k_sync_track + k_track_back and the whole decode in both sync modes, 48 kHz x 900 s.

Prints one JSON line with the card's name and power limit (read in the same run), the per-kernel times of the tracked
decode (decoder profiling events, median over --reps jobs) and the wall time of a host decode in each mode (median,
modes alternating).  APTB200_TRACK_CLUSTER=4|8|16 selects the cluster size of k_sync_track."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import noaa_apt_b200 as na  # noqa: E402
from noaa_apt_b200 import synth  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=int, default=900)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    x = synth.apt_pcm16(48000, seconds=a.seconds, seed=1)
    out = {"card": card(), "seconds": a.seconds, "cluster": int(os.environ.get("APTB200_TRACK_CLUSTER", "8"))}
    with na.Decoder(48000, max_samples=x.size) as dec:
        dec.decode(x)
        dec.set_sync_mode("track")
        dec.decode(x)
        dec.set_profiling(True)
        ks = {}
        for _ in range(a.reps):
            dec.decode(x)
            for name, ms in dec.kernel_times_ms():
                ks.setdefault(name, []).append(ms)
        dec.set_profiling(False)
        out["kernel_ms"] = {k: float(np.median(v)) for k, v in ks.items()}
        wall = {"peaks": [], "track": []}
        for _ in range(a.reps):
            for mode in ("peaks", "track"):
                dec.set_sync_mode(mode)
                t = time.perf_counter()
                dec.decode(x)
                wall[mode].append((time.perf_counter() - t) * 1e3)
        out["decode_ms"] = {k: float(np.median(v)) for k, v in wall.items()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
