"""Config 1 of BASELINE.json: decode the reference's own test recording on the
CPU (plumbing run).  The reference cannot be executed (no Rust toolchain), so
this checks the oracle against the independent numpy-f32 cross-check numbers
recorded in SURVEY.md Appendix C.

The recording itself (18 MB of incompressible PCM16) is not part of the
repository; its two excerpts in tests/golden/test_11025hz_excerpts.npz
(tests/golden/make_wav_excerpt.py) are.  Between them they hold every extreme
and every sync spacing Appendix C quotes, and the start excerpt the first sync
positions of the whole file.  The per-excerpt counts and means are the
oracle's own (a drift guard).
"""
import os

import numpy as np

import oracle

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "test_11025hz_excerpts.npz")


def _decode(g, name):
    return oracle.decode_steps(oracle.pcm16_to_f32(g[f"pcm_{name}"]), 11025)


def test_decode_reference_recording_matches_survey_numbers():
    g = np.load(GOLDEN)
    assert int(g["rate"]) == 11025
    assert str(g["sha256"]).startswith("50160851becd5997")
    (out_s, st_s), (out_d, st_d) = _decode(g, "start"), _decode(g, "dup")
    # [0 s, 40 s) and [230 s, 250 s): 441 000 and 220 500 input samples
    assert (g["pcm_start"].size, g["pcm_dup"].size) == (441_000, 220_500)
    assert (st_s["resampled"].size, st_d["resampled"].size) == (499_191, 249_591)
    assert (st_s["sync_pos"].size, st_d["sync_pos"].size) == (79, 39)
    assert (out_s.size, out_d.size) == (78 * 2080, 37 * 2080)
    assert st_s["sync_pos"][:4].tolist() == [3989, 13153, 19644, 26047]
    d = np.concatenate([np.diff(st_s["sync_pos"].astype(np.int64)), np.diff(st_d["sync_pos"].astype(np.int64))])
    assert (np.median(d), d.min(), d.max()) == (6240, 0, 18708)
    res = np.concatenate([st_s["resampled"], st_d["resampled"]])
    assert abs(float(res.min()) - (-26.86)) < 0.01
    assert abs(float(res.max()) - 32.86) < 0.01
    assert abs(float(max(st_s["demodulated"].max(), st_d["demodulated"].max())) - 67.60) < 0.01
    out = np.concatenate([out_s, out_d])
    assert abs(float(out.min()) - (-3.02)) < 0.01 and abs(float(out.max()) - 44.78) < 0.01
    assert abs(float(out_s.mean(dtype=np.float64)) - 9.76) < 0.01
    assert abs(float(out_d.mean(dtype=np.float64)) - 8.86) < 0.01
