"""The streamed peak picker of apt_stream (kernels_stream.cuh), restated in numpy and run without a GPU.

carried_walk() feeds the correlation to the picker in growing final prefixes, as the stream does step by step: the roots
of the positions whose window (p, p+D] is final, the seed once corr[0..D] is final, then the orbit walk of
F(s) = max(firstroot(s) + D + 1, row*(s/row + 1)) with its duplicate pushes, stopping wherever the next start or its first
root is not decided yet.  At every split it also applies the stream's emission rule and its envelope retention.  The
positions must equal oracle.find_sync's on the whole correlation for any split; the rows released must cover what the
documented rule promises; the retained envelope must stay inside the bound the stream allocates for.
"""
import os

import numpy as np
import pytest

import noaa_apt_b200 as na
from noaa_apt_b200 import _lib, synth
from noaa_apt_b200.err import Error
import oracle
from _sync_oracle import carried_walk

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HALO = 80


def correlation(x, rate):
    steps = oracle.decode_steps(x, rate)[1]
    pos, corr = oracle.find_sync(steps["filtered"], 12480, want_corr=True)
    return pos, corr


def split_points(corr, pos, D, seed):
    rng = np.random.default_rng(seed)
    n = corr.size
    pts = set(rng.integers(1, n, size=40).tolist())
    pts |= set(rng.integers(1, D + 1, size=6).tolist()) | {D, D + 1}
    dup = np.nonzero(np.diff(pos.astype(np.int64)) == 0)[0]
    for i in dup[:6]:
        p = int(pos[i])
        pts |= {p, p + 1, p + D, p + D + 1}
    return sorted(x for x in pts if 0 < x < n)


def fade_out(rate, before, fade, after):
    """APT, then a carrier fading out (a rising correlation with no root: the reference's last peak chases it and the
    rows come out later as a run of duplicates), then APT again."""
    a = synth.apt_pcm16(rate, seconds=before, seed=6).astype(np.float32)
    n = rate * fade
    t = np.arange(n, dtype=np.float64) / rate
    carrier = (np.linspace(1.0, 0.01, n) * 12000 * np.sin(2 * np.pi * 2400 * t)).astype(np.float32)
    b = synth.apt_pcm16(rate, seconds=after, seed=7).astype(np.float32)
    return np.concatenate([a, carrier, b])


def recordings():
    z = np.load(os.path.join(ROOT, "tests", "golden", "test_11025hz_excerpts.npz"))
    return {
        "synth48k": (synth.apt_pcm16(48000, seconds=30, seed=4).astype(np.float32), 48000),
        "synth11k": (synth.apt_pcm16(11025, seconds=30, seed=5).astype(np.float32), 11025),
        "silence": (np.zeros(48000 * 20, np.float32), 48000),
        "fade_out": (fade_out(11025, 10, 200, 10), 11025),
        "excerpt_start": (z["pcm_start"].astype(np.float32), 11025),
        "excerpt_dup": (z["pcm_dup"].astype(np.float32), 11025),
    }


@pytest.fixture(scope="module")
def recs():
    return {k: (x, r) + correlation(x, r) for k, (x, r) in recordings().items()}


@pytest.mark.parametrize("name", ["synth48k", "synth11k", "silence", "fade_out", "excerpt_start", "excerpt_dup"])
@pytest.mark.parametrize("seed", [0, 1])
def test_carried_walk_equals_find_sync(recs, name, seed):
    x, rate, pos, corr = recs[name]
    D = 6240 * 8 // 10
    got = carried_walk(corr, 12480, split_points(corr, pos, D, seed))
    assert np.array_equal(got, pos)
    assert np.array_equal(carried_walk(corr, 12480, []), pos)          # one push of the whole file
    assert np.array_equal(carried_walk(corr, 12480, range(1, corr.size, 997)), pos)


def test_golden_excerpts_hold_a_duplicate(recs):
    pos = recs["excerpt_dup"][2]
    assert np.any(np.diff(pos.astype(np.int64)) == 0)


def test_fade_out_duplicate_run(recs):
    """A fade-out longer than the run ring holds rows makes one run of hundreds of duplicates whose rows are not final
    when it is pushed: the walk must wait for them (not spin) and still end on find_sync's positions, also with a ring
    of 2 runs and a row list of 1 (the end of the recording then drops runs whose rows cannot fit)."""
    x, rate, pos, corr = recs["fade_out"]
    p = pos.astype(np.int64)
    same = np.diff(p) == 0
    longest, run = 0, 0
    for v in same:
        run = run + 1 if v else 0
        longest = max(longest, run)
    assert longest > 256                                   # more duplicates than the run ring has entries
    pending = []
    for run_cap, gather_cap in ((256, 8), (2, 1)):
        got = carried_walk(corr, 12480, range(1000, corr.size, 1000),
                           lambda c, pk, st: pending.append(st["pending_runs"]), run_cap=run_cap, gather_cap=gather_cap)
        assert np.array_equal(got, pos)
    assert max(pending) <= 8
    got = carried_walk(corr, 12480, [corr.size - 7000], run_cap=2, gather_cap=1)   # the run appears only at the end
    assert np.array_equal(got, pos)


@pytest.mark.parametrize("name", ["synth48k", "silence", "fade_out", "excerpt_dup"])
def test_emission_rule_and_retention(recs, name):
    """After every step the rows the stream releases (k + 1 < peaks, p_k + row < work_final) cover the documented rule,
    and the envelope the stream keeps (from the first sample a pending row or peak can read) fits its bound."""
    x, rate, pos, corr = recs[name]
    row, G = 6240, 114
    D = row * 8 // 10
    geom = na.stream_geometry(rate, None, True, 24000)
    lat = geom["latency_work"]
    assert lat <= D + G
    final = pos.astype(np.int64)
    bound = row + D + G + HALO + 64           # the envelope tail the stream sizes its window for (stream.cu make_geom)
    seen = []

    def on_step(c_end, peaks, st):
        wf = c_end + G
        released = min(st["gathered"], max(len(peaks) - 1, 0))
        due = 0
        for k in range(final.size - 1):
            if max(final[k] + row, final[k + 1] + G) + lat <= wf:
                due = k + 1
            else:
                break
        assert released >= due, (c_end, released, due)
        if st["first_pending"] is not None:
            keep = st["first_pending"]
        elif st["seed_state"] < 2:
            keep = 0
        else:
            keep = st["s"] if st["s"] >= c_end else max(st["s"], st["decided"])
        keep = max(min(keep, c_end & ~15) - HALO, 0) & ~15
        if c_end > 2 * D + G:
            seen.append(wf - keep)
            assert wf - keep <= bound, (c_end, wf - keep, bound)

    carried_walk(corr, 12480, range(1000, corr.size, 1000), on_step)
    assert seen
    assert geom["device_bytes"] >= 2 * 4 * bound


def test_geometry_depends_on_parameters_only():
    a = na.stream_geometry(48000, None, True, 48000)
    b = na.stream_geometry(48000, na.Settings(), True, 48000)
    assert a == b
    assert a["max_push"] == 48000 and a["samples_in"] == 0
    assert na.stream_geometry(48000, None, True, 96000)["device_bytes"] > a["device_bytes"]
    for rate in (48000, 96000, 11025, 24960):
        for prof in ("standard", "fast", "slow"):
            s = na.Settings() if prof == "standard" else na.Settings.profile(prof)
            g = na.stream_geometry(rate, s, True, 24000)
            d = 2080 * (s.work_rate // 4160) * 8 // 10
            assert 0 < g["latency_work"] <= d + 38 * (s.work_rate // 4160)
            assert na.stream_geometry(rate, s, False, 24000)["latency_work"] == 0


@pytest.mark.parametrize("rate,work_rate,sync,max_push,code", [
    (0, None, True, 48000, _lib.ERR_BAD_ARG),
    (48000, None, True, 0, _lib.ERR_BAD_ARG),
    (48000, 11025, True, 48000, _lib.ERR_WORK_RATE),
    (48000, 11025, False, 48000, _lib.ERR_BAD_ARG),
])
def test_argument_errors_without_device(rate, work_rate, sync, max_push, code):
    s = na.Settings()
    if work_rate:
        s.work_rate = work_rate
    with pytest.raises(Error) as e:
        na.stream_geometry(rate, s, sync, max_push)
    assert e.value.code == code
    with pytest.raises(Error) as e:
        na.Stream(rate, s, sync=sync, max_push=max_push)
    assert e.value.code == code
