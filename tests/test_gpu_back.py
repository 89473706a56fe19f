"""The back half of decode() (back.hpp) on the GPU, every kind it can run, both by the input that selects it and by the
switch that forces it: Records (48 kHz standard / fast / slow, 11 025 Hz), Hbm (a record-pool overflow, and
APTB200_LEGACY_SYNC), Generic (a low-pass of 47 taps, and APTB200_GENERIC_LOWPASS), with and without sync, the final
resample of a work rate that is not a multiple of 4160, and apt_find_sync.  Each is checked against the CPU oracle, the
roots against their definition on the correlation, and the profiling slots and launch count of a job against fixed lists
(slot names and launch counts are part of what a profiling user sees)."""
import numpy as np
import pytest

import noaa_apt_b200 as na
from noaa_apt_b200 import synth
import oracle
from test_gpu_parity import _roots_direct, nerr

pytestmark = pytest.mark.gpu

TOL = 1e-5

FRONT = ["resample_envelope"]
SYNC_SLOTS = {
    "records": FRONT + ["lowpass_records", "resolve_roots", "sync_pick", "gather_rows"],
    "hbm": FRONT + ["lowpass_correlation", "sync_roots", "sync_pick", "gather_rows"],
    "generic": FRONT + ["lowpass", "sync_correlation", "sync_roots", "sync_pick", "gather_rows"],
}
# the overflow job runs the Records kernels, then the Hbm kernels again on the same envelope
SYNC_SLOTS["redo"] = SYNC_SLOTS["records"] + SYNC_SLOTS["hbm"][1:]
NOSYNC_SLOTS = {
    "records": FRONT + ["gather_rows"],
    "hbm": FRONT + ["lowpass", "gather_rows"],
    "generic": FRONT + ["lowpass", "gather_rows"],
    # 11 025 Hz input at work rate 11 025: the first stage is filter + decimate (L = 1)
    "final": ["filter_decimate", "envelope", "lowpass", "final_resample"],
}


def settings_pair(profile="standard", **kw):
    """(library settings, oracle settings) of a profile with some fields replaced."""
    s = na.Settings.profile(profile)
    for k, v in kw.items():
        setattr(s, k, v)
    o = oracle.default_settings()
    for k in ("work_rate", "resample_atten", "resample_delta_freq", "resample_cutout", "demodulation_atten"):
        setattr(o, k, getattr(s, k))
    return s, o


def run(rate, settings, x, sync):
    """One profiled decode: rows, positions, roots, f, corr, slot names, launches of the job."""
    with na.Decoder(rate, settings, max_samples=x.size) as dec:
        dec.set_profiling(True)
        before = dec.launch_count
        rows = dec.decode(x, sync=sync)
        launches = dec.launch_count - before
        slots = [name for name, _ in dec.kernel_times_ms()]
        pos = dec.last_sync() if sync else None
        roots = dec.last_roots() if sync else None
        f = dec.read_stage("filtered")
        corr = dec.read_stage("correlation") if sync else None
    return rows, pos, roots, f, corr, slots, launches


def check(rate, x, settings, osettings, sync, slots):
    rows, pos, roots, f, corr, got_slots, launches = run(rate, settings, x, sync)
    ref, st = oracle.decode_steps(x, rate, osettings, sync=sync) if sync else (oracle.decode(x, rate, osettings, sync=False), None)
    assert got_slots == slots
    assert launches == len(slots)
    assert rows.size == ref.size and nerr(rows, ref) <= TOL
    if not sync:
        return
    assert np.array_equal(pos, st["sync_pos"])
    assert nerr(f, st["filtered"]) <= TOL
    _, ref_corr = oracle.find_sync(st["filtered"], settings.work_rate, want_corr=True)
    assert nerr(corr, ref_corr) <= TOL
    dist = (2080 * settings.work_rate // 4160) * 8 // 10
    assert np.array_equal(roots, _roots_direct(corr, dist))


@pytest.mark.parametrize("rate,profile", [(48000, "standard"), (48000, "fast"), (48000, "slow"), (11025, "standard")])
@pytest.mark.parametrize("sync", [True, False])
def test_records(rate, profile, sync):
    s, o = settings_pair(profile)
    x = synth.apt_signal(rate, 14, seed=41)
    check(rate, x, s, o, sync, (SYNC_SLOTS if sync else NOSYNC_SLOTS)["records"])


def test_hbm_after_pool_overflow(monkeypatch):
    monkeypatch.setenv("APTB200_RECORD_POOL", "4096")
    s, o = settings_pair()
    x = synth.apt_signal(48000, 14, seed=42)
    x[x.size // 2:] = 0.0                       # silence: every index a record
    check(48000, x, s, o, True, SYNC_SLOTS["redo"])


@pytest.mark.parametrize("sync", [True, False])
def test_hbm_forced(sync, monkeypatch):
    monkeypatch.setenv("APTB200_LEGACY_SYNC", "1")
    s, o = settings_pair()
    x = synth.apt_signal(48000, 14, seed=43)
    check(48000, x, s, o, sync, (SYNC_SLOTS if sync else NOSYNC_SLOTS)["hbm"])


@pytest.mark.parametrize("sync", [True, False])
def test_generic_low_pass(sync):
    s, o = settings_pair(demodulation_atten=30.0)   # 47 taps at 12 480 Hz: no fused kernel
    x = synth.apt_signal(48000, 14, seed=44)
    check(48000, x, s, o, sync, (SYNC_SLOTS if sync else NOSYNC_SLOTS)["generic"])


@pytest.mark.parametrize("sync", [True, False])
def test_generic_forced(sync, monkeypatch):
    monkeypatch.setenv("APTB200_GENERIC_LOWPASS", "1")
    s, o = settings_pair()
    x = synth.apt_signal(11025, 20, seed=45)
    check(11025, x, s, o, sync, (SYNC_SLOTS if sync else NOSYNC_SLOTS)["generic"])


def test_generic_final_resample():
    s, o = settings_pair(work_rate=11025)
    x = synth.apt_signal(11025, 14, seed=46)
    check(11025, x, s, o, False, NOSYNC_SLOTS["final"])


@pytest.mark.parametrize("sequential", [False, True])
def test_find_sync(sequential, monkeypatch):
    if sequential:
        monkeypatch.setenv("APTB200_SEQUENTIAL_PICK", "1")
    x = synth.apt_signal(48000, 14, seed=47)
    _, st = oracle.decode_steps(x, 48000)
    pos, corr = na.find_sync(na.Context(), st["filtered"], 12480, want_correlation=True)
    ref_pos, ref_corr = oracle.find_sync(st["filtered"], 12480, want_corr=True)
    assert np.array_equal(pos, ref_pos)
    assert np.array_equal(corr.view(np.uint32), ref_corr.view(np.uint32))


@pytest.mark.parametrize("legacy", [False, True])
def test_grid_and_cluster_walks_agree(legacy, monkeypatch):
    """Both walks on one recording; the Records kind counts the cluster walk's two kernels, the Hbm kind counts one."""
    if legacy:
        monkeypatch.setenv("APTB200_LEGACY_SYNC", "1")
    x = synth.apt_signal(48000, 30, seed=48)
    _, st = oracle.decode_steps(x, 48000)
    slots = SYNC_SLOTS["hbm" if legacy else "records"]
    for walk, extra in (("grid", 0), ("cluster", 0 if legacy else 1)):
        monkeypatch.setenv("APTB200_PICK", walk)
        _, pos, _, _, _, got_slots, launches = run(48000, na.Settings(), x, True)
        assert np.array_equal(pos, st["sync_pos"]), walk
        assert got_slots == slots and launches == len(slots) + extra, walk


def test_find_sync_refuses_a_work_rate_beyond_the_picker():
    # 41 600 Hz: min_distance 16 640 > 16 384, the most k_roots holds; decode() refuses sync there too
    with pytest.raises(na.err.InvalidInput):
        na.find_sync(na.Context(), np.ones(20800 * 3, np.float32), 41600)
