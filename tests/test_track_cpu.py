"""Tracked sync on the host (_track_oracle.py): the float32 restatement against the float64 rule, the positions against
the reference's picker on clean recordings, the noise tables of DESIGN.md "Tracked sync", and the settings checks."""
import ctypes as C
import os

import numpy as np
import pytest

import __graft_entry__ as entry
import noaa_apt_b200 as na
from noaa_apt_b200 import _lib, synth
import _track_oracle as to
import oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", autouse=True)
def built():
    entry.build()


def _steps(x, rate):
    _, st = oracle.decode_steps(np.asarray(x, dtype=np.float32), rate)
    f = st["filtered"]
    _, corr = oracle.find_sync(f, 12480, want_corr=True)
    return f, corr, st["sync_pos"].astype(np.int64)


@pytest.fixture(scope="module")
def clean3():
    return _steps(synth.apt_signal(11025, seconds=120, seed=3), 11025)


@pytest.fixture(scope="module")
def excerpt():
    z = np.load(os.path.join(ROOT, "tests", "golden", "test_11025hz_excerpts.npz"))
    return _steps(z["pcm_start"].astype(np.float32), int(z["rate"]))


def test_f32_matches_f64_rule(clean3, excerpt):
    for f, corr, _ in (clean3, excerpt):
        for delta, lam in ((2, 0.25), (1, 0.0), (8, 1.0)):
            p32, _, _ = to.track_f32(corr, 6240, delta, lam)
            p64 = to.track_f64(corr, 6240, delta, lam)
            np.testing.assert_array_equal(p32, p64)


def test_clean_seed3_positions(clean3):
    _, corr, ref = clean3
    pos, _, _ = to.track_f32(corr, 6240)
    d = np.abs(pos[None, :] - ref[:, None]).min(axis=1)
    assert d.max() <= 1, d.max()
    exact = np.isin(pos, ref).sum()
    one_off = sum(1 for p in pos if p not in set(ref.tolist()) and np.abs(ref - p).min() == 1)
    extra = [int(p) for p in pos if np.abs(ref - p).min() > 1]
    assert (pos.size, exact, one_off) == (240, 144, 95), (pos.size, exact, one_off)
    assert extra == [6250], extra


def test_real_excerpt_covers_reference(excerpt):
    """The excerpt starts in noise, where the reference's rows land anywhere; every reference position one row period
    (+-2) from the next is on the signal's row lattice, and there tracked sync agrees within 1 sample."""
    _, corr, ref = excerpt
    pos, _, _ = to.track_f32(corr, 6240)
    steady = ref[:-1][np.abs(np.diff(ref) - 6240) <= 2]
    assert steady.size >= 20
    assert np.abs(pos[None, :] - steady[:, None]).min(axis=1).max() <= 1


@pytest.mark.parametrize("rate", [11025, 48000])
def test_noise_table(rate):
    """The σ = 20 000 row of the table: the reference's picker loses the rows, tracked sync keeps them.  The noise is
    white over the input band, so at 48 000 Hz σ grows with sqrt(48 000 / 11 025) for the same noise in the APT band."""
    clean = synth.apt_signal(rate, seconds=120, seed=3)
    _, _, truth = _steps(clean, rate)
    rng = np.random.default_rng(1)
    noisy = (clean + rng.normal(0.0, 20000.0 * np.sqrt(rate / 11025), clean.size)).astype(np.float32)
    _, corr, ref = _steps(noisy, rate)
    pos, _, _ = to.track_f32(corr, 6240)
    assert to.score(ref, truth) < 0.2
    assert to.score(pos, truth) > 0.95


@pytest.mark.parametrize("sigma,ref_below", [(10000, 0.7), (20000, 0.1)])
def test_clock_drift_table(sigma, ref_below):
    """Content synthesised at 11 027 Hz and declared 11 025 Hz (181 ppm: the period drifts by about one sample per row);
    truth is the reference on the clean drifted signal."""
    drift = synth.apt_signal(11027, seconds=120, seed=3)[: 120 * 11025]
    _, _, truth = _steps(drift, 11025)
    rng = np.random.default_rng(1)
    _, corr, ref = _steps(drift + rng.normal(0.0, sigma, drift.size), 11025)
    assert to.score(ref, truth) < ref_below
    assert to.score(to.track_f32(corr, 6240)[0], truth) > 0.95


def test_sigma_40000_row():
    """At σ = 40 000 the outcome depends on the noise draw (DESIGN.md §15); on this draw the reference keeps no row and
    tracked sync more than half of them."""
    clean = synth.apt_signal(11025, seconds=120, seed=3)
    _, _, truth = _steps(clean, 11025)
    rng = np.random.default_rng(2)
    _, corr, ref = _steps(clean + rng.normal(0.0, 40000.0, clean.size), 11025)
    assert to.score(ref, truth) < 0.01
    assert to.score(to.track_f32(corr, 6240)[0], truth) > 0.5


def test_rows_rule():
    f = np.arange(100000, dtype=np.float32)
    rows = to.rows_from_positions(f, np.array([0, 6240, 12480, 93000]), 6240, 3, f.size)
    assert rows.size == 3 * 2080 and rows[2080] == 6240.0 and rows[1] == 3.0 and rows[0] == 0.0


def _set(delta, lam, mode=1):
    """apt_decoder_set_sync_mode on no decoder: the mode and the settings are checked first, on the host."""
    lib = _lib.load()
    ts = _lib.CTrackSettings(delta, lam)
    rc = lib.apt_decoder_set_sync_mode(None, mode, C.byref(ts))
    return rc, lib.apt_last_error().decode()


def test_default_settings():
    ts = _lib.CTrackSettings()
    _lib.load().apt_default_track_settings(C.byref(ts))
    assert (ts.delta, ts.lambda_) == (2, 0.25)


@pytest.mark.parametrize("delta,lam,mode,what", [
    (0, 0.25, 1, "delta"), (9, 0.25, 1, "delta"), (2, -0.5, 1, "lambda"), (2, float("nan"), 1, "lambda"),
    (2, float("inf"), 1, "lambda"), (2, 0.25, 2, "mode"), (2, 0.25, -1, "mode"),
    (1, 0.0, 1, "null decoder"), (8, 3.0, 1, "null decoder"), (0, -1.0, 0, "null decoder"),
])
def test_settings_checks(delta, lam, mode, what):
    rc, msg = _set(delta, lam, mode)
    assert rc == _lib.ERR_BAD_ARG
    assert what in msg, msg


def test_python_rejects_unknown_mode():
    d = na.Decoder.__new__(na.Decoder)
    d._lib, d._h = _lib.load(), None
    with pytest.raises(ValueError):
        d.set_sync_mode("nearest")
    with pytest.raises(ValueError):
        na.decode(None, None, np.zeros(10, np.float32), 11025, sync="nearest")
