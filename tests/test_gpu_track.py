"""Tracked sync on the GPU (DESIGN.md "Tracked sync"): k_sync_track + k_track_back against the float32 restatement
(_track_oracle.py) on the correlation the decoder itself computed, the rows against the oracle's, the image and PNG
modes against apt_process / apt_png_encode of those rows, the switch back to the reference's picker, the statuses, and
the noise table."""
import numpy as np
import pytest

import __graft_entry__ as entry
import _track_oracle as to
import oracle
from noaa_apt_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def na():
    entry.build()
    import noaa_apt_b200
    return noaa_apt_b200


def _run(na, x, rate, settings=None, delta=2, lam=0.25):
    with na.Decoder(rate, settings, max_samples=x.size) as dec:
        dec.set_sync_mode("track", delta, lam)
        rows = dec.decode(x)
        pos = dec.last_sync().astype(np.int64)
        corr = dec.read_stage("correlation")
        f = dec.read_stage("filtered")
        counts = dec.last_counts()
    return rows, pos, corr, f, counts


def _check(rows, pos, corr, f, counts, row, dec, delta=2, lam=0.25):
    want, _, _ = to.track_f32(corr, row, delta, lam)
    np.testing.assert_array_equal(pos, want)
    ref_rows = to.rows_from_positions(f, pos, row, dec, f.size)
    np.testing.assert_array_equal(rows, ref_rows)
    assert counts["n_peaks"] == pos.size and counts["n_rows"] * 2080 == rows.size


@pytest.mark.parametrize("rate", [11025, 22050, 48000, 96000])
@pytest.mark.parametrize("profile", ["standard", "fast", "slow"])
def test_positions_and_rows(na, rate, profile):
    st = na.Settings.profile(profile)
    x = synth.apt_signal(rate, seconds=30, seed=5)
    rows, pos, corr, f, counts = _run(na, x, rate, st)
    row = st.work_rate // 2
    _check(rows, pos, corr, f, counts, row, st.work_rate // 4160)
    # the rows against the oracle's filtered signal at the same positions
    o = oracle.default_settings()
    for k in ("work_rate", "resample_atten", "resample_delta_freq", "resample_cutout", "demodulation_atten"):
        setattr(o, k, getattr(st, k))
    _, steps = oracle.decode_steps(x, rate, o)
    want = to.rows_from_positions(steps["filtered"], pos, row, st.work_rate // 4160, steps["filtered"].size)
    assert rows.size == want.size
    assert np.max(np.abs(rows - want)) / np.max(np.abs(want)) <= 1e-5


@pytest.mark.parametrize("delta", range(1, 9))
def test_delta(na, delta):
    rng = np.random.default_rng(delta)
    x = (synth.apt_signal(11025, seconds=40, seed=2) + rng.normal(0, 15000, 40 * 11025)).astype(np.float32)
    lam = [0.0, 0.25, 1.0, 3.5][delta % 4]
    rows, pos, corr, f, counts = _run(na, x, 11025, delta=delta, lam=lam)
    _check(rows, pos, corr, f, counts, 6240, 3, delta, lam)


def test_pcm16(na):
    x = synth.apt_pcm16(48000, seconds=30, seed=9)
    rows, pos, corr, f, counts = _run(na, x, 48000)
    _check(rows, pos, corr, f, counts, 6240, 3)
    _, pos32, _, _, _ = _run(na, x.astype(np.float32), 48000)
    np.testing.assert_array_equal(pos, pos32)


def test_long_recording(na):
    """10 minutes: about 1200 blocks through every CTA of the cluster, and noise so that the path moves."""
    rng = np.random.default_rng(4)
    x = (synth.apt_signal(11025, seconds=600, seed=6) + rng.normal(0, 25000, 600 * 11025)).astype(np.float32)
    rows, pos, corr, f, counts = _run(na, x, 11025)
    _check(rows, pos, corr, f, counts, 6240, 3)


def test_image_and_png_modes(na):
    from noaa_apt_b200 import image
    x = synth.apt_pcm16(48000, seconds=40, seed=12)
    rows, _, _, _, _ = _run(na, x, 48000)
    with na.Decoder(48000, max_samples=x.size) as dec:
        dec.set_sync_mode("track")
        dec.set_process_mode(contrast=image.MINMAX)
        img = dec.decode(x)
        dec.set_png_mode()
        png = dec.decode(x)
    want, _ = image.process(rows, image.MINMAX)
    np.testing.assert_array_equal(img, want)
    assert png == image.encode_png(want)


def test_switch_back_to_peaks(na):
    x = synth.apt_pcm16(48000, seconds=30, seed=7)
    with na.Decoder(48000, max_samples=x.size) as dec:
        before = dec.decode(x)
        pos_before = dec.last_sync()
        dec.set_sync_mode("track")
        dec.decode(x)
        dec.set_sync_mode("peaks")
        after = dec.decode(x)
        np.testing.assert_array_equal(dec.last_sync(), pos_before)
    np.testing.assert_array_equal(after, before)


def test_decode_function(na):
    x = synth.apt_signal(11025, seconds=30, seed=5)
    rows, _, _, _, _ = _run(na, x, 11025)
    np.testing.assert_array_equal(na.decode(None, None, x, 11025, sync="track"), rows)


def test_statuses(na):
    """Under ten rows is APT_ERR_TOO_SHORT.  From ten rows on the walk back steps at most P + delta, so it finds at least
    nine positions: APT_ERR_FEW_SYNC_FRAMES cannot come back, and ten rows of silence decode (z = 0 everywhere)."""
    x = synth.apt_signal(11025, seconds=30, seed=5)
    with na.Decoder(11025, max_samples=x.size) as dec:
        dec.set_sync_mode("track")
        with pytest.raises(na.err.Error) as e:
            dec.decode(x[: 11025 * 4])
        assert e.value.code == na._lib.ERR_TOO_SHORT
        silent = np.zeros(11025 * 6, np.float32)
        rows = dec.decode(silent)
        pos = dec.last_sync().astype(np.int64)
        assert pos.size >= 9 and rows.size == dec.last_counts()["n_rows"] * 2080
        np.testing.assert_array_equal(pos, to.track_f32(dec.read_stage("correlation"), 6240)[0])
        with pytest.raises(na.err.Error) as e:
            dec.set_sync_mode("track", delta=9)
        assert e.value.code == na._lib.ERR_BAD_ARG


def test_noise_table_on_gpu(na):
    clean = synth.apt_signal(11025, seconds=120, seed=3)
    _, st = oracle.decode_steps(clean, 11025)
    truth = st["sync_pos"].astype(np.int64)
    rng = np.random.default_rng(1)
    noisy = (clean + rng.normal(0.0, 20000.0, clean.size)).astype(np.float32)
    _, pos, corr, _, _ = _run(na, noisy, 11025)
    np.testing.assert_array_equal(pos, to.track_f32(corr, 6240)[0])
    assert to.score(pos, truth) > 0.95


@pytest.mark.parametrize("delta,rem", [(2, 1), (8, 1), (8, 7)])
def test_last_block_shorter_than_delta(na, delta, rem):
    """ncorr % P in 1 .. delta - 1: the last block has fewer columns than the first-delta-columns head that the last CTA
    computes again, and the decoder holds exactly ncorr correlation values (max_samples = the recording)."""
    P, G = 6240, 114
    x0 = synth.apt_signal(12480, n_samples=30 * 12480, seed=8)
    with na.Decoder(12480, max_samples=x0.size) as dec:
        dec.decode(x0, sync=False)
        nwork0 = dec.last_counts()["n_work"]
    n = x0.size + (rem - (nwork0 - G)) % P
    x = synth.apt_signal(12480, n_samples=n, seed=8)
    rng = np.random.default_rng(rem)
    x = (x + rng.normal(0, 15000, x.size)).astype(np.float32)
    rows, pos, corr, f, counts = _run(na, x, 12480, delta=delta)
    assert corr.size % P == rem, corr.size
    _check(rows, pos, corr, f, counts, P, 3, delta)


@pytest.mark.parametrize("work_rate", [8320, 20800, 37440])
def test_other_work_rates(na, work_rate):
    """P = 4160, 10400 and 18720: other slice widths per CTA (W = 520 .. 2340 of the 2560 a CTA holds)."""
    st = na.Settings.profile("standard")
    st.work_rate = work_rate
    rng = np.random.default_rng(work_rate)
    x = (synth.apt_signal(48000, seconds=40, seed=3) + rng.normal(0, 20000, 40 * 48000)).astype(np.float32)
    rows, pos, corr, f, counts = _run(na, x, 48000, st)
    _check(rows, pos, corr, f, counts, work_rate // 2, work_rate // 4160)


def test_generic_lowpass_route(na, monkeypatch):
    """A decoder whose low-pass has no fused kernel (here forced by APTB200_GENERIC_LOWPASS) materialises f and corr with
    the exact-order Generic kernels before the tracked sync."""
    monkeypatch.setenv("APTB200_GENERIC_LOWPASS", "1")
    x = synth.apt_signal(11025, seconds=30, seed=5)
    with na.Decoder(11025, max_samples=x.size) as dec:
        dec.set_sync_mode("track")
        dec.set_profiling(True)
        rows = dec.decode(x)
        names = [n for n, _ in dec.kernel_times_ms()]
        pos = dec.last_sync().astype(np.int64)
        corr, f, counts = dec.read_stage("correlation"), dec.read_stage("filtered"), dec.last_counts()
    assert "lowpass" in names and "sync_correlation" in names and "lowpass_correlation" not in names, names
    assert "sync_track" in names and "sync_backtrack" in names, names
    _check(rows, pos, corr, f, counts, 6240, 3)
