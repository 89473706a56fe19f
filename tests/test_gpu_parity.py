"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle on the same inputs.

Tolerance (BASELINE.json north_star): decoded f32 values within 1e-5 of the reference.  Per-element
relative error is meaningless near envelope zeros (dsp.rs:373 subtracts nearly equal terms), so the
metric is  max|gpu - ref| / max|ref|  per stage, <= 1e-5; lengths and sync positions must be equal
exactly.  The only arithmetic difference to the oracle is FMA contraction in the FIR sums.
"""
import numpy as np
import pytest

import noaa_apt_b200 as na
from noaa_apt_b200 import synth
import oracle
from _sync_oracle import roots_direct

pytestmark = pytest.mark.gpu

TOL = 1e-5


def nerr(got, ref):
    assert got.shape == ref.shape, (got.shape, ref.shape)
    scale = float(np.max(np.abs(ref))) if ref.size else 1.0
    return float(np.max(np.abs(got.astype(np.float64) - ref.astype(np.float64)))) / (scale or 1.0)


@pytest.fixture(scope="module")
def rng():
    return np.random.default_rng(1234)


# ------------------------------------------------------------------------------- stages

@pytest.mark.parametrize("in_rate,out_rate", [(11025, 12480), (48000, 12480), (96000, 12480), (44100, 12480),
                                              (22050, 12480), (11025, 20800), (48000, 16640)])
def test_resample_with_filter_polyphase(rng, in_rate, out_rate):
    x = (rng.standard_normal(in_rate // 2) * 3000).astype(np.float32)
    f = na.filters.LowpassDcRemoval(na.Freq.hz(4800, in_rate), 30.0, na.Freq.hz(1000, in_rate))
    got = na.dsp.resample_with_filter(na.Context(), x, in_rate, out_rate, f)
    ref = oracle.resample_with_filter(x, in_rate, out_rate, oracle.FILTER_LOWPASS_DC,
                                      oracle.freq_hz(4800, in_rate), 30.0, oracle.freq_hz(1000, in_rate))
    assert nerr(got, ref) <= TOL


@pytest.mark.parametrize("in_rate,out_rate", [(24960, 12480), (12480, 12480), (12480, 4160), (49920, 12480)])
def test_resample_with_filter_l_equals_one(rng, in_rate, out_rate):
    # dsp.rs:105-123: filter (not resampled) then decimate
    x = (rng.standard_normal(30000) * 3000).astype(np.float32)
    f = na.filters.Lowpass(na.Freq.hz(4000, in_rate), 30.0, na.Freq.hz(1500, in_rate))
    got = na.dsp.resample_with_filter(na.Context(), x, in_rate, out_rate, f)
    ref = oracle.resample_with_filter(x, in_rate, out_rate, oracle.FILTER_LOWPASS,
                                      oracle.freq_hz(4000, in_rate), 30.0, oracle.freq_hz(1500, in_rate))
    assert nerr(got, ref) <= TOL


def test_resample_nofilter_decimate_zeroes_first_sample(rng):
    # decode.rs:158-159: NoFilter + decimate(3); dsp.rs:399 never reads signal[0]
    x = (rng.standard_normal(6240 * 4) * 10).astype(np.float32)
    got = na.dsp.resample_with_filter(na.Context(), x, 12480, 4160, na.filters.NoFilter())
    ref = oracle.resample_with_filter(x, 12480, 4160, oracle.FILTER_NONE)
    assert got[0] == 0.0
    assert np.array_equal(got, ref)


@pytest.mark.parametrize("in_rate,out_rate", [(11025, 48000), (11025, 6000), (11025, 3675), (11025, 80000),
                                              (11025, 11025)])
def test_wav_resample_tool_rates(rng, in_rate, out_rate):
    # test/test.sh:47-51 resamples the test recording to these rates (resample.rs:36-43 parameters)
    x = (rng.standard_normal(20000) * 8000).astype(np.float32)
    got = na.dsp.resample(na.Context(), x, in_rate, out_rate, 40.0, na.Freq.pi_rad(0.1))
    ref = oracle.resample(x, in_rate, out_rate, 40.0, 0.1)
    assert nerr(got, ref) <= TOL


def test_fast_resampling_zero_input_smoke():
    # dsp.rs:440-468: zeros in, no overflow, zeros out; also taps longer than the signal
    got = na.dsp.resample_with_filter(na.Context(), np.zeros(1000, np.float32), 1000, 1500, na.filters.NoFilter())
    assert got.size == oracle.resample_with_filter(np.zeros(1000, np.float32), 1000, 1500, oracle.FILTER_NONE).size
    assert not got.any()
    short = np.zeros(100, np.float32)
    f = na.filters.Lowpass(na.Freq.pi_rad(0.25), 60.0, na.Freq.pi_rad(0.005))   # thousands of taps
    got = na.dsp.resample_with_filter(na.Context(), short, 1000, 1500, f)
    ref = oracle.resample_with_filter(short, 1000, 1500, oracle.FILTER_LOWPASS, 0.25, 60.0, 0.005)
    assert got.size == ref.size and not got.any()


def test_demodulate_bit_exact(rng):
    # every op of dsp.rs:373 is rounded on its own on the device too -> identical bits
    x = (rng.standard_normal(100000) * 30).astype(np.float32)
    carrier = na.Freq.hz(2400, 12480)
    got = na.dsp.demodulate(na.Context(), x, carrier)
    ref = oracle.demodulate(x, oracle.freq_hz(2400, 12480))
    assert got[0] == 0.0
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))


def test_filter_lowpass(rng):
    x = np.abs(rng.standard_normal(50000) * 30).astype(np.float32)
    cut = np.float32(4160) / np.float32(12480)
    f = na.filters.Lowpass(na.Freq.pi_rad(cut), 25.0, na.Freq.pi_rad(cut) / 5.0)
    taps = f.design()
    assert taps.size == 37
    assert np.array_equal(taps, oracle.design(oracle.FILTER_LOWPASS, cut, 25.0, cut / np.float32(5)))
    got = na.dsp.filter(na.Context(), x, f)
    ref = oracle.filter(x, taps)
    assert got[0] == 0.0
    assert nerr(got, ref) <= TOL


def test_filter_short_signal(rng):
    x = rng.standard_normal(10).astype(np.float32)
    taps = rng.standard_normal(37).astype(np.float32)
    assert nerr(na.dsp.filter(na.Context(), x, taps), oracle.filter(x, taps)) <= TOL


def _oracle_filtered(rate, seconds, seed):
    x = synth.apt_signal(rate, seconds, seed)
    _, st = oracle.decode_steps(x, rate)
    return x, st


@pytest.mark.parametrize("work_rate", [12480, 16640, 20800])
def test_find_sync_positions_and_correlation(work_rate):
    prof = na.Settings.profile({12480: "standard", 16640: "fast", 20800: "slow"}[work_rate])
    s = oracle.default_settings()
    s.work_rate, s.resample_atten, s.resample_delta_freq = work_rate, prof.resample_atten, prof.resample_delta_freq
    s.resample_cutout, s.demodulation_atten = prof.resample_cutout, prof.demodulation_atten
    x = synth.apt_signal(11025, 20, seed=3)
    _, st = oracle.decode_steps(x, 11025, s)
    f = st["filtered"]
    pos, corr = na.find_sync(na.Context(), f, work_rate, want_correlation=True)
    ref_pos, ref_corr = oracle.find_sync(f, work_rate, want_corr=True)
    assert np.array_equal(corr.view(np.uint32), ref_corr.view(np.uint32))   # adds only, same order
    assert np.array_equal(pos, ref_pos)
    # inside decode() the correlation comes from the fused low-pass kernel (box sums: different summation
    # order, same values to fp32 rounding) -- the positions must still be the reference's
    with na.Decoder(11025, na.Settings.profile({12480: "standard", 16640: "fast", 20800: "slow"}[work_rate]),
                    max_samples=x.size) as dec:
        dec.decode(x)
        assert np.array_equal(dec.last_sync(), st["sync_pos"])
        assert nerr(dec.read_stage("correlation"), ref_corr) <= TOL
        assert nerr(dec.read_stage("filtered"), f) <= TOL


def test_find_sync_on_noise_and_silence(rng):
    # noisy stretch: the `while` at decode.rs:244 pushes duplicates; silence: every index is a root
    noise = np.abs(rng.standard_normal(6240 * 30)).astype(np.float32)
    assert np.array_equal(na.find_sync(na.Context(), noise, 12480), oracle.find_sync(noise, 12480))
    silence = np.zeros(6240 * 12, np.float32)
    assert np.array_equal(na.find_sync(na.Context(), silence, 12480), oracle.find_sync(silence, 12480))
    ramp = np.linspace(0, 100, 6240 * 12, dtype=np.float32)            # monotone: roots only at the end
    assert np.array_equal(na.find_sync(na.Context(), ramp, 12480), oracle.find_sync(ramp, 12480))
    neg = -np.abs(rng.standard_normal(6240 * 12)).astype(np.float32) - 1     # corr may stay <= 0: seed survives
    assert np.array_equal(na.find_sync(na.Context(), neg, 12480), oracle.find_sync(neg, 12480))


# ------------------------------------------------------------------------------- decode()

@pytest.mark.parametrize("rate,seconds", [(11025, 30), (48000, 20), (96000, 12), (44100, 12), (22050, 12)])
def test_decode_matches_oracle(rate, seconds):
    x = synth.apt_signal(rate, seconds, seed=rate % 97)
    ctx = na.Context()
    with na.Decoder(rate, na.Settings(), max_samples=x.size) as dec:
        got = dec.decode(x, sync=True)
        gpu_pos = dec.last_sync()
        env = dec.read_stage("demodulated")
        flt = dec.read_stage("filtered")
    ref, st = oracle.decode_steps(x, rate)
    assert env.size == st["demodulated"].size
    assert nerr(env, st["demodulated"]) <= TOL
    assert nerr(flt, st["filtered"]) <= TOL
    assert np.array_equal(gpu_pos, st["sync_pos"])
    assert got.size == ref.size and got.size % 2080 == 0
    assert nerr(got, ref) <= TOL
    # the one-shot entry point (noaa_apt::decode signature) gives the same rows and fires the
    # reference's status callbacks (decode.rs:63,87,93,107,154)
    got2 = na.decode(ctx, na.Settings(), x, na.Rate.hz(rate), True)
    assert np.array_equal(got2, got)
    assert [p for p, _ in ctx.log] == pytest.approx([0.1, 0.4, 0.42, 0.5, 0.9])
    assert ctx.log[0][1] == "Resampling to 12480" and ctx.log[3][1] == "Syncing"


@pytest.mark.parametrize("rate,profile", [(48000, "fast"), (48000, "slow"), (96000, "slow")])
def test_decode_other_profiles(rate, profile):
    # 48 kHz fast: L = 26, the tiled kernel's unrolled (3, 0, 3, 2) loop; 48 kHz slow (L/M = 13/30) and 96 kHz slow
    # (13/60): the tiled kernel's runtime loop with one half, 14 and 28 iterations (test_gpu_resampler_exact.py pins
    # every shape exactly)
    x = synth.apt_signal(rate, 12, seed=11)
    settings = na.Settings.profile(profile)
    os_ = oracle.default_settings()
    os_.work_rate, os_.resample_atten = settings.work_rate, settings.resample_atten
    os_.resample_delta_freq, os_.resample_cutout = settings.resample_delta_freq, settings.resample_cutout
    os_.demodulation_atten = settings.demodulation_atten
    got = na.decode(na.Context(), settings, x, rate, True)
    ref = oracle.decode(x, rate, os_)
    assert got.size == ref.size
    assert nerr(got, ref) <= TOL


def test_decode_pcm16_equals_f32():
    rate = 48000
    pcm = synth.apt_pcm16(rate, 12, seed=5)
    a = na.decode(na.Context(), na.Settings(), pcm, rate, True)
    b = na.decode(na.Context(), na.Settings(), pcm.astype(np.float32), rate, True)
    # both against the oracle fed with the `as f32` cast of wav.rs:37 (not against each other)
    ref = oracle.decode(oracle.pcm16_to_f32(pcm), rate)
    assert a.size == ref.size and nerr(a, ref) <= TOL
    assert b.size == ref.size and nerr(b, ref) <= TOL


def test_decode_no_sync():
    rate = 11025
    x = synth.apt_signal(rate, 12, seed=2)
    ctx = na.Context()
    got = na.decode(ctx, na.Settings(), x, rate, False)
    ref = oracle.decode(x, rate, sync=False)
    assert got.size == ref.size and got[0] == 0.0
    assert nerr(got, ref) <= TOL
    assert ctx.log[3][1] == "Skipping Syncing"


def test_decode_no_sync_work_rate_not_multiple_of_final_rate():
    # the final stage becomes a real L/M resample with the one-tap NoFilter (dsp.rs:79-98)
    rate = 11025
    x = synth.apt_signal(rate, 12, seed=2)
    settings = na.Settings(work_rate=11025)
    os_ = oracle.default_settings()
    os_.work_rate = 11025
    got = na.decode(na.Context(), settings, x, rate, False)
    ref = oracle.decode(x, rate, os_, sync=False)
    assert got.size == ref.size
    assert nerr(got, ref) <= TOL


def test_decode_errors_match_reference():
    # decode.rs:79-83
    with pytest.raises(na.err.Internal) as e:
        na.decode(na.Context(), na.Settings(), np.zeros(20000, np.float32), 11025, True)
    assert e.value.code == na._lib.ERR_TOO_SHORT
    # decode.rs:172-176 (sync needs work_rate % 4160 == 0)
    x = synth.apt_signal(11025, 12, seed=2)
    with pytest.raises(na.err.Internal) as e:
        na.decode(na.Context(), na.Settings(work_rate=11025), x, 11025, True)
    assert e.value.code == na._lib.ERR_WORK_RATE
    # dsp.rs:82-91
    with pytest.raises(na.err.RateOverflow):
        na.decode(na.Context(), na.Settings(work_rate=93911), x, 99371, True)
    # empty signal: the reference panics at dsp.rs:367
    with pytest.raises(na.err.InvalidInput):
        na.decode(na.Context(), na.Settings(), np.zeros(0, np.float32), 11025, True)


def test_decode_few_sync_frames():
    # decode.rs:112-118: 10-11 rows of signal give < 5 peaks only if the picker starts late; build a
    # signal whose oracle run reports the same condition, whatever it is
    rate = 11025
    x = synth.apt_signal(rate, 6, seed=9)   # ~12 rows at work rate: enough samples, few frames
    try:
        ref = oracle.decode(x, rate)
        ref_err = None
    except oracle.OracleError as e:
        ref, ref_err = None, e.code
    if ref_err is None:
        got = na.decode(na.Context(), na.Settings(), x, rate, True)
        assert got.size == ref.size
    else:
        with pytest.raises(na.err.Internal) as e:
            na.decode(na.Context(), na.Settings(), x, rate, True)
        assert e.value.code == ref_err


def test_decoder_reuse_and_batch():
    rate = 48000
    sigs = [synth.apt_signal(rate, 12 + i, seed=20 + i) for i in range(5)]
    refs = [oracle.decode(x, rate) for x in sigs]
    with na.Decoder(rate, na.Settings(), max_samples=max(s.size for s in sigs)) as dec:
        for x, ref in zip(sigs, refs):
            got = dec.decode(x)
            assert got.size == ref.size and nerr(got, ref) <= TOL
    outs, statuses = na.decode_batch(sigs, rate, na.Settings(), True, devices=[0], streams_per_device=3)
    assert statuses == [0] * 5
    for got, ref in zip(outs, refs):
        assert got.size == ref.size and nerr(got, ref) <= TOL


def test_decode_golden_fixture():
    """Committed golden rows (tests/golden/make_golden.py, generated with the CPU oracle)."""
    import os
    path = os.path.join(os.path.dirname(__file__), "golden", "decode_golden.npz")
    g = np.load(path)
    for rate in (11025, 48000, 96000):
        pcm = synth.apt_pcm16(rate, float(g[f"seconds_{rate}"]), seed=int(g[f"seed_{rate}"]))
        got = na.decode(na.Context(), na.Settings(), pcm, rate, True)
        ref = g[f"rows_{rate}"]
        assert got.size == ref.size
        assert nerr(got, ref) <= TOL


def test_parallel_and_sequential_picker_agree(monkeypatch):
    # k_pick_parallel (pointer doubling) and the one-thread walk must give the same peak list
    x = synth.apt_signal(48000, 40, seed=4)
    _, st = oracle.decode_steps(x, 48000)
    f = st["filtered"]
    par = na.find_sync(na.Context(), f, 12480)
    monkeypatch.setenv("APTB200_SEQUENTIAL_PICK", "1")
    seq = na.find_sync(na.Context(), f, 12480)
    assert np.array_equal(par, st["sync_pos"])
    assert np.array_equal(seq, st["sync_pos"])


@pytest.mark.parametrize("rate", [48000, 11025])
def test_chunked_upload_of_long_recordings(rate, monkeypatch):
    """BASELINE configs[2] in miniature: a recording longer than the staging chunk is uploaded in chunks with the
    filter-length overlap while the previous chunk is resampled; the result must not depend on the chunking."""
    pcm = synth.apt_pcm16(rate, 20, seed=31)
    x = pcm.astype(np.float32)
    ref, st = oracle.decode_steps(x, rate)
    with na.Decoder(rate, na.Settings(), max_samples=x.size) as dec:
        whole = dec.decode(x)
        whole_env = dec.read_stage("demodulated")
    monkeypatch.setenv("APTB200_CHUNK_SAMPLES", "150000")
    with na.Decoder(rate, na.Settings(), max_samples=x.size) as dec:
        got = dec.decode(x)
        env = dec.read_stage("demodulated")
        assert np.array_equal(dec.last_sync(), st["sync_pos"])
        got16 = dec.decode(pcm)
    assert np.array_equal(env, whole_env)          # same kernels, same tiles: bit-identical to the one-shot upload
    assert np.array_equal(got, whole)
    assert got.size == ref.size and nerr(got, ref) <= TOL
    assert got16.size == ref.size and nerr(got16, ref) <= TOL


# ------------------------------------------------------------------------------- fused sync stage

_roots_direct = roots_direct


@pytest.mark.parametrize("rate,profile,seconds", [(48000, "standard", 30), (11025, "standard", 40), (48000, "fast", 16),
                                                  (48000, "slow", 16)])
def test_fused_sync_stage_roots_match_definition(rate, profile, seconds):
    """kernels_sync2.cuh: the roots that come out of the per-tile records (f and corr never written) must be exactly the
    roots, by the definition, of the correlation read_stage materialises with k_lowpass_corr.  The two kernels share one
    low-pass, box-sum and correlation order, so that correlation has the record kernel's bits (test_gpu_sync_exact.py
    compares both with the float32 restatement)."""
    x = synth.apt_signal(rate, seconds, seed=17)
    settings = na.Settings.profile(profile)
    with na.Decoder(rate, settings, max_samples=x.size) as dec:
        dec.decode(x)
        roots = dec.last_roots()
        corr = dec.read_stage("correlation")          # materialised on demand by k_lowpass_corr
    dist = (2080 * settings.work_rate // 4160) * 8 // 10
    assert np.array_equal(roots, _roots_direct(corr, dist))


def test_fused_sync_stage_pool_overflow_redo(monkeypatch):
    """Silence: every index is a record, the pool overflows, wait() re-runs the sync stage with the legacy kernels."""
    rate = 48000
    x = synth.apt_signal(rate, 12, seed=5)
    x[x.size // 2:] = 0.0
    ref, st = oracle.decode_steps(x, rate)
    monkeypatch.setenv("APTB200_RECORD_POOL", "4096")
    with na.Decoder(rate, na.Settings(), max_samples=x.size) as dec:
        got = dec.decode(x)
        assert np.array_equal(dec.last_sync(), st["sync_pos"])
    assert got.size == ref.size and nerr(got, ref) <= TOL
    monkeypatch.delenv("APTB200_RECORD_POOL")
    with na.Decoder(rate, na.Settings(), max_samples=x.size) as dec:
        got = dec.decode(x)
        assert np.array_equal(dec.last_sync(), st["sync_pos"])
    assert got.size == ref.size and nerr(got, ref) <= TOL
