"""The first stage on the GPU, pinned exactly on impulse trains (_impulse.py) at every kernel and loop shape the input
rates select: the resampled values bit for bit against the index-arithmetic restatement of fast_resampling, the fused
envelope element by element within a few ulp of the oracle's envelope of those exact values.

This sees what a max-normalised error bound cannot: a dropped or misplaced small tap, a wrong previous sample at a tile,
group, row or half boundary (the halo row, the exchange array, group 12's split rows), and any unit, chunk or tail
boundary that loses or repeats a sample.  The end-to-end checks cover the rates no other GPU test decodes."""
import numpy as np
import pytest

import noaa_apt_b200 as na
from noaa_apt_b200 import _lib, synth
import _impulse as imp
import _parity
import oracle
import test_gpu_stream

pytestmark = pytest.mark.gpu

IDS = [f"{r}-{p}" for r, p, *_ in imp.REPRESENTATIVES]
REPS = [r[:2] for r in imp.REPRESENTATIVES]
CHUNKED = [r[:2] for r in imp.REPRESENTATIVES if r[2] != "decimate"]
CHUNKED_IDS = [f"{r}-{p}" for r, p in CHUNKED]
# (rate, profile) pairs no other GPU test decodes end to end
NEW_RATES = [(32000, "fast"), (8000, "slow"), (20800, "standard"), (12000, "standard"), (24000, "standard"), (64000, "fast"),
             (24960, "fast"), (24960, "slow"), (120000, "standard"), (144000, "standard"), (37500, "standard"),
             (8000, "fast"), (16000, "standard"), (32000, "standard"), (64000, "standard"), (20800, "slow")]


def choice(rate, profile):
    return imp.settings(profile), imp.front_choice(rate, imp.settings(profile))


def resample(c, s, x):
    return na.dsp.resample_with_filter(na.Context(), x, c["rate"], s.work_rate, imp.front_filter(c["rate"], s))


def assert_exact(got, want, c, what=""):
    assert got.shape == want.shape, (what, got.shape, want.shape)
    assert not np.isnan(got).any(), what
    bad = np.flatnonzero(got != want)                   # +0 == -0
    assert bad.size == 0, f"{what}: " + imp.describe(bad, c["unit_out"])


def assert_envelope(env, r, s, c, what=""):
    miss = imp.envelope_misses(env, r, s.work_rate)
    assert miss.size == 0, f"{what}: " + imp.describe(miss, c["unit_out"], "envelope values")


def train(c, n, dtype=np.float32, seed=0, extra=()):
    w = imp.window(c["l"], c["m"], c["taps"].size)
    return imp.impulse_train(n, c["l"], c["m"], c["taps"].size, seed=c["rate"] % 97 + seed, dtype=dtype,
                             force=imp.unit_force(n, c["unit_in"], w, extra))


def decode_len(rate, s):
    """Input samples for a decode of ten work rows (decode.rs:79-83) and a little more."""
    return int(5.3 * rate) + 64


def envelope_of(c, s, x, sync=False):
    with na.Decoder(c["rate"], s, max_samples=x.size) as dec:
        dec.decode(x, sync=sync)
        return dec.read_stage("demodulated")


@pytest.mark.parametrize("rate,profile", REPS, ids=IDS)
def test_resampler_bit_exact(rate, profile):
    s, c = choice(rate, profile)
    x = imp.representative_train(c)
    assert_exact(resample(c, s, x), imp.exact_resample(x, c["l"], c["m"], c["taps"]), c)


def tail_lengths(c):
    """(outputs, input length) pairs whose last unit holds 1, 2, 3, 4, R-1, R, R+1, p_out-1, p_out, unit_out-1 and
    unit_out outputs (or the next count a length reaches where L > M skips some), each at four consecutive lengths
    (n mod 4 = 0..3: the bulk copy takes n & ~3 samples and the tail is stored by hand), and one length shorter than a
    unit.  Kinds whose unit is one output take 64 outputs as their unit."""
    l, m, nt = c["l"], c["m"], c["taps"].size
    uo = c["unit_out"] if c["unit_out"] > 1 else 64
    wants = sorted({j for j in (1, 2, 3, 4, c["R"] - 1, c["R"], c["R"] + 1, c["p_out"] - 1, c["p_out"], uo - 1, uo)
                    if 1 <= j <= uo})
    out = set()
    for k in [2 * uo + j for j in wants] + [max(uo // 2, 1)]:
        n = max(1, (k - 1) * m // l)
        while imp.exact_len(n, l, m, nt) < k:
            n += 1
        out |= {(imp.exact_len(v, l, m, nt), v) for v in range(n, n + 4)}
    return sorted(out)


@pytest.mark.parametrize("rate,profile", REPS, ids=IDS)
def test_resampler_tails(rate, profile):
    s, c = choice(rate, profile)
    for i, (k, n) in enumerate(tail_lengths(c)):
        x = train(c, n, seed=i)
        want = imp.exact_resample(x, c["l"], c["m"], c["taps"])
        assert_exact(resample(c, s, x), want, c, f"n = {n}, {k} outputs")


@pytest.mark.parametrize("dtype", [np.float32, np.int16])
@pytest.mark.parametrize("rate,profile", REPS, ids=IDS)
def test_fused_envelope(rate, profile, dtype):
    s, c = choice(rate, profile)
    x = train(c, decode_len(rate, s), dtype)
    r = imp.exact_resample(x, c["l"], c["m"], c["taps"])
    assert_envelope(envelope_of(c, s, x), r, s, c, np.dtype(dtype).name)


@pytest.mark.parametrize("rate,profile", CHUNKED, ids=CHUNKED_IDS)
def test_chunk_seams(rate, profile, monkeypatch):
    s, c = choice(rate, profile)
    caps = imp.seam_caps(c)
    n = max(decode_len(rate, s), 3 * max(caps) + 1000)
    seams = sorted({p for cap in caps for p in imp.seam_inputs(c, n, cap)})
    w = imp.window(c["l"], c["m"], c["taps"].size)
    keep = []                                           # seams of different caps may fall within one window
    for p in seams:
        if not keep or p - keep[-1] >= w + 2:
            keep.append(p)
    x = train(c, n, extra=keep)
    r = imp.exact_resample(x, c["l"], c["m"], c["taps"])
    monkeypatch.delenv("APTB200_CHUNK_SAMPLES", raising=False)
    whole = envelope_of(c, s, x)
    assert_envelope(whole, r, s, c, "whole upload")
    for cap in caps:
        monkeypatch.setenv("APTB200_CHUNK_SAMPLES", str(cap))
        env = envelope_of(c, s, x)
        assert_envelope(env, r, s, c, f"chunks of {cap}")
        assert np.array_equal(env.view(np.uint32), whole.view(np.uint32)), f"chunks of {cap}"


def same_kernel(kind, dtype, offset):
    """Whether device input `offset` samples into an allocation runs the kernel that offset 0 runs (front_launch): the
    uniform-tap kernel wants 16-byte aligned f32, and the tiled and uniform-tap kernels take PCM16 only through an
    aligned f32 copy; the generic kernel serves the rest."""
    if kind in ("tiled", "uniform-tap") and dtype == np.int16:
        return offset % 8 == 0
    if kind == "uniform-tap":
        return offset % 4 == 0
    return True


def envelope_device(c, s, x, offset):
    import torch
    buf = torch.zeros(x.size + 8, dtype=torch.int16 if x.dtype == np.int16 else torch.float32, device="cuda")
    buf[offset:offset + x.size] = torch.from_numpy(x).cuda()
    fmt = _lib.PCM16 if x.dtype == np.int16 else _lib.F32
    with na.Decoder(c["rate"], s, max_samples=x.size) as dec:
        bound = dec.out_bound(x.size)
        out = torch.empty(bound, dtype=torch.float32, device="cuda")
        dec.submit_device(buf.data_ptr() + offset * buf.element_size(), fmt, x.size, False, out.data_ptr(), bound)
        dec.wait()
        return dec.read_stage("demodulated")


@pytest.mark.parametrize("dtype", [np.float32, np.int16])
@pytest.mark.parametrize("rate,profile", REPS, ids=IDS)
def test_input_alignment(rate, profile, dtype):
    s, c = choice(rate, profile)
    x = train(c, decode_len(rate, s), dtype, seed=1)
    r = imp.exact_resample(x, c["l"], c["m"], c["taps"])
    base = envelope_device(c, s, x, 0)
    assert_envelope(base, r, s, c, "offset 0")
    for offset in range(1, 4 if dtype == np.float32 else 8):
        env = envelope_device(c, s, x, offset)
        assert_envelope(env, r, s, c, f"offset {offset}")
        if same_kernel(c["kind"], dtype, offset):
            assert np.array_equal(env.view(np.uint32), base.view(np.uint32)), f"offset {offset}"


def oracle_settings(s):
    o = oracle.default_settings()
    o.work_rate, o.resample_atten = s.work_rate, s.resample_atten
    o.resample_delta_freq, o.resample_cutout = s.resample_delta_freq, s.resample_cutout
    o.demodulation_atten = s.demodulation_atten
    return o


@pytest.mark.parametrize("rate,profile", NEW_RATES, ids=[f"{r}-{p}" for r, p in NEW_RATES])
def test_end_to_end_new_rates(rate, profile):
    s = imp.settings(profile)
    x = synth.apt_signal(rate, 12, seed=rate % 31)
    with na.Decoder(rate, s, max_samples=x.size) as dec:
        got = dec.decode(x)
        pos = dec.last_sync()
    ref, st = oracle.decode_steps(x, rate, oracle_settings(s))
    ties = _parity.sync_ties(pos, st["sync_pos"], st["filtered"], s.work_rate)
    a, b = _parity.rows_without(got, ties), _parity.rows_without(ref, ties)
    assert a.shape == b.shape
    assert float(np.max(np.abs(a.astype(np.float64) - b))) / float(np.max(np.abs(b))) <= 1e-5
    test_gpu_stream.check_equal(x, rate, s, True, which=("random",))
