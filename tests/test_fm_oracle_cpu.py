"""The float32 restatement of the FM demodulator (_fm_oracle.py), checked without a GPU.

- atan2f is within 2 ulp of the float64 atan2 on 10^7 random pairs, and equal to it rounded on the special values;
- P and W are the float32 phasors oracle_fm_demod uses, except at the exact points of sincospi, and every phasor the
  GPU file uses is far enough from a float32 rounding boundary for libm's and CUDA's errors not to matter;
- the restated z is within float32 rounding of the exact channel filter, and the audio is oracle_fm_demod's to 1e-5
  where the discriminator is well conditioned;
- the plan restatement gives DESIGN.md §10's defaults and the tile shapes of the GPU file;
- a comparison with the restatement can fail: a reordered tap loop, reversed partitions, float32 phasors, an FMA in
  the discriminator or a correctly rounded atan2 each change outputs on the GPU file's inputs.
"""
import numpy as np
import pytest

import __graft_entry__ as entry
import noaa_apt_b200 as na
import _fm_oracle as fo
import oracle
from test_gpu_fm_exact import SHAPES, clamp, mixed_settings, signal
from test_iq_cpu import TABLE, _phasor, oracle_for

F32 = np.float32


@pytest.fixture(scope="module", autouse=True)
def built():
    entry.build()


def ordered(a):
    """float32 bits as integers in the order of the values (for ulp distances)."""
    b = np.ascontiguousarray(a, F32).view(np.int32).astype(np.int64)
    return np.where(b < 0, -(b & 0x7FFFFFFF), b)


def ulps(a, b):
    return np.abs(ordered(a) - ordered(b))


def rn_atan2(y, x):
    return np.arctan2(np.asarray(y, np.float64), np.asarray(x, np.float64)).astype(F32)


def test_atan2f_random_pairs():
    rng = np.random.default_rng(5)
    worst = 0
    for k in range(10):
        n = 1_000_000
        mag = np.float64(2.0) ** rng.uniform(-40, 40, (2, n))
        v = (mag * rng.choice([-1.0, 1.0], (2, n))).astype(F32)
        if k % 2:                                    # ratios near 1: where |y| > |x| switches branch
            v[1] = (v[0] * (1 + rng.uniform(-1e-3, 1e-3, n))).astype(F32) * rng.choice([-1, 1], n).astype(F32)
        got = fo.atan2f(v[0], v[1])
        worst = max(worst, int(ulps(got, rn_atan2(v[0], v[1])).max()))
    assert worst <= 2, worst


def test_atan2f_special_values():
    f = np.finfo(F32)
    one, nxt = F32(1), np.nextafter(F32(1), F32(2))
    tiny = np.array([1, 2, 3, 0x7FFFFF, 0x400000], np.uint32).view(F32)     # subnormals
    vals = [0.0, -0.0, 1.0, -1.0, np.inf, -np.inf, 3.5, -7.25, f.max, -f.max, f.tiny, -f.tiny]
    ys, xs = np.meshgrid(np.array(vals + list(tiny) + list(-tiny), F32), np.array(vals + list(tiny), F32))
    y, x = ys.ravel(), xs.ravel()
    got, want = fo.atan2f(y, x), rn_atan2(y, x)
    exact = (y == 0) | (x == 0) | np.isinf(y) | np.isinf(x)
    # the signed-zero combinations, infinities and x = -0 are exact, signs included
    assert np.array_equal(got[exact].view(np.uint32), want[exact].view(np.uint32))
    # |y| = |x|, subnormals over normals and over each other, ratios next to 1: within the bound
    assert ulps(got, want).max() <= 2
    eq = np.array([1.0, 3.0, 1e-30, 1e30, 5e-39], F32)
    for sy in (1, -1):
        for sx in (1, -1):
            g = fo.atan2f(sy * eq, sx * eq)
            assert np.all(g == g[0]) and ulps(g, rn_atan2(sy * eq, sx * eq)).max() <= 1
    for a, b in ((one, nxt), (nxt, one), (-one, nxt), (one, -nxt)):
        assert ulps(fo.atan2f(a, b), rn_atan2(a, b)).max() <= 1
    # a subnormal over 1 is returned unchanged: atan(t) rounds to t
    assert np.array_equal(fo.atan2f(tiny, np.ones_like(tiny)), tiny)
    nan = fo.atan2f(np.array([np.nan, 1, np.nan, np.inf], F32), np.array([1, np.nan, np.nan, np.nan], F32))
    assert np.all(np.isnan(nan))


@pytest.mark.parametrize("iq_rate,offset", [(2_400_000, 37_000), (2_400_000, -120_000), (1_200_000, 577_999),
                                            (2_048_000, 1000), (250_000, -102_000), (2_400_000, 600_000)])
def test_phasors(iq_rate, offset):
    plan = fo.Plan(na.iq.IqSettings(iq_rate, offset_hz=offset))
    fs = np.uint64(iq_rate)
    q = np.arange(4096, dtype=np.uint64)
    Pr, Pi = fo.p_table(plan, q.size)
    want_r, want_i = _phasor(((q * np.uint64(fo.B)) % fs) * np.uint64(plan.f) % fs, iq_rate)
    s, c, exact = fo._sincospi_precise(fo._p_args(plan, q))
    m = np.minimum(fo._margin(s), fo._margin(c))
    listed = exact | (m < 64)
    differ = (Pr.view(np.uint32) != want_r.view(np.uint32)) | (Pi.view(np.uint32) != want_i.view(np.uint32))
    assert not np.any(differ & ~listed), np.flatnonzero(differ & ~listed)[:8]
    # at the exact points the values are the exact ones; cos(2 pi v / fs) in double is off by rounding there
    assert np.all(np.isin(Pr[exact], [0, 1, -1])) and np.all(np.isin(Pi[exact], [0, 1, -1]))
    Wr, Wi = fo.w_table(plan)
    wr, wi = _phasor((np.arange(fo.B, dtype=np.uint64) * np.uint64(plan.f)) % fs, iq_rate)
    a = fo._exact_ld(fo._w_angles(plan))
    mw = np.minimum(fo._margin(np.cos(a)), fo._margin(np.sin(a)))
    wdiff = (Wr.view(np.uint32) != wr.view(np.uint32)) | (Wi.view(np.uint32) != wi.view(np.uint32))
    assert not np.any(wdiff & (mw >= 64))
    print(f"{iq_rate} {offset}: {exact.sum()} exact P points, {int((differ & listed).sum())} P and {int(wdiff.sum())} W values "
          f"differ from cos / sin of 2 pi v / fs in double")


def test_exact_points_and_signed_zeros():
    s, c, exact = fo._sincospi_precise(np.array([-0.0, -0.5, -1.0, -1.5, -0.25]))
    assert exact.tolist() == [True, True, True, True, False]
    assert np.signbit(s[0]) and s[0] == 0 and c[0] == 1               # v = 0: P = (1, -0)
    assert c[1] == 0 and not np.signbit(c[1]) and s[1] == -1
    assert c[2] == -1 and s[2] == 0 and np.signbit(s[2])              # sinpi(-1) = -0
    assert c[3] == 0 and not np.signbit(c[3]) and s[3] == 1


def test_phasor_margins_of_the_gpu_cases():
    for iq_rate, kw, off in mixed_settings():
        plan = fo.Plan(na.iq.IqSettings(iq_rate, offset_hz=off, **kw))
        mp, mw = fo.phasor_margin(plan, iq_rate)                     # one second: more than any case uses
        assert mp > 2 * fo.SINCOSPI_ULP and mw > 2 * fo.LIBM_ULP, (iq_rate, kw, off, mp, mw)


@pytest.mark.parametrize("iq_rate,offset,fmt", [(2_400_000, 37_000, "cu8"), (1_200_000, -120_000, "cf32"),
                                                (250_000, 0, "cs16")])
def test_agrees_with_oracle_fm_demod(iq_rate, offset, fmt):
    s = na.iq.IqSettings(iq_rate, offset_hz=offset)
    x = signal(iq_rate, fmt, offset, seconds=0.1, noise_s=0.02)
    st = fo.fm_stages(x, fmt, s)
    plan = st["plan"]
    h = oracle.design(oracle.FILTER_LOWPASS, oracle.freq_hz(s.cutout, iq_rate), s.atten, oracle.freq_hz(s.delta_freq, iq_rate))
    assert np.array_equal(h, plan.h)
    # z against the exact filter of the staged samples: each side within N 2^-24 sum |h| |s| of it, so the restated z and
    # oracle_fm_demod's (ascending k, no FMA) are within N 2^-23 sum |h| |s| of each other
    D, N = plan.D, plan.N
    sc = st["sr"].astype(np.float64) + 1j * st["si"].astype(np.float64)
    full = np.convolve(sc, h.astype(np.float64))[: sc.size][::D]
    bound = N * 2.0 ** -24 * np.convolve(np.abs(sc), np.abs(h.astype(np.float64)))[: sc.size][::D]
    z = st["zr"].astype(np.float64) + 1j * st["zi"].astype(np.float64)
    assert np.all(np.abs(z.real - full.real) <= bound) and np.all(np.abs(z.imag - full.imag) <= bound)
    ref = oracle_for(x, fmt, s)
    first = int(iq_rate * 0.02) // D + 20
    err = np.max(np.abs(st["a"][first:] - ref[first:])) / np.max(np.abs(ref[first:]))
    assert err <= 1e-5, err


def test_plan_restatement():
    for iq_rate, (audio, D, taps) in TABLE.items():
        p = fo.Plan(na.iq.IqSettings(iq_rate))
        assert (p.audio_rate, p.D, p.N, p.qpad) == (audio, D, taps, 16)
        assert (p.tz, p.parts) == ((256, 16) if iq_rate in (2_400_000, 2_048_000) else (512, 8))
    assert fo.Plan(na.iq.IqSettings(2_400_000)).smem(256) == 109_328             # DESIGN.md §10: 110 KB at 2.4 Msps
    for (iq_rate, kw), want in SHAPES.values():
        p = fo.Plan(na.iq.IqSettings(iq_rate, **kw))
        assert (p.D, p.qpad, p.tz, p.parts) == want
    p = fo.Plan(na.iq.IqSettings(2_400_000, audio_rate=12_000, cutout=5000.0))
    assert [len(range(r, p.D, p.parts)) for r in (0, 71, 72, 127)] == [2, 2, 1, 1]
    p = fo.Plan(na.iq.IqSettings(2_400_000, audio_rate=4800, cutout=2000.0))
    assert p.smem(p.tz) > fo.SMEM_TWO and p.smem(p.tz) <= fo.SMEM_MAX                 # one CTA per SM
    for tile, want in ((16, 16), (32, 32), (64, 64), (128, 128), (256, 256), (512, 512), (48, 512), (8, 512), (1024, 512)):
        assert fo.Plan(na.iq.IqSettings(1_200_000), tile).tz == want
        assert fo.Plan(na.iq.IqSettings(1_200_000), tile).parts == fo.THREADS // (want // 16)
    assert fo.Plan(na.iq.IqSettings(2_400_000, audio_rate=4800, cutout=2000.0), 512).tz == 32     # does not fit: ignored


def test_nonfinite_samples_are_staged_as_zero():
    s = na.iq.IqSettings(1_200_000, offset_hz=37_000)
    x = signal(1_200_000, "cf32", 37_000, seconds=0.02, noise_s=0.0).copy()
    y = x.copy()
    for i, v in ((1000, np.nan), (2000, np.inf), (3000, complex(1.0, -np.inf))):
        x[i] = v
        y[i] = 0
    a, b = fo.fm_stages(x, "cf32", s), fo.fm_stages(y, "cf32", s)
    assert np.array_equal(a["a"].view(np.uint32), b["a"].view(np.uint32)) and np.all(np.isfinite(a["a"]))


@pytest.mark.parametrize("variant", fo.VARIANTS)
def test_the_comparison_can_fail(variant):
    """Each variant changes one step; on the GPU file's inputs it must change outputs, or the GPU file could not see it."""
    total = 0
    for iq_rate, fmt, off, kw in ((2_400_000, "cu8", 37_000, {}), (1_200_000, "cf32", clamp(1_200_000, -120_000), {}),
                                  (250_000, "cs16", 37_000, dict(delta_freq=1000.0))):
        s = na.iq.IqSettings(iq_rate, offset_hz=off, **kw)
        x = signal(iq_rate, fmt, off)
        want = fo.fm_stages(x, fmt, s)["a"]
        got = fo.fm_stages(x, fmt, s, variant=variant)["a"]
        n = int(np.sum(got.view(np.uint32) != want.view(np.uint32)))
        print(f"{variant}: {n} of {want.size} outputs differ at {iq_rate} {fmt} offset {off}")
        total += n
    assert total > 0
