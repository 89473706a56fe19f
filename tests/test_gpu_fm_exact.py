"""The FM demodulator on the GPU, pinned bit for bit against its float32 restatement (_fm_oracle.py): every output of
apt_fm_demod and of every channel of apt_fm_demod_channels, the noise in front of a pass included.

The five default rates select only two tile shapes (tz 512 with 8 plane partitions, tz 256 with 16).  The other shapes
DESIGN.md §10 accepts run here too: 16-output tiles with 128 partitions holding one or two planes each, the one-CTA-per-SM
fallback, D = 1, several 16-tap blocks per plane, and every APTB200_IQ_TILE that fits.  Each changes the order of the
sums, which a comparison to within 1e-5 of oracle_fm_demod cannot see.  Around them: the three formats, offsets that
skip the mix and that hit the exact points of sincospi, chunk seams, lengths at the grid edge, exact-zero stretches,
full-scale cs16, subnormal and overflowing cf32, eight channels in one launch, and NaN / Inf samples, which are staged
as 0 wherever a chunk window starts.
"""
import contextlib
import os

import numpy as np
import pytest

import _fm_oracle as fo
from test_gpu_iq import _pass

pytestmark = pytest.mark.gpu

RATES = [2_400_000, 1_200_000, 1_024_000, 2_048_000, 250_000]
FORMATS = ["cu8", "cs16", "cf32"]

# settings -> (D, qpad, tz, partitions) of the plan: the shapes the default rates never select
SHAPES = {
    "2.4M-audio12k": ((2_400_000, dict(audio_rate=12_000, cutout=5000.0)), (200, 16, 32, 128)),
    "2.4M-audio4k8": ((2_400_000, dict(audio_rate=4800, cutout=2000.0)), (500, 16, 32, 128)),
    "prime-96001": ((96_001, {}), (1, 32, 512, 8)),
    "1.2M-df3k": ((1_200_000, dict(delta_freq=3000.0)), (25, 48, 512, 8)),
    "250k-df1k": ((250_000, dict(delta_freq=1000.0)), (5, 112, 512, 8)),
}

EIGHT = [0, 37_000, -120_000, 37_000, 250_000, -400_000, 600_000, 1000]


def mixed_settings():
    """(iq_rate, settings keywords, offset_hz) of every case below; test_fm_oracle_cpu checks their phasor margins too."""
    out = [(r, {}, clamp(r, o)) for r in RATES for o in (37_000, -120_000)]
    for (r, kw), _ in SHAPES.values():
        off = 20_000 if r < 200_000 else 37_000
        out += [(r, kw, off), (r, kw, -off)]
    return out + [(2_400_000, {}, o) for o in EIGHT + [-600_000]]


@pytest.fixture(scope="module")
def na():
    import __graft_entry__ as entry
    entry.build()
    import noaa_apt_b200
    if noaa_apt_b200.device_count() < 1:
        pytest.skip("needs a CUDA device")
    return noaa_apt_b200


@contextlib.contextmanager
def env(name, value):
    old = os.environ.get(name)
    if value is None:
        os.environ.pop(name, None)
    else:
        os.environ[name] = str(value)
    try:
        yield
    finally:
        if old is None:
            os.environ.pop(name, None)
        else:
            os.environ[name] = old


def fmt_of(x):
    return {np.dtype(np.uint8): "cu8", np.dtype(np.int16): "cs16"}.get(x.dtype, "cf32")


def n_of(x):
    return x.size if x.dtype == np.complex64 else x.size // 2


def bits(a):
    """float32 bits with every NaN as 0x7fffffff: the device's and the host's NaNs differ in sign and payload."""
    a = np.ascontiguousarray(a, np.float32)
    return np.where(np.isnan(a), np.uint32(0x7FFFFFFF), a.view(np.uint32))


def clamp(iq_rate, offset):
    """offset, pulled inside |offset| + cutout < iq_rate / 2 as test_gpu_iq does."""
    if 2 * (abs(offset) + 22_000) >= iq_rate:
        return 0 if offset == 0 else int(np.sign(offset)) * (iq_rate // 2 - 22_000 - 1000)
    return offset


def assert_margin(plan, n):
    mp, mw = fo.phasor_margin(plan, n)
    assert mp > 2 * fo.SINCOSPI_ULP and mw > 2 * fo.LIBM_ULP, (plan.fs, plan.offset, mp, mw)


def assert_exact(got, st, what):
    want = st["a"]
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.flatnonzero(bits(got) != bits(want))
    if bad.size == 0:
        return
    m = int(bad[0])
    msg = f"{what}: {bad.size} of {want.size} outputs differ, first at {m}: device {got[m]!r}, restated {want[m]!r}"
    if m >= 1:
        zr, zi, re, im = st["zr"], st["zi"], st["re"][m - 1], st["im"][m - 1]
        msg += (f"; restated z[m-1] = ({zr[m - 1]!r}, {zi[m - 1]!r}), z[m] = ({zr[m]!r}, {zi[m]!r}), re = {re!r}, im = {im!r}, "
                f"atan2f restated {fo.atan2f(im, re)[0]!r}, correctly rounded atan2 {np.float32(np.arctan2(float(im), float(re)))!r}. "
                "The atan2f restatement is the code nvcc 12.9 emits for sm_90a: a toolkit change can invalidate it")
    raise AssertionError(msg)


def check(na, x, s, what, tile=None, chunk=None, st=None):
    """fm_demod of x on the device (APTB200_IQ_TILE = tile, APTB200_IQ_CHUNK = chunk) against the restatement."""
    fmt = fmt_of(x)
    st = st or fo.fm_stages(x, fmt, s, tile)
    assert_margin(st["plan"], n_of(x))
    with env("APTB200_IQ_TILE", tile), env("APTB200_IQ_CHUNK", chunk):
        got = na.iq.fm_demod(x, s)
    assert_exact(got, st, what)
    return st


def signal(iq_rate, fmt, offset, seconds=0.06, seed=11, noise_s=0.01):
    """noise_s seconds of noise, then a synthetic pass at offset."""
    return _pass(iq_rate, seconds, seed, offset, fmt, noise_s)


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("iq_rate", RATES)
def test_default_rates(na, iq_rate, fmt):
    offsets = [0, clamp(iq_rate, 37_000), clamp(iq_rate, -120_000)]
    x = signal(iq_rate, fmt, offsets[1])
    s0 = na.iq.IqSettings(iq_rate)
    sts = []
    for off in offsets:
        s = na.iq.IqSettings(iq_rate, offset_hz=off)
        sts.append(check(na, x, s, f"{iq_rate} {fmt} offset {off}"))
    for off, got, st in zip(offsets, na.iq.fm_demod_channels(x, s0, offsets), sts):
        assert_exact(got, st, f"{iq_rate} {fmt} channel at {off}")


@pytest.mark.parametrize("fmt", ["cu8", "cf32"])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_plan_shapes(na, shape, fmt):
    (iq_rate, kw), want = SHAPES[shape]
    off = 20_000 if iq_rate < 200_000 else 37_000
    s = na.iq.IqSettings(iq_rate, offset_hz=off, **kw)
    plan = fo.Plan(s)
    assert (plan.D, plan.qpad, plan.tz, plan.parts) == want
    x = signal(iq_rate, fmt, off, seconds=max(0.06, 600 * plan.D / iq_rate))
    check(na, x, s, f"{shape} {fmt}")
    s.offset_hz = -off
    check(na, x, s, f"{shape} {fmt} offset {-off}")


@pytest.mark.parametrize("tile", [16, 32, 64, 128, 256, 512])
def test_forced_tiles(na, tile):
    s = na.iq.IqSettings(1_200_000, offset_hz=-120_000)
    x = signal(1_200_000, "cs16", -120_000)
    assert fo.Plan(s, tile).tz == tile
    check(na, x, s, f"APTB200_IQ_TILE={tile}", tile=tile)


def test_forced_tiles_that_do_not_fit(na):
    s = na.iq.IqSettings(2_400_000, offset_hz=37_000, audio_rate=4800, cutout=2000.0)
    x = signal(2_400_000, "cu8", 37_000, seconds=0.3)
    for tile in (512, 48, 8):
        assert fo.Plan(s, tile).tz == 32
        check(na, x, s, f"APTB200_IQ_TILE={tile} ignored", tile=tile)


@pytest.mark.parametrize("offset", [600_000, -600_000])
def test_exact_sincospi_points(na, offset):
    """offset fs/4: every P is at a multiple of 1/2, where sincospi is exact (+-0 and +-1)."""
    s = na.iq.IqSettings(2_400_000, offset_hz=offset)
    plan = fo.Plan(s)
    _, _, exact = fo._sincospi_precise(fo._p_args(plan, np.arange(64)))
    assert exact.all()
    for fmt in FORMATS:
        check(na, signal(2_400_000, fmt, offset), s, f"fs/4 {offset} {fmt}")


@pytest.mark.parametrize("fmt", ["cu8", "cf32"])
def test_chunk_seams(na, fmt):
    s = na.iq.IqSettings(1_200_000, offset_hz=37_000)
    D = s.decimation
    x = signal(1_200_000, fmt, 37_000)
    st = check(na, x, s, "whole")
    for chunk in (D - 1, D, D + 1, 7919):
        check(na, x, s, f"APTB200_IQ_CHUNK={chunk}", chunk=chunk, st=st)
    short = x[: 2 * 6000] if fmt == "cu8" else x[:6000]
    check(na, short, s, "APTB200_IQ_CHUNK=1", chunk=1)


def test_lengths_mod_D(na):
    s = na.iq.IqSettings(1_200_000, offset_hz=-120_000)
    D = s.decimation
    x = signal(1_200_000, "cf32", -120_000, seconds=0.02, noise_s=0.0)
    for k in range(D):
        xs = x[: 400 * D + k]
        check(na, xs, s, f"n = 400 D + {k}")


@pytest.mark.parametrize("fmt", FORMATS)
def test_short_inputs(na, fmt):
    s = na.iq.IqSettings(1_200_000, offset_hz=37_000)
    D, N = s.decimation, fo.Plan(s).N
    x = signal(1_200_000, fmt, 37_000, seconds=0.01, noise_s=0.0)
    for n in (1, 2, D - 1, D, D + 1, N - 1, N, N + 1):
        xs = x[: 2 * n] if fmt != "cf32" else x[:n]
        check(na, xs, s, f"n = {n}")


@pytest.mark.parametrize("iq_rate", [2_400_000, 1_200_000])
def test_grid_edge(na, iq_rate):
    s = na.iq.IqSettings(iq_rate, offset_hz=37_000)
    plan = fo.Plan(s)
    D, tz = plan.D, plan.tz
    x = signal(iq_rate, "cu8", 37_000, seconds=(3 * (tz - 1) + 2) * D / iq_rate + 0.001, noise_s=0.0)
    for k in (1, 2, 3):
        for M in (k * (tz - 1) - 1, k * (tz - 1), k * (tz - 1) + 1):
            n = M * D - (k % D)                      # ceil(n / D) == M
            assert plan.out_len(n) == M
            check(na, x[: 2 * n], s, f"{M} outputs")


@pytest.mark.parametrize("fmt", ["cs16", "cf32"])
def test_zero_stretches(na, fmt):
    """Exact zeros make z exactly 0: atan2(+0, -0) then gives one-sample +audio_rate/2 outputs at some silence edges."""
    s = na.iq.IqSettings(1_200_000, offset_hz=37_000)
    x = signal(1_200_000, fmt, 37_000).copy()
    v = x.view(np.float32) if fmt == "cf32" else x
    for a, b in ((5_000, 9_000), (30_000, 30_700), (50_001, 58_333)):
        v[2 * a: 2 * b] = 0
    st = check(na, x, s, f"zero stretches {fmt}")
    assert np.any((st["zr"] == 0) & (st["zi"] == 0))


def test_cs16_full_scale(na):
    s = na.iq.IqSettings(1_200_000, offset_hz=-120_000)
    x = signal(1_200_000, "cf32", -120_000, noise_s=0.0)
    v = np.clip(np.rint(np.stack([x.real, x.imag], 1).ravel() * 40_000.0), -32768, 32767).astype(np.int16)
    v[100:140] = -32768
    v[1000:1040] = 32767
    check(na, v, s, "cs16 full scale")


def test_cf32_subnormal(na):
    s = na.iq.IqSettings(1_200_000, offset_hz=37_000)
    x = (signal(1_200_000, "cf32", 37_000) * np.float32(2.0 ** -135)).astype(np.complex64)
    assert np.any((x.real != 0) & (np.abs(x.real) < np.finfo(np.float32).tiny))
    check(na, x, s, "subnormal cf32")


def test_cf32_overflow(na):
    """re = z1.x z0.x + z1.y z0.y overflows: the NaN and Inf positions must be the restatement's."""
    s = na.iq.IqSettings(1_200_000, offset_hz=37_000)
    x = (signal(1_200_000, "cf32", 37_000) * np.float32(3e19)).astype(np.complex64)
    st = check(na, x, s, "overflowing cf32")
    assert not np.all(np.isfinite(st["re"]))


@pytest.mark.parametrize("fmt", ["cu8", "cf32"])
def test_eight_channels(na, fmt):
    offsets = EIGHT
    s0 = na.iq.IqSettings(2_400_000)
    x = signal(2_400_000, fmt, 37_000)
    sts = []
    for off in offsets:
        st = fo.fm_stages(x, fmt, na.iq.IqSettings(2_400_000, offset_hz=off))
        assert_margin(st["plan"], n_of(x))
        sts.append(st)
    for chunk in (None, 7919):
        with env("APTB200_IQ_CHUNK", chunk):
            outs = na.iq.fm_demod_channels(x, s0, offsets)
        for off, got, st in zip(offsets, outs, sts):
            assert_exact(got, st, f"channel at {off}, chunk {chunk}")


def test_nonfinite_samples(na):
    """A NaN and an Inf just in front of a chunk's halo and mid-tile: staged as 0, so whole and chunked agree."""
    s = na.iq.IqSettings(1_200_000, offset_hz=37_000)
    plan = fo.Plan(s)
    D, N, chunk = plan.D, plan.N, 7919
    x = signal(1_200_000, "cf32", 37_000).copy()

    def halo_start(c_hi):
        m = (c_hi - 1) // D + 1                      # the next chunk's first output
        return (m - 1) * D - (N - 1)                 # ... reads back to this sample

    bad = {halo_start(chunk) - 1: np.nan, halo_start(2 * chunk) - 1: np.inf, halo_start(3 * chunk) - 2: -np.inf,
           20_000 + 7: complex(np.nan, 0.5), 33_333: complex(1.0, np.inf)}
    for i, v in bad.items():
        x[i] = v
    st = fo.fm_stages(x, "cf32", s)
    assert np.all(np.isfinite(st["a"]))
    check(na, x, s, "non-finite samples, whole", st=st)
    check(na, x, s, f"non-finite samples, APTB200_IQ_CHUNK={chunk}", chunk=chunk, st=st)
    outs = na.iq.fm_demod_channels(x, na.iq.IqSettings(1_200_000), [37_000, 0])
    assert_exact(outs[0], st, "non-finite samples, channel")
    assert_exact(outs[1], fo.fm_stages(x, "cf32", na.iq.IqSettings(1_200_000)), "non-finite samples, channel at 0")
