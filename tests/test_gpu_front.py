"""The first stage of decode() (front.hpp) on the GPU, one input rate per kind it can choose: 48 000 Hz tiled, 192 000 Hz
uniform-tap, 11 025 Hz phase-major, 8000 Hz generic, 24 960 Hz decimate (L = 1).  Every path into the first stage -- the
whole-recording submit, the chunked upload of a long host recording, the stream, device input that is not 16-byte
aligned, and the stand-alone resampler -- must give the rows the whole-recording decode gives, and that decode must match
the CPU oracle."""
import numpy as np
import pytest

import noaa_apt_b200 as na
from noaa_apt_b200 import _lib, synth
import oracle
import test_gpu_stream

pytestmark = pytest.mark.gpu

TOL = 1e-5
SECONDS = 16
RATES = [48000, 192000, 11025, 8000, 24960]
POLYPHASE = [48000, 192000, 11025, 8000]


def nerr(got, ref):
    assert got.shape == ref.shape, (got.shape, ref.shape)
    return float(np.max(np.abs(got.astype(np.float64) - ref.astype(np.float64)))) / float(np.max(np.abs(ref)))


def pcm(rate):
    return synth.apt_pcm16(rate, SECONDS, seed=rate % 89)


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("rate", RATES)
@pytest.mark.parametrize("sync", [True, False])
def test_stream_equals_decode(rate, sync):
    test_gpu_stream.check_equal(pcm(rate).astype(np.float32), rate, na.Settings(), sync, which=("fixed4800", "random"))


@pytest.mark.parametrize("rate", POLYPHASE)
def test_chunked_upload_equals_whole(rate, monkeypatch):
    x16 = pcm(rate)
    for x in (x16.astype(np.float32), x16):
        monkeypatch.delenv("APTB200_CHUNK_SAMPLES", raising=False)
        with na.Decoder(rate, na.Settings(), max_samples=x.size) as dec:
            whole = dec.decode(x)
            whole_env = dec.read_stage("demodulated")
        monkeypatch.setenv("APTB200_CHUNK_SAMPLES", "100000")
        with na.Decoder(rate, na.Settings(), max_samples=x.size) as dec:
            got = dec.decode(x)
            env = dec.read_stage("demodulated")
        assert same_bits(env, whole_env), x.dtype
        assert same_bits(got, whole), x.dtype


def decode_device(rate, x, offset):
    """Rows of a sync decode of device-resident samples that start `offset` samples into their allocation."""
    import torch
    buf = torch.zeros(x.size + 1, dtype=torch.int16 if x.dtype == np.int16 else torch.float32, device="cuda")
    buf[offset:offset + x.size] = torch.from_numpy(x).cuda()
    fmt = _lib.PCM16 if x.dtype == np.int16 else _lib.F32
    with na.Decoder(rate, na.Settings(), max_samples=x.size) as dec:
        bound = dec.out_bound(x.size)
        out = torch.empty(bound, dtype=torch.float32, device="cuda")
        dec.submit_device(buf.data_ptr() + offset * buf.element_size(), fmt, x.size, True, out.data_ptr(), bound)
        n = dec.wait()
    return out[:n].cpu().numpy()


@pytest.mark.parametrize("rate", POLYPHASE)
@pytest.mark.parametrize("dtype", [np.float32, np.int16])
def test_misaligned_device_input(rate, dtype, monkeypatch):
    """f32 that is not 16-byte aligned (uniform-tap) and PCM16 that cannot be cast to an aligned f32 copy (tiled,
    uniform-tap) run on the generic kernel; the tiled and phase-major kernels take misaligned f32 as it is, and the
    phase-major kernel misaligned PCM16 too."""
    x = pcm(rate).astype(dtype)
    got = decode_device(rate, x, 1)
    generic = (rate == 192000) or (dtype == np.int16 and rate == 48000)
    if generic:
        monkeypatch.setenv("APTB200_GENERIC_RESAMPLER", "1")
    ref = decode_device(rate, x, 0)
    assert same_bits(got, ref)


@pytest.mark.parametrize("rate", RATES)
def test_decode_matches_oracle(rate):
    x = pcm(rate).astype(np.float32)
    with na.Decoder(rate, na.Settings(), max_samples=x.size) as dec:
        got = dec.decode(x)
        pos = dec.last_sync()
    ref, st = oracle.decode_steps(x, rate)
    assert np.array_equal(pos, st["sync_pos"])
    assert nerr(got, ref) <= TOL


@pytest.mark.parametrize("rate", RATES)
def test_resample_with_filter_matches_oracle(rate):
    x = pcm(rate)[: rate * 2].astype(np.float32)
    f = na.filters.LowpassDcRemoval(na.Freq.hz(4800, rate), 30.0, na.Freq.hz(1000, rate))
    got = na.dsp.resample_with_filter(na.Context(), x, rate, 12480, f)
    ref = oracle.resample_with_filter(x, rate, 12480, oracle.FILTER_LOWPASS_DC, oracle.freq_hz(4800, rate), 30.0,
                                      oracle.freq_hz(1000, rate))
    assert nerr(got, ref) <= TOL
