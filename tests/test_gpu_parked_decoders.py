"""One parked apt_decoder moving between the convenience entry points.  Each of them borrows a decoder of one (device,
rate, settings) key from the library's cache and hands it back; whatever the previous borrower set up (process or PNG
mode, a kept image, a status callback, a stager lent by a batch), the next call's output must be the one it gives on a
fresh decoder."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

RATE = 48_000
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def na():
    import __graft_entry__ as entry
    entry.build()
    import noaa_apt_b200
    if noaa_apt_b200.device_count() < 1:
        pytest.skip("needs a CUDA device")
    return noaa_apt_b200


@pytest.fixture(scope="module")
def inputs(na):
    from noaa_apt_b200 import synth
    x = synth.apt_pcm16(RATE, 12.0, seed=5)
    other = synth.apt_pcm16(RATE, 11.0, seed=6)
    iq_s = na.iq.IqSettings(1_200_000, offset_hz=-120_000, audio_rate=RATE)
    iq = synth.apt_iq(1_200_000, 12.0, seed=7, offset_hz=-120_000, fmt="cu8")
    palette = np.load(os.path.join(GOLDEN, "palettes.npz"))["noaa-apt-daylight"]
    return x, other, iq_s, iq, palette


def _steps(na, inputs):
    """(name, call) in the order the decoder moves through them; every call uses the key (device 0, 48 kHz, standard)."""
    from noaa_apt_b200 import image
    x, other, iq_s, iq, palette = inputs
    xf, otherf = x.astype(np.float32), other.astype(np.float32)

    def recording():
        with na.Recording(x, RATE) as rec:
            return rec.decode_image([(0, x.size), (7_777, x.size - 20_000)], contrast=image.TELEMETRY, rotate=True)

    def decode_iq():
        ctx = na.Context()
        return na.iq.decode_iq(iq, iq_s, context=ctx), ctx.log

    return [
        ("apt_decode_png", lambda: image.decode_png(None, None, x, RATE, contrast=image.PERCENT, palette=palette)),
        ("apt_decode_batch_image", lambda: image.decode_batch_png([other, x], RATE, png=True, streams_per_device=2)),
        ("apt_recording_decode", recording),
        ("apt_decode_iq", decode_iq),
        ("apt_decode", lambda: na.decode(None, None, xf, RATE)),
        ("apt_decode_pcm16", lambda: na.decode(None, None, x, RATE)),
        ("apt_decode_batch", lambda: na.decode_batch([xf, otherf], RATE, streams_per_device=2)),
    ]


def _same(got, want, what):
    if isinstance(want, (list, tuple)):
        assert isinstance(got, (list, tuple)) and len(got) == len(want), what
        for k, (g, w) in enumerate(zip(got, want)):
            _same(g, w, f"{what}[{k}]")
    elif isinstance(want, dict):
        assert isinstance(got, dict) and got.keys() == want.keys(), what
        for k in want:
            _same(got[k], want[k], f"{what}[{k!r}]")
    elif isinstance(want, np.ndarray):
        assert isinstance(got, np.ndarray) and got.dtype == want.dtype and got.shape == want.shape, what
        assert got.tobytes() == want.tobytes(), f"{what}: the bytes differ"
    else:
        assert got == want, what


def test_parked_decoder_between_entry_points(na, inputs, monkeypatch):
    lib = na._lib.load()
    steps = _steps(na, inputs)
    lib.apt_cache_clear()
    moved = [call() for _, call in steps]
    for (name, call), got in zip(steps, moved):
        lib.apt_cache_clear()
        _same(got, call(), name)
    x, other, *_ = inputs
    log = moved[3][1]
    assert log and any(desc == "Syncing" for _, desc in log), log

    # the rows also equal an explicit decoder's
    with na.Decoder(RATE, max_samples=x.size) as dec:
        want_x = dec.decode(x.astype(np.float32))
        _same(moved[4], want_x, "apt_decode vs Decoder")
        _same(moved[5], dec.decode(x), "apt_decode_pcm16 vs Decoder")
        rows, sts = moved[6]
        assert sts == [na._lib.OK] * 2
        _same(rows[0], want_x, "apt_decode_batch[0] vs Decoder")
        _same(rows[1], dec.decode(other.astype(np.float32)), "apt_decode_batch[1] vs Decoder")

    # the batch without the staging ring
    monkeypatch.setenv("APTB200_NO_STAGER", "1")
    lib.apt_cache_clear()
    _same(steps[6][1](), moved[6], "apt_decode_batch with APTB200_NO_STAGER")
    lib.apt_cache_clear()
