"""The PNG encoder on the device (kernels_png.cuh) against the CPU restatement of DESIGN.md §11 in tests/_png_oracle.py:
the bytes must be identical.  Then the decode + process + PNG paths: apt_decode_png, the decoder's PNG mode and
apt_decode_wav_png, whose images must be exactly apt_decode_image's."""
import io
import os

import numpy as np
import pytest
from PIL import Image

import noaa_apt_b200 as na
from noaa_apt_b200 import image, synth
import _png_oracle as po

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def excerpt():
    return np.load(os.path.join(GOLDEN, "argentina_excerpt.npz"))["grey"]


@pytest.fixture(scope="module")
def palette():
    return np.load(os.path.join(GOLDEN, "palettes.npz"))["noaa-apt-daylight"]


def _rgba(grey):
    out = np.empty(grey.shape + (4,), dtype=np.uint8)
    out[..., :3] = grey[..., None]
    out[..., 3] = 255
    return out


def _pixels(png):
    with Image.open(io.BytesIO(png)) as im:
        return np.asarray(im)


def _same(got, ref):
    assert len(got) == len(ref), (len(got), len(ref))
    a, b = np.frombuffer(got, np.uint8), np.frombuffer(ref, np.uint8)
    bad = np.nonzero(a != b)[0]
    assert bad.size == 0, f"{bad.size} bytes differ, first at {bad[0]} of {a.size}"


def _synthetic(h, w, ch, seed):
    """Smooth gradients, flat runs and noise: every filter type wins somewhere and matches of every length occur."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    base = ((x * 3 + y * 5) % 256).astype(np.uint8)
    base[h // 3: h // 2] = 77
    noise = rng.integers(0, 256, (h, w), dtype=np.uint8)
    img = np.where((x // 5 + y // 3) % 4 == 0, noise, base).astype(np.uint8)
    if ch == 1:
        return img
    out = np.stack([img, img[::-1], np.roll(img, 7, axis=1), np.full_like(img, 255)][:ch], axis=2)
    return np.ascontiguousarray(out)


@pytest.mark.parametrize("block_bytes", [4096, 16384, 65536])
@pytest.mark.parametrize("filt", [-1, 0, 1, 2, 3, 4])
def test_excerpt_grey_bit_identical(excerpt, filt, block_bytes):
    img = excerpt[:120]
    got = image.encode_png(img, filt, True, block_bytes)
    _same(got, po.encode(img, filt, 1, block_bytes))
    assert np.array_equal(_pixels(got), img)


@pytest.mark.parametrize("matches", [True, False])
@pytest.mark.parametrize("block_bytes", [4096, 65536])
def test_excerpt_rgba_bit_identical(excerpt, matches, block_bytes):
    img = _rgba(excerpt[:200])
    got = image.encode_png(img, -1, matches, block_bytes)
    _same(got, po.encode(img, -1, int(matches), block_bytes))
    got3 = image.encode_png(img, -1, matches, block_bytes, rgb_from_rgba=True)
    _same(got3, po.encode(img, -1, int(matches), block_bytes, rgb_from_rgba=1))
    assert np.array_equal(_pixels(got3), img[..., :3])


@pytest.mark.parametrize("ch", [1, 3, 4])
@pytest.mark.parametrize("w", [1, 7, 2080])
def test_synthetic_bit_identical(ch, w):
    h = {1: 3000, 7: 700, 2080: 40}[w]
    img = _synthetic(h, w, ch, seed=w * 10 + ch)
    if ch == 1:
        img = img[:, :]
    for filt, matches, bb in ((-1, 1, 4096), (-1, 0, 65536), (4, 1, 8192), (1, 1, 65536)):
        got = image.encode_png(img, filt, bool(matches), bb)
        _same(got, po.encode(img, filt, matches, bb))
        assert np.array_equal(_pixels(got).reshape(img.shape), img)


def test_skewed_inputs_bit_identical():
    rng = np.random.default_rng(5)
    cases = [np.zeros((64, 2080), np.uint8), np.full((10, 3, 4), 255, np.uint8),
             rng.integers(0, 256, (100, 1000), dtype=np.uint8), np.arange(256, dtype=np.uint8)[None, :].repeat(9, 0)]
    for img in cases:
        for bb in (4096, 65536):
            got = image.encode_png(img, -1, True, bb)
            _same(got, po.encode(img, -1, 1, bb))


def test_repeated_calls_identical(excerpt):
    img = _rgba(excerpt)
    a = image.encode_png(img)
    for _ in range(3):
        assert image.encode_png(img) == a
    assert len(a) <= image.png_bound(2080, img.shape[0], 4)


def test_72000_row_rgba_round_trip(excerpt):
    rows = 72000
    reps = -(-rows // excerpt.shape[0])
    grey = np.tile(excerpt, (reps, 1))[:rows]
    grey[::97] ^= 0x5A                       # break the period so the image is not one long match
    img = _rgba(grey)
    del grey
    png = image.encode_png(img)
    assert len(png) <= image.png_bound(2080, rows, 4)
    Image.MAX_IMAGE_PIXELS = None
    back = _pixels(png)
    assert back.shape == img.shape and np.array_equal(back, img)


# ---------------------------------------------------------------------------------------- decode + process + PNG

@pytest.fixture(scope="module")
def pass_48k():
    pcm = synth.apt_pcm16(48000, seconds=900, seed=21)
    return pcm


VARIANTS = [
    dict(contrast=image.MINMAX),
    dict(contrast=image.MINMAX, rgba=True),
    dict(contrast=image.PERCENT, rotate=True, palette="daylight", tune=(0.4, -0.3, -0.6, 0.8)),
    dict(contrast=image.HISTOGRAM),
    dict(contrast=image.TELEMETRY, rgba=True),
]


def _kw(v, palette):
    kw = dict(v)
    if kw.get("palette") == "daylight":
        kw["palette"] = palette
    return kw


@pytest.mark.parametrize("fmt", ["f32", "pcm16"])
def test_decode_png_equals_decode_image(pass_48k, palette, fmt):
    sig = pass_48k if fmt == "pcm16" else pass_48k.astype(np.float32)
    for v in VARIANTS:
        kw = _kw(v, palette)
        img, info = image.decode_image(na.Context(), na.Settings(), sig, 48000, True, **kw)
        png, info2 = image.decode_png(na.Context(), na.Settings(), sig, 48000, True, **kw)
        assert info2["rows"] == info["rows"] == img.shape[0]
        assert np.array_equal(_pixels(png), img), v
        assert png == image.encode_png(img), v
        if img.ndim == 3:
            png3, _ = image.decode_png(na.Context(), na.Settings(), sig, 48000, True, rgb_from_rgba=True, **kw)
            assert png3 == image.encode_png(img, rgb_from_rgba=True)


def test_decode_png_from_fm_demod_audio(palette):
    # a full 900 s pass at 250 ksps cu8; the audio apt_fm_demod returns (50 kHz) is decoded as f32
    iq = synth.apt_iq(250_000, seconds=900, seed=4, offset_hz=37000, fmt="cu8")
    s = na.iq.IqSettings(250_000, offset_hz=37000)
    audio = na.iq.fm_demod(iq, s)
    del iq
    for kw in (dict(contrast=image.MINMAX), dict(contrast=image.TELEMETRY, rotate=True, palette=palette, rgba=True)):
        img, _ = image.decode_image(na.Context(), na.Settings(), audio, s.audio_rate, True, **kw)
        png, _ = image.decode_png(na.Context(), na.Settings(), audio, s.audio_rate, True, **kw)
        assert img.shape[0] > 1700
        assert np.array_equal(_pixels(png), img) and png == image.encode_png(img)


def test_decoder_png_mode_jobs_and_switching(pass_48k, palette):
    x = pass_48k.astype(np.float32)
    lens = [x.size, 48000 * 300, 48000 * 41, 48000 * 700]
    with na.Decoder(48000, na.Settings(), max_samples=x.size) as dec:
        rows_before = dec.decode(x[: lens[2]])
        dec.set_process_mode(image.MINMAX, rgba=True, palette=palette)
        imgs = [dec.decode(x[:n]) for n in lens]
        dec.set_png_mode(block_bytes=32768)
        pngs = [dec.decode(x[:n]) for n in lens]
        for img, png in zip(imgs, pngs):
            assert isinstance(png, bytes) and png == image.encode_png(img, block_bytes=32768)
        dec.set_png_mode(False)
        assert np.array_equal(dec.decode(x[: lens[1]]), imgs[1])
        dec.set_png_mode()
        assert dec.decode(x[: lens[3]]) == image.encode_png(imgs[3])
        dec.set_process_mode(None)
        assert np.array_equal(dec.decode(x[: lens[2]]), rows_before)
        with pytest.raises(na.err.InvalidInput):
            dec.set_png_mode()              # PNG mode needs image or process mode
    with na.Decoder(48000, na.Settings(), max_samples=x.size) as d2:
        d2.set_process_mode(image.MINMAX, rgba=True, palette=palette)
        d2.set_png_mode(block_bytes=32768)
        assert d2.decode(x[: lens[1]]) == pngs[1]


def test_decoder_png_mode_capacity():
    x = synth.apt_signal(48000, 60, seed=3)
    with na.Decoder(48000, na.Settings(), max_samples=x.size) as dec:
        dec.set_process_mode(image.MINMAX)
        dec.set_png_mode()
        out = np.empty(100, dtype=np.uint8)
        dec.submit(x, True, out=out)
        with pytest.raises(na.err.InvalidInput) as e:
            dec.wait()
        assert e.value.code == na._lib.ERR_CAPACITY
        png = dec.decode(x)                  # the decoder is usable afterwards
        assert _pixels(png).shape[1] == 2080


def test_decode_wav_png_writes_decode_png_bytes(tmp_path, palette):
    pcm = synth.apt_pcm16(11025, seconds=120, seed=8)
    wav = tmp_path / "in.wav"
    na.wav.write_wav_i16(str(wav), pcm, 11025)
    out = tmp_path / "out.png"
    kw = dict(contrast=image.TELEMETRY, rotate=True, palette=palette, rgba=True)
    info = image.decode_wav_png(wav, out, **kw)
    png, info2 = image.decode_png(na.Context(), na.Settings(), pcm, 11025, True, **kw)
    assert out.read_bytes() == png
    assert info["rows"] == info2["rows"] > 0


def test_kept_workspace_across_sizes_and_cache_clear(excerpt):
    """apt_png_encode keeps its device workspace between calls: a smaller image after a larger one (stale buffers), a
    different channel count, and an encode after apt_cache_clear freed it all give the restatement's bytes."""
    big = _rgba(excerpt)
    small = excerpt[:9, :301]
    assert image.encode_png(big, block_bytes=4096) == po.encode(big, block_bytes=4096)
    _same(image.encode_png(small, block_bytes=4096), po.encode(small, block_bytes=4096))
    na._lib.load().apt_cache_clear()
    _same(image.encode_png(small[:, :, None].repeat(3, 2)), po.encode(small[:, :, None].repeat(3, 2)))
