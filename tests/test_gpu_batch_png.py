"""apt_decode_batch_image on the device: every recording of a batch ends in exactly the PNG file apt_decode_png gives for
it alone (or, without PNG, exactly apt_decode_image's pixels), with the same info and status, whatever the grouping of
the batched encode; failures and a short output buffer stay with their recording; the group's files also equal the CPU
restatement of DESIGN.md §11."""
import ctypes as C
import os

import numpy as np
import pytest

import noaa_apt_b200 as na
from noaa_apt_b200 import image, synth
import _png_oracle as po

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# mixed lengths, so groups of mixed heights; three passes long enough for the telemetry wedges (a frame and more)
SECONDS = [10, 35, 120, 17, 60, 12, 150, 25, 45, 11, 135, 30]


@pytest.fixture(scope="module")
def palette():
    return np.load(os.path.join(GOLDEN, "palettes.npz"))["noaa-apt-daylight"]


_recs = {}


def recordings(rate):
    if rate not in _recs:
        _recs[rate] = [synth.apt_pcm16(rate, s, seed=300 + k) for k, s in enumerate(SECONDS)]
    return _recs[rate]


def modes(palette):
    return {
        "grey_minmax": (dict(contrast=image.MINMAX), True),
        "grey_histogram": (dict(contrast=image.HISTOGRAM), True),
        "rgba_telemetry_rotate": (dict(contrast=image.TELEMETRY, rotate=True, palette=palette, rgba=True), True),
        "nosync": (dict(contrast=image.MINMAX), False),
    }


def _signals(rate, fmt):
    pcm = recordings(rate)
    return [p.astype(np.float32) for p in pcm] if fmt == "f32" else pcm


def _one_shot(fn, sig, rate, sync, **kw):
    """(result, info, status) of a one-shot call; an image-stage failure (telemetry on a pass shorter than a frame) is a
    status like any other."""
    try:
        got, info = fn(na.Context(), na.Settings(), sig, rate, sync, **kw)
        return got, info, 0
    except na.err.Error as e:
        return None, None, e.code


def _same_bytes(got, ref, what):
    assert got is not None, what
    assert len(got) == len(ref), (what, len(got), len(ref))
    assert got == ref, f"{what}: bytes differ"


def _same_info(got, ref, what):
    assert got is not None, what
    for k in ("low", "high", "rows", "telemetry_row"):
        assert got[k] == ref[k], (what, k, got[k], ref[k])
    for k in ("wedges_a", "wedges_b"):
        assert np.array_equal(got[k], ref[k]), (what, k)


@pytest.mark.parametrize("rate", [48000, 11025])
@pytest.mark.parametrize("fmt", ["f32", "pcm16"])
@pytest.mark.parametrize("mode", ["grey_minmax", "grey_histogram", "rgba_telemetry_rotate", "nosync"])
def test_batch_equals_one_shot(palette, rate, fmt, mode):
    kw, sync = modes(palette)[mode]
    sigs = _signals(rate, fmt)
    files, infos, statuses = image.decode_batch_png(sigs, rate, sync=sync, png=True, streams_per_device=4, **kw)
    ok = 0
    for i, sig in enumerate(sigs):
        ref, ref_info, ref_st = _one_shot(image.decode_png, sig, rate, sync, **kw)
        assert statuses[i] == ref_st, (i, statuses[i], ref_st)
        if ref_st:
            assert files[i] is None and infos[i] is None
            continue
        ok += 1
        _same_bytes(files[i], ref, f"PNG of recording {i}")
        _same_info(infos[i], ref_info, f"info of recording {i}")
    assert ok >= 3
    pixels, infos, statuses = image.decode_batch_png(sigs, rate, sync=sync, png=False, streams_per_device=4, **kw)
    for i, sig in enumerate(sigs):
        ref, ref_info, ref_st = _one_shot(image.decode_image, sig, rate, sync, **kw)
        assert statuses[i] == ref_st, (i, statuses[i], ref_st)
        if ref_st:
            assert pixels[i] is None and infos[i] is None
            continue
        assert pixels[i].shape == ref.shape and np.array_equal(pixels[i], ref), f"pixels of recording {i}"
        _same_info(infos[i], ref_info, f"info of recording {i}")


@pytest.mark.parametrize("mode", ["grey_minmax", "rgba_telemetry_rotate"])
def test_grouping_does_not_change_the_bytes(palette, mode):
    kw, sync = modes(palette)[mode]
    sigs = _signals(48000, "pcm16")
    base, _, st0 = image.decode_batch_png(sigs, 48000, sync=sync, streams_per_device=4, **kw)
    assert st0.count(0) >= 3
    for spd in (1, 3, 8):
        got, _, st = image.decode_batch_png(sigs, 48000, sync=sync, streams_per_device=spd, **kw)
        assert st == st0
        for i in range(len(sigs)):
            if st0[i] == 0:
                _same_bytes(got[i], base[i], f"streams_per_device={spd}, recording {i}")
    rev, _, st = image.decode_batch_png(sigs[::-1], 48000, sync=sync, streams_per_device=3, **kw)
    assert st[::-1] == st0
    for i in range(len(sigs)):
        if st0[i] == 0:
            _same_bytes(rev[len(sigs) - 1 - i], base[i], f"reversed order, recording {i}")


def test_failures_in_the_middle_of_a_batch(palette):
    kw = dict(contrast=image.MINMAX, rotate=True, palette=palette, rgba=True)
    sigs = list(_signals(48000, "f32")[:8])
    sigs[2] = np.zeros(20000, np.float32)                                                      # too short
    sigs[5] = (np.random.default_rng(5).standard_normal(48000 * 30) * 3000).astype(np.float32)   # pure noise
    sigs[6] = synth.apt_signal(48000, 5.3, seed=9)                           # just over 10 rows: few sync frames, if any
    want = [_one_shot(image.decode_png, x, 48000, True, **kw) for x in sigs]
    assert want[2][2] == na._lib.ERR_TOO_SHORT
    for png in (True, False):
        files, infos, statuses = image.decode_batch_png(sigs, 48000, png=png, streams_per_device=3, **kw)
        assert statuses == [w[2] for w in want]
        for i, (ref, ref_info, ref_st) in enumerate(want):
            if ref_st:
                assert files[i] is None and infos[i] is None
            elif png:
                _same_bytes(files[i], ref, f"recording {i}")
                _same_info(infos[i], ref_info, f"recording {i}")


def test_one_output_one_byte_short():
    lib = na._lib.load()
    sigs = _signals(48000, "f32")[:6]
    refs = [image.decode_png(na.Context(), na.Settings(), x, 48000, True)[0] for x in sigs]
    short = 3
    count = len(sigs)
    outs = [np.zeros(len(r) + 64, np.uint8) for r in refs]
    caps = (C.c_uint64 * count)(*[len(r) - 1 if i == short else len(r) for i, r in enumerate(refs)])
    sig_ptrs = (C.c_void_p * count)(*[x.ctypes.data for x in sigs])
    out_ptrs = (C.c_void_p * count)(*[o.ctypes.data for o in outs])
    lens = (C.c_uint64 * count)(*[x.size for x in sigs])
    nouts = (C.c_uint64 * count)()
    infos = (na._lib.CImageInfo * count)()
    statuses = (C.c_int * count)()
    ps, _, _ = image.process_settings(image.MINMAX)
    png = image.png_settings()
    s = na.Settings().to_c()
    rc = lib.apt_decode_batch_image(sig_ptrs, na._lib.F32, lens, count, 48000, C.byref(s), 1, C.byref(ps), C.byref(png),
                                    out_ptrs, caps, nouts, infos, statuses, None, 0, 2)
    assert rc == na._lib.ERR_CAPACITY
    assert statuses[short] == na._lib.ERR_CAPACITY and nouts[short] == len(refs[short])
    for i in range(count):
        if i != short:
            assert statuses[i] == 0 and nouts[i] == len(refs[i])
            assert outs[i][: nouts[i]].tobytes() == refs[i]


@pytest.mark.parametrize("rgba", [False, True])
def test_group_files_equal_the_cpu_restatement(palette, rgba):
    """Short recordings and 4 KiB blocks, several blocks per image, checked against tests/_png_oracle.py directly.  How
    the feeder groups them depends on timing; test_encode_batch_groups fixes the groups."""
    kw = dict(contrast=image.MINMAX, palette=palette if rgba else None, rgba=rgba)
    sigs = [synth.apt_pcm16(48000, s, seed=500 + s) for s in (10, 13, 11, 14)]
    files, _, statuses = image.decode_batch_png(sigs, 48000, block_bytes=4096, streams_per_device=2, **kw)
    assert statuses == [0] * len(sigs)
    for i, sig in enumerate(sigs):
        px, _ = image.decode_image(na.Context(), na.Settings(), sig, 48000, True, **kw)
        _same_bytes(files[i], po.encode(px, -1, 1, 4096), f"recording {i}")


def _group_images(kind):
    """Images of one width and mixed heights: one row, a few rows, and several 4 KiB blocks; the excerpt of a real pass
    with rows of noise, so that matches, literals and every filter type occur and reach across rows."""
    grey = np.load(os.path.join(GOLDEN, "argentina_excerpt.npz"))["grey"][:, :700]
    rng = np.random.default_rng(11)
    out = []
    for k, h in enumerate((1, 3, 40, 7, 97, 2, 23)):
        g = np.ascontiguousarray(grey[9 * k: 9 * k + h])
        g[::5] = rng.integers(0, 256, g[::5].shape, dtype=np.uint8)
        if kind == "grey":
            out.append(g)
            continue
        rgba = np.empty(g.shape + (4,), dtype=np.uint8)
        rgba[..., 0], rgba[..., 1], rgba[..., 2] = g, g[::-1], np.roll(g, 3, axis=1)
        rgba[..., 3] = 255 if kind == "rgb_from_rgba" else (g >> 1) | 0x80
        out.append(rgba)
    return out


@pytest.mark.parametrize("kind", ["grey", "rgba", "rgb_from_rgba"])
def test_encode_batch_groups(kind):
    """apt_png_encode_batch: one group of seven images of mixed heights; every file equals the CPU restatement and
    apt_png_encode of that image alone, whatever group it is encoded in."""
    imgs = _group_images(kind)
    rgb = kind == "rgb_from_rgba"
    files = image.encode_png_batch(imgs, block_bytes=4096, rgb_from_rgba=rgb)
    assert len(files) == len(imgs)
    for k, img in enumerate(imgs):
        ref = po.encode(img, -1, 1, 4096, rgb_from_rgba=int(rgb))
        _same_bytes(files[k], ref, f"image {k} against the restatement")
        _same_bytes(image.encode_png(img, block_bytes=4096, rgb_from_rgba=rgb), ref, f"image {k} alone")
    # the same images in other groups: reversed, and a sub-group
    rev = image.encode_png_batch(imgs[::-1], block_bytes=4096, rgb_from_rgba=rgb)
    for k in range(len(imgs)):
        _same_bytes(rev[len(imgs) - 1 - k], files[k], f"image {k}, reversed group")
    sub = image.encode_png_batch(imgs[2:5], block_bytes=4096, rgb_from_rgba=rgb)
    for k in range(3):
        _same_bytes(sub[k], files[2 + k], f"image {2 + k}, sub-group")


def test_encode_batch_one_cap_one_byte_short():
    imgs = _group_images("rgba")
    refs = image.encode_png_batch(imgs)
    n, short = len(imgs), 2
    outs = [np.zeros(len(r) + 64, np.uint8) for r in refs]
    caps = (C.c_uint64 * n)(*[len(r) - 1 if k == short else len(r) for k, r in enumerate(refs)])
    nouts = (C.c_uint64 * n)()
    ps = image.png_settings()
    rc = na._lib.load().apt_png_encode_batch((C.c_void_p * n)(*[x.ctypes.data for x in imgs]),
                                             (C.c_uint32 * n)(*[x.shape[0] for x in imgs]), n, imgs[0].shape[1], 4,
                                             C.byref(ps), (C.c_void_p * n)(*[o.ctypes.data for o in outs]), caps, nouts)
    assert rc == na._lib.ERR_CAPACITY
    assert nouts[short] == len(refs[short]) and not outs[short].any()
    for k in range(n):
        if k != short:
            assert nouts[k] == len(refs[k]) and outs[k][: nouts[k]].tobytes() == refs[k], k


def test_batch_on_all_devices(palette):
    g = na.device_count()
    if g < 2:
        pytest.skip("needs more than one GPU")
    kw = dict(contrast=image.TELEMETRY, rotate=True, palette=palette, rgba=True)
    sigs = _signals(48000, "pcm16")
    one, _, st1 = image.decode_batch_png(sigs, 48000, streams_per_device=3, **kw)
    many, _, st = image.decode_batch_png(sigs, 48000, devices=list(range(g)), streams_per_device=3, **kw)
    assert st1 == st and st.count(0) >= 3
    for i in range(len(sigs)):
        if st[i] == 0:
            _same_bytes(many[i], one[i], f"recording {i}")
