"""Pins the CPU restatement of the rest of noaa_apt::process (tests/_process_oracle.py) on hand-checkable cases, and the
argument rules of apt_process / apt_decode_image, which the library checks before it looks for a device."""
import ctypes as C
import os

import numpy as np
import pytest

import __graft_entry__ as entry
import _process_oracle as po

rng = np.random.default_rng(2024)


@pytest.fixture(scope="module")
def na():
    entry.build()
    import noaa_apt_b200
    return noaa_apt_b200


def test_rotation_is_an_involution_and_keeps_the_other_columns():
    grey = rng.integers(0, 256, (37, 2080), dtype=np.uint8)
    once = po.rotate(grey)
    assert np.array_equal(po.rotate(once), grey)
    outside = np.ones(2080, bool)
    outside[86:995] = outside[1126:2035] = False
    assert np.array_equal(once[:, outside], grey[:, outside])            # sync, space and telemetry columns stay
    # (x0 + i, y) <-> (x0 + 908 - i, rows - 1 - y)
    for x0 in (86, 1126):
        for i, y in ((0, 0), (908, 36), (5, 17), (454, 18)):
            assert once[y, x0 + i] == grey[36 - y, x0 + 908 - i]
    rgba = np.stack([grey, grey // 2, grey // 3, np.full_like(grey, 255)], axis=-1)
    assert np.array_equal(po.rotate(po.rotate(rgba)), rgba)
    assert np.array_equal(po.rotate(rgba)[..., 1], po.rotate(grey // 2))


def _expected_lut(counts):
    """The reference's formula written out with numpy float32 scalars from a known histogram."""
    cum = np.cumsum(np.asarray(counts, dtype=np.int64))
    total = np.float32(int(cum[-1]))
    out = []
    for c in cum:
        v = np.float32(255.0) * (np.float32(int(c)) / total)
        out.append(int(v))
    return np.array(out, dtype=np.uint8)


def test_equalisation_of_a_known_histogram():
    # channel A: values 0, 100, 200, 255 in counts 1 : 2 : 3 : 4 of the half; channel B constant 7
    rows = 10
    a = np.repeat(np.array([0, 100, 200, 255], np.uint8), [104, 208, 312, 416])
    grey = np.empty((rows, 2080), np.uint8)
    grey[:, :1040] = a
    grey[:, 1040:] = 7
    eq = po.equalize(grey)
    counts = np.zeros(256, np.int64)
    counts[[0, 100, 200, 255]] = np.array([104, 208, 312, 416]) * rows
    lut = _expected_lut(counts)
    assert lut[0] == 25 and lut[100] == 76 and lut[200] == 153 and lut[255] == 255       # 255 * 0.1 / 0.3 / 0.6 / 1
    assert np.array_equal(eq[:, :1040], lut[grey[:, :1040]])
    assert (eq[:, 1040:] == 255).all()                                                  # one value: cumulative = total


def test_equalisation_rounds_counts_above_2_24_pixels():
    # 16 200 rows: 16 848 000 pixels per half, more than 2^24, so `hist[v] as f32` and `total as f32` round
    rows = 16200
    n = rows * 1040
    assert n > 1 << 24
    counts = np.zeros(256, np.int64)
    counts[3] = 5_000_001
    counts[10] = n - 1 - counts[3]           # cumulative n - 1 = 16 847 999: odd above 2^24, `as f32` gives 16 848 000
    counts[200] = 1
    half = np.repeat(np.arange(256, dtype=np.uint8), counts).reshape(rows, 1040)
    grey = np.concatenate([half, half[::-1]], axis=1)
    lut = po.equalize_lut(half)
    assert np.array_equal(lut, _expected_lut(counts))
    # the f32 conversion is visible: exact arithmetic gives 254 for value 10, the reference's f32 arithmetic 255
    cum = np.cumsum(counts)
    assert (255 * int(cum[10])) // int(cum[-1]) == 254 and lut[10] == 255
    assert lut[3] == 75 and lut[200] == 255
    eq = po.equalize(grey)
    assert np.array_equal(eq[:, :1040], lut[half]) and np.array_equal(eq[:, 1040:], lut[half[::-1]])


def test_identity_palette_returns_the_grey_of_both_channels():
    # P[b][a] = (a, b, 0): with zero tunes the colour region holds (grey A, grey B, 0, 255)
    pal = np.zeros((256, 256, 3), np.uint8)
    pal[..., 0] = np.arange(256)[None, :]
    pal[..., 1] = np.arange(256)[:, None]
    grey = rng.integers(0, 256, (23, 2080), dtype=np.uint8)
    img = po.process_grey(grey, po.MINMAX, palette=pal)
    assert img.shape == (23, 2080, 4)
    assert np.array_equal(img[:, 86:995, 0], grey[:, 86:995])
    assert np.array_equal(img[:, 86:995, 1], grey[:, 1126:2035])
    assert (img[:, 86:995, 2] == 0).all() and (img[..., 3] == 255).all()
    rest = np.ones(2080, bool)
    rest[86:995] = False
    for ch in range(3):
        assert np.array_equal(img[:, rest, ch], grey[:, rest])                       # R = G = B = grey elsewhere
    # rotation after false colour moves the coloured pixels with the rectangle
    rot = po.process_grey(grey, po.MINMAX, rotate_=True, palette=pal)
    assert np.array_equal(rot, po.rotate(img))


def test_tunes_follow_the_f32_formula_and_clamp():
    v = np.arange(256, dtype=np.uint8)
    assert np.array_equal(po.tune_values(v, 0.0, 0.0), v.astype(np.uint32))
    # start 0.5, end 0.2: s = 0.15, e = 0.06 (f32), out = v * ((1 + e) - s) - s * 255
    s, e = np.float32(0.5) * np.float32(0.3), np.float32(0.2) * np.float32(0.3)
    k = (np.float32(1) + e) - s
    want = [min(max(np.float32(x) * k - s * np.float32(255), np.float32(0)), np.float32(255)) for x in range(256)]
    assert np.array_equal(po.tune_values(v, 0.5, 0.2), np.array([int(w) for w in want], np.uint32))
    got = po.tune_values(v, 0.5, 0.2)
    assert got[0] == 0 and got[42] == 0 and got[255] == int(np.float32(255) * k - s * np.float32(255))   # 193
    assert got[255] == 193
    # negative start raises the floor; a large end saturates at 255
    assert po.tune_values(v, -1.0, 0.0)[0] == 76 and po.tune_values(v, 0.0, 5.0)[200] == 255
    assert po.tune_values(v, float("nan"), 0.0).max() == 0                        # NaN `as u32` is 0


def test_colour_histogram_and_grey_palette_are_refused_by_the_oracle():
    pal = np.zeros((256, 256, 3), np.uint8)
    grey = np.zeros((4, 2080), np.uint8)
    with pytest.raises(ValueError, match="colour histogram"):
        po.process_grey(grey, po.HISTOGRAM, palette=pal)
    with pytest.raises(ValueError):
        po.process_grey(grey, po.MINMAX, palette=pal, rgba=False)


def test_argument_errors_without_a_device(na):
    from noaa_apt_b200 import image
    lib = na._lib.load()
    rows = np.zeros(2080 * 4, np.float32)
    out = np.zeros(rows.size * 4, np.uint8)
    n = C.c_uint64(0)
    pal = np.zeros((256, 256, 3), np.uint8)

    def call(**kw):
        ps, _, _keep = image.process_settings(**kw)
        return lib.apt_process(rows.ctypes.data, rows.size, C.byref(ps), out.ctypes.data, out.size, C.byref(n), None)

    assert call(contrast=image.HISTOGRAM, palette=pal) == na._lib.ERR_BAD_ARG
    assert b"colour histogram equalisation is not available" in lib.apt_last_error()
    assert call(contrast=image.MINMAX, palette=pal, rgba=False) == na._lib.ERR_BAD_ARG
    assert call(contrast=4) == na._lib.ERR_BAD_ARG and b"unknown contrast" in lib.apt_last_error()
    assert call(contrast=-1) == na._lib.ERR_BAD_ARG
    assert call(contrast=image.PERCENT, percent=1.5) == na._lib.ERR_BAD_ARG
    assert lib.apt_process(rows.ctypes.data, rows.size, None, out.ctypes.data, out.size, C.byref(n), None) == na._lib.ERR_BAD_ARG
    # decode + process: the same rules, before the recording is even looked at
    s = na.Settings().to_c()
    ps, _, _keep = image.process_settings(image.HISTOGRAM, palette=pal)
    x = np.zeros(100000, np.float32)
    assert lib.apt_decode_image(x.ctypes.data, na._lib.F32, x.size, 11025, C.byref(s), 1, C.byref(ps), out.ctypes.data,
                                out.size, C.byref(n), None, na._lib.STATUS_CB(0), None) == na._lib.ERR_BAD_ARG
    with pytest.raises(na.err.InvalidInput, match="colour histogram"):
        image.decode_image(na.Context(), na.Settings(), x, 11025, contrast=image.HISTOGRAM, palette=pal)
    with pytest.raises(na.err.InvalidInput):
        image.process(rows, image.MINMAX, palette=np.zeros((255, 256, 3), np.uint8))
    # the existing image-mode entry point keeps refusing Contrast::Histogram
    assert lib.apt_decode_image_u8(x.ctypes.data, na._lib.F32, x.size, 11025, C.byref(s), 1, image.HISTOGRAM, 0.98,
                                   out.ctypes.data, out.size, C.byref(n), None, na._lib.STATUS_CB(0), None) == na._lib.ERR_BAD_ARG
    # a short output buffer reports the RGBA size; valid arguments then need a device
    ps, _, _keep = image.process_settings(image.MINMAX, rgba=True)
    assert lib.apt_process(rows.ctypes.data, rows.size, C.byref(ps), out.ctypes.data, rows.size, C.byref(n), None) == na._lib.ERR_CAPACITY
    assert str(rows.size * 4).encode() in lib.apt_last_error()
    if na.device_count() == 0:
        assert lib.apt_process(rows.ctypes.data, rows.size, C.byref(ps), out.ctypes.data, out.size, C.byref(n), None) == na._lib.ERR_CUDA


def test_load_palette_drops_alpha_and_checks_the_size(tmp_path, na):
    from PIL import Image
    from noaa_apt_b200 import image
    px = rng.integers(0, 256, (256, 256, 4), dtype=np.uint8)
    Image.fromarray(px, "RGBA").save(tmp_path / "p.png")
    assert np.array_equal(image.load_palette(str(tmp_path / "p.png")), px[..., :3])
    Image.fromarray(px[:128], "RGBA").save(tmp_path / "small.png")
    with pytest.raises(na.err.InvalidInput):
        image.load_palette(str(tmp_path / "small.png"))
    fx = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "palettes.npz"))
    assert set(fx.files) == {"noaa-apt-daylight", "WXtoImg-NO"}
    assert all(fx[k].shape == (256, 256, 3) and fx[k].dtype == np.uint8 for k in fx.files)
