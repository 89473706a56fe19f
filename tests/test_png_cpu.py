"""The PNG definition of DESIGN.md §11 on the CPU: the restatement in tests/_png_oracle.py writes files that Pillow and
zlib read back exactly, its filter choice, code lengths, checksums and bound hold on their own terms, its sizes clear the
bars DESIGN.md §11 sets, and every PNG entry point rejects bad arguments before it needs a device."""
import ctypes as C
import io
import os
import zlib

import numpy as np
import pytest
from PIL import Image

import __graft_entry__ as entry
import _png_oracle as po

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def na():
    entry.build()
    import noaa_apt_b200
    return noaa_apt_b200


@pytest.fixture(scope="module")
def excerpt():
    return np.load(os.path.join(GOLDEN, "argentina_excerpt.npz"))["grey"]


def _rgba(grey):
    out = np.empty(grey.shape + (4,), dtype=np.uint8)
    out[..., :3] = grey[..., None]
    out[..., 3] = 255
    return out


def _chunks(png):
    assert png[:8] == po.PNG_SIGNATURE
    k, out = 8, []
    while k < len(png):
        n = int.from_bytes(png[k:k + 4], "big")
        kind, data, crc = png[k + 4:k + 8], png[k + 8:k + 8 + n], int.from_bytes(png[k + 8 + n:k + 12 + n], "big")
        out.append((kind, data, crc))
        k += 12 + n
    return out


def _check_file(png, img, rgb_from_rgba=False):
    with Image.open(io.BytesIO(png)) as im:
        back = np.asarray(im)
    want = img[..., :3] if rgb_from_rgba else img
    assert np.array_equal(back.reshape(want.shape), want)
    ch = _chunks(png)
    assert [c[0] for c in ch] == [b"IHDR", b"IDAT", b"IEND"]
    for kind, data, crc in ch:
        assert zlib.crc32(kind + data) == crc
    return ch


@pytest.mark.parametrize("ch", [1, 3, 4])
@pytest.mark.parametrize("w", [1, 7, 2080])
def test_files_read_back_exactly(ch, w):
    rng = np.random.default_rng(w + ch)
    h = {1: 900, 7: 200, 2080: 12}[w]
    base = (np.add.outer(np.arange(h) * 3, np.arange(w * ch)) % 251).astype(np.uint8)
    img = np.where(rng.random(base.shape) < 0.2, rng.integers(0, 256, base.shape), base).astype(np.uint8)
    img = img.reshape(h, w, ch) if ch > 1 else img
    if ch == 4:
        img[..., 3] = 255
    for bb in (4096, 8192, 16384, 32768, 65536):
        for filt in (-1, 0, 1, 2, 3, 4):
            for matches in (0, 1):
                if filt not in (-1, 4) and (matches == 0 or bb not in (4096, 65536)):
                    continue
                info = {}
                png = po.encode(img, filt, matches, bb, info=info)
                _check_file(png, img)
                f = info["F"]
                z = _chunks(png)[1][1]
                assert zlib.decompress(z) == f.tobytes()
                assert int.from_bytes(z[-4:], "big") == zlib.adler32(f.tobytes()) == po.adler32(f)
                assert len(png) <= po.bound(w, h, ch, bb)
    if ch == 4:
        png = po.encode(img, rgb_from_rgba=1)
        _check_file(png, img, rgb_from_rgba=True)


def test_crc_restatement_matches_zlib():
    rng = np.random.default_rng(1)
    for n in (0, 1, 5, 1000):
        data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        assert po.crc32(data) == zlib.crc32(data)
    img = rng.integers(0, 256, (20, 13, 3), dtype=np.uint8)
    assert po.encode(img, crc=po.crc32) == po.encode(img)


def test_filter_choice_is_the_minimum_absolute_sum(excerpt):
    img = _rgba(excerpt[:150]).reshape(150, -1)
    types = po.filter_types(img, 4)
    x = img.astype(np.int64)
    a = np.zeros_like(x)
    a[:, 4:] = x[:, :-4]
    b = np.zeros_like(x)
    b[1:] = x[:-1]
    c = np.zeros_like(x)
    c[1:, 4:] = x[:-1, :-4]
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    pae = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
    scores = []
    for pred in (0, a, b, (a + b) // 2, pae):
        r = (x - pred) % 256
        scores.append(np.minimum(r, 256 - r).sum(axis=1))
    scores = np.stack(scores)
    assert np.array_equal(types, np.argmin(scores, axis=0))
    assert set(np.unique(types)) > {0}


def test_package_merge_limits_and_completeness():
    fib = [1, 1]
    while len(fib) < 30:
        fib.append(fib[-1] + fib[-2])
    lit = po.package_merge(fib + [0] * 256, 15)
    assert max(lit) == 15 and po.kraft_ok(lit, 15)
    assert po.package_merge(fib[:19], 7) and po.kraft_ok(po.package_merge(fib[:19], 7), 7)
    assert po.package_merge([0] * 30, 15)[:2] == [1, 1]
    one = po.package_merge([0] * 5 + [9] + [0] * 24, 15)
    assert one[0] == one[5] == 1 and sum(one) == 2
    zero = po.package_merge([4] + [0] * 29, 15)
    assert zero[0] == zero[1] == 1 and sum(zero) == 2
    # unlimited optimum where the limit does not bind: Huffman cost
    rng = np.random.default_rng(3)
    f = rng.integers(1, 50, 40).tolist()
    L = po.package_merge(f, 15)
    import heapq
    h = list(f)
    heapq.heapify(h)
    cost = 0
    while len(h) > 1:
        s = heapq.heappop(h) + heapq.heappop(h)
        cost += s
        heapq.heappush(h, s)
    assert sum(a * b for a, b in zip(f, L)) == cost


@pytest.mark.parametrize("kind", ["constant", "no_matches", "random"])
def test_trees_on_skewed_images(kind):
    rng = np.random.default_rng(7)
    if kind == "constant":
        img = np.full((40, 500), 9, np.uint8)
    elif kind == "no_matches":
        img = np.arange(256, dtype=np.uint8)[None, :].repeat(3, 0)
    else:
        img = rng.integers(0, 256, (60, 700), dtype=np.uint8)
    for bb in (4096, 65536):
        info = {}
        png = po.encode(img, -1, 1, bb, info=info)
        _check_file(png, img)
        for ll, dl, cl in info["trees"]:
            assert po.kraft_ok(ll, 15) and po.kraft_ok(dl, 15) and po.kraft_ok(cl, 7)
        assert len(png) <= po.bound(img.shape[1], img.shape[0], 1, bb)


def _zlib6(f):
    return len(zlib.compress(f.tobytes(), 6))


def test_size_bars_on_the_excerpt(excerpt, capsys):
    grey = excerpt
    png = po.encode(grey)
    f, _ = po.filtered_stream(grey, 1)
    idat = len(_chunks(png)[1][1])
    assert idat <= 1.00 * _zlib6(f)
    rgba = _rgba(grey)
    png4 = po.encode(rgba)
    f4, _ = po.filtered_stream(rgba, 4)
    idat4 = len(_chunks(png4)[1][1])
    b = io.BytesIO()
    Image.fromarray(rgba).save(b, format="PNG")
    assert idat4 <= 1.30 * _zlib6(f4)
    assert len(png4) <= 0.85 * len(b.getvalue())
    with capsys.disabled():
        print(f"\nexcerpt {grey.shape}: grey {idat / _zlib6(f):.3f} x zlib-6, {idat / grey.size:.3f} of raw; "
              f"RGBA {idat4 / _zlib6(f4):.3f} x zlib-6, {len(png4) / len(b.getvalue()):.3f} x Pillow")


def test_false_colour_size(excerpt, capsys):
    import _process_oracle as pro
    pal = np.load(os.path.join(GOLDEN, "palettes.npz"))["noaa-apt-daylight"]
    img = pro.process_grey(excerpt, pro.MINMAX, False, pal, (0, 0, 0, 0), True)
    png = po.encode(img)
    f, _ = po.filtered_stream(img, 4)
    idat = len(_chunks(png)[1][1])
    with capsys.disabled():
        print(f"\nfalse colour RGBA: {idat / _zlib6(f):.3f} x zlib-6, {len(png) / img.size:.3f} of raw")
    assert idat <= 1.30 * _zlib6(f)


def test_bound_matches_the_library(na):
    lib = na._lib.load()
    for w, h, ch, bb in ((1, 1, 1, 4096), (2080, 1800, 4, 65536), (7, 300, 3, 8192), (2080, 72000, 4, 65536)):
        assert na.image.png_bound(w, h, ch, block_bytes=bb) == po.bound(w, h, ch, bb)
    ps = na._lib.CPngSettings()
    lib.apt_png_default_settings(C.byref(ps))
    assert (ps.filter, ps.matches, ps.block_bytes, ps.rgb_from_rgba) == (-1, 1, 65536, 0)
    assert na.image.png_bound(2080, 1800, 4, rgb_from_rgba=True) == po.bound(2080, 1800, 4, rgb_from_rgba=1)


def test_argument_errors_without_a_device(na, tmp_path):
    lib = na._lib.load()
    img = np.zeros((4, 5), np.uint8)
    bad = na.err.InvalidInput
    for kw in (dict(filter=5), dict(filter=-2), dict(block_bytes=2048), dict(block_bytes=65536 * 2), dict(block_bytes=5000)):
        with pytest.raises(bad):
            na.image.encode_png(img, **kw)
        with pytest.raises(bad):
            na.image.png_bound(5, 4, 1, **kw)
    with pytest.raises(bad):
        na.image.encode_png(np.zeros((4, 5, 2), np.uint8))
    with pytest.raises(bad):
        na.image.encode_png(np.zeros((0, 5), np.uint8))
    with pytest.raises(bad):
        na.image.encode_png(np.zeros((4, 5, 3), np.uint8), rgb_from_rgba=True)        # not RGBA
    rgba = np.full((4, 5, 4), 255, np.uint8)
    rgba[2, 3, 3] = 254
    with pytest.raises(bad):
        na.image.encode_png(rgba, rgb_from_rgba=True)                                   # alpha != 255
    ps = na.image.png_settings()
    n = C.c_uint64(0)
    out = np.empty(100, np.uint8)
    assert lib.apt_png_encode(None, 5, 4, 1, C.byref(ps), out.ctypes.data, 100, C.byref(n)) == na._lib.ERR_BAD_ARG
    assert lib.apt_png_encode(img.ctypes.data, 5, 4, 1, None, out.ctypes.data, 100, C.byref(n)) == na._lib.ERR_BAD_ARG
    assert lib.apt_png_encode(img.ctypes.data, 5, 4, 1, C.byref(ps), None, 100, C.byref(n)) == na._lib.ERR_BAD_ARG
    assert lib.apt_png_encode(img.ctypes.data, 5, 4, 2, C.byref(ps), out.ctypes.data, 100, C.byref(n)) == na._lib.ERR_BAD_ARG
    assert lib.apt_png_bound(5, 4, 1, C.byref(ps), None) == na._lib.ERR_BAD_ARG
    assert lib.apt_png_bound(1 << 20, 1 << 14, 4, C.byref(ps), C.byref(n)) == na._lib.ERR_BAD_ARG   # IDAT over 2^31 - 1
    # decode_png: process rules, then PNG rules, before any device
    x = np.zeros(48000 * 10, np.float32)
    with pytest.raises(bad):
        na.image.decode_png(None, None, x, 48000, filter=7)
    with pytest.raises(bad):
        na.image.decode_png(None, None, x, 48000, rgb_from_rgba=True)                   # grey output
    with pytest.raises(bad):
        na.image.decode_png(None, None, x, 48000, contrast=9)
    s = na.Settings().to_c()
    pps, _, _ = na.image.process_settings(na.image.MINMAX)
    assert lib.apt_decode_png(x.ctypes.data, 0, x.size, 48000, C.byref(s), 1, C.byref(pps), None, out.ctypes.data, 100,
                              C.byref(n), None, na._lib.STATUS_CB(0), None) == na._lib.ERR_BAD_ARG
    assert lib.apt_decode_png(x.ctypes.data, 0, x.size, 48000, C.byref(s), 1, None, C.byref(ps), out.ctypes.data, 100,
                              C.byref(n), None, na._lib.STATUS_CB(0), None) == na._lib.ERR_BAD_ARG
    assert lib.apt_decode_png(x.ctypes.data, 0, x.size, 48000, C.byref(s), 1, C.byref(pps), C.byref(ps), None, 100,
                              C.byref(n), None, na._lib.STATUS_CB(0), None) == na._lib.ERR_BAD_ARG
    assert lib.apt_decoder_set_png_mode(None, C.byref(ps)) == na._lib.ERR_BAD_ARG
    with pytest.raises(bad):
        na.image.decode_wav_png(tmp_path / "in.wav", tmp_path / "out.png", block_bytes=3)
    assert lib.apt_decode_wav_png(None, b"x.png", C.byref(s), 1, C.byref(pps), C.byref(ps), None) == na._lib.ERR_BAD_ARG
    with pytest.raises(na.err.Io):
        na.image.decode_wav_png(tmp_path / "missing.wav", tmp_path / "out.png")
