"""apt_decode_batch_image and the batched PNG encoder's layout without a device: every argument rule comes back as
APT_ERR_BAD_ARG before a device is touched, count == 0 is a success, the Python wrapper checks its own arguments, and
the host layout of a group (apt_png_group_plan) gives each image disjoint regions, blocks of its own and the right
bounds."""
import ctypes as C

import numpy as np
import pytest

import __graft_entry__ as entry


@pytest.fixture(scope="module")
def na():
    entry.build()
    import noaa_apt_b200
    return noaa_apt_b200


def _call(na, signals=True, lens=True, count=2, rate=48000, s=True, sync=1, ps=True, png=True, outs=True, caps=True,
          nouts=True, infos=True, statuses=True, fmt=None, ps_fields=None, png_fields=None, settings=None, out_null=None):
    L = na._lib
    lib = L.load()
    x = np.zeros(48000 * 12, dtype=np.float32)
    bufs = [np.empty(1 << 16, dtype=np.uint8) for _ in range(max(count, 1))]
    sig = (C.c_void_p * max(count, 1))(*([x.ctypes.data] * max(count, 1)))
    ln = (C.c_uint64 * max(count, 1))(*([x.size] * max(count, 1)))
    optr = (C.c_void_p * max(count, 1))(*[b.ctypes.data for b in bufs])
    if out_null is not None:
        optr[out_null] = None
    cp = (C.c_uint64 * max(count, 1))(*([1 << 16] * max(count, 1)))
    no = (C.c_uint64 * max(count, 1))()
    inf = (L.CImageInfo * max(count, 1))()
    st = (C.c_int * max(count, 1))()
    cs = (settings or na.Settings()).to_c()
    pss, _bpp, _pal = na.image.process_settings(na.image.MINMAX)
    for k, v in (ps_fields or {}).items():
        setattr(pss, k, v)
    pngs = na.image.png_settings()
    for k, v in (png_fields or {}).items():
        setattr(pngs, k, v)
    rc = lib.apt_decode_batch_image(sig if signals else None, L.F32 if fmt is None else fmt, ln if lens else None, count, rate,
                                    C.byref(cs) if s else None, sync, C.byref(pss) if ps else None,
                                    C.byref(pngs) if png else None, optr if outs else None, cp if caps else None,
                                    no if nouts else None, inf if infos else None, st if statuses else None, None, 0, 1)
    return rc


def test_argument_errors_are_bad_arg_without_a_device(na):
    BAD = na._lib.ERR_BAD_ARG
    assert _call(na, signals=False) == BAD
    assert _call(na, lens=False) == BAD
    assert _call(na, s=False) == BAD
    assert _call(na, ps=False) == BAD
    assert _call(na, outs=False) == BAD
    assert _call(na, caps=False) == BAD
    assert _call(na, nouts=False) == BAD
    assert _call(na, count=-1) == BAD
    assert _call(na, out_null=1) == BAD
    assert _call(na, fmt=7) == BAD
    # apt_process's settings rules
    assert _call(na, ps_fields={"contrast": 9}) == BAD
    assert _call(na, ps_fields={"contrast": na.image.PERCENT, "percent": 1.5}) == BAD
    pal = np.zeros((256, 256, 3), np.uint8)
    assert _call(na, ps_fields={"palette": pal.ctypes.data, "rgba": 0}) == BAD        # false colour needs RGBA output
    assert _call(na, ps_fields={"palette": pal.ctypes.data, "rgba": 1,               # colour histogram (Lab) is not offered
                                "contrast": na.image.HISTOGRAM}) == BAD
    # apt_png_encode's settings rules, and rgb_from_rgba on grey output
    assert _call(na, png_fields={"filter": 5}) == BAD
    assert _call(na, png_fields={"filter": -2}) == BAD
    assert _call(na, png_fields={"block_bytes": 3000}) == BAD
    assert _call(na, png_fields={"block_bytes": 1 << 17}) == BAD
    assert _call(na, png_fields={"rgb_from_rgba": 1}) == BAD
    # infos and statuses may be NULL: the rules above do not depend on them
    assert _call(na, infos=False, statuses=False, png_fields={"filter": 5}) == BAD


def test_count_zero_is_ok_without_a_device(na):
    assert _call(na, count=0) == na._lib.OK
    assert _call(na, count=0, png=False) == na._lib.OK


def test_python_wrapper_arguments(na):
    from noaa_apt_b200 import image
    from noaa_apt_b200.err import InvalidInput
    assert image.decode_batch_png([], 48000) == ([], [], [])
    x = np.zeros(48000 * 12, dtype=np.float32)
    with pytest.raises(TypeError):
        image.decode_batch_png([x, x.astype(np.int16)], 48000)
    with pytest.raises(TypeError):
        image.decode_batch_png([x.astype(np.float64)], 48000)
    with pytest.raises(InvalidInput):
        image.decode_batch_png([x], 48000, palette=np.zeros((10, 10, 3), np.uint8))
    with pytest.raises(Exception) as e:
        image.decode_batch_png([x], 48000, block_bytes=1000)
    assert not isinstance(e.value, TypeError)
    with pytest.raises(Exception):
        image.decode_batch_png([x], 48000, rgb_from_rgba=True)   # grey output


def test_python_wrapper_raises_what_the_library_rejects(na):
    """Rules the library checks before it writes any status are raised, not returned as a list of failures."""
    from noaa_apt_b200 import image
    from noaa_apt_b200.err import InvalidInput, Internal
    x = np.zeros(48000 * 12, dtype=np.float32)
    with pytest.raises(InvalidInput):
        image.decode_batch_png([x, x], 48000, contrast=image.PERCENT, percent=1.5)
    with pytest.raises(InvalidInput):
        image.decode_batch_png([x, x], 48000, png=False, contrast=image.PERCENT, percent=1.5)
    odd = na.Settings(work_rate=10000)                       # not a multiple of 4160: no rows of 2080 pixels
    with pytest.raises(InvalidInput):
        image.decode_batch_png([x, x], 48000, settings=odd, sync=False)
    with pytest.raises(Internal) as e:
        image.decode_batch_png([x, x], 48000, settings=odd, sync=True)
    assert e.value.code == na._lib.ERR_WORK_RATE


@pytest.mark.parametrize("channels,block_bytes,rgb", [(1, 65536, False), (4, 65536, False), (4, 4096, True), (3, 16384, False)])
def test_group_layout_mixed_heights(na, channels, block_bytes, rgb):
    from noaa_apt_b200 import image
    heights = [1800, 11, 1, 960, 1801, 37, 2400, 5]
    width = 2080
    info, ims = image.png_group_plan(width, channels, heights, block_bytes=block_bytes, rgb_from_rgba=rgb)
    ch = 3 if rgb else channels
    assert len(ims) == len(heights)
    rows = spans = blocks = chunks = 0
    stream_end = out_end = 0
    for h, im in zip(heights, ims):
        n = h * (1 + width * ch)
        assert im["stream_bytes"] == n
        assert im["bound"] == image.png_bound(width, h, channels, block_bytes=block_bytes, rgb_from_rgba=rgb)
        # regions in order, aligned and disjoint: the stream plus its 16 bytes of padding, the file's bound
        assert im["stream_offset"] % 64 == 0 and im["stream_offset"] >= stream_end
        stream_end = im["stream_offset"] + n + 16
        assert im["out_offset"] % 8 == 0 and im["out_offset"] >= out_end
        assert im["out_bytes"] >= im["bound"] and im["out_bytes"] % 4 == 0
        out_end = im["out_offset"] + im["out_bytes"]
        # every block of an image lies inside it: its blocks cover exactly its stream
        assert im["blocks"] == -(-n // block_bytes)
        assert im["first_block"] == blocks and im["first_row"] == rows and im["first_span"] == spans
        assert im["first_chunk"] == chunks and im["first_chunk"] % 32 == 0
        rows += h
        spans += -(-n // 32736)
        blocks += im["blocks"]
        chunks += -(-(-(-(im["bound"] - 37) // 1024)) // 32) * 32
    assert info["rows"] == rows == sum(heights)
    assert info["spans"] == spans and info["blocks"] == blocks and info["chunks"] == chunks
    assert info["stream_bytes"] >= stream_end
    assert info["out_bytes"] >= out_end
    # the output buffer is the prefix sum of the per-image bounds (rounded to words, then to 8 bytes)
    assert info["out_bytes"] == sum(-(-im["out_bytes"] // 8) * 8 for im in ims)
    assert info["out_bytes"] >= sum(im["bound"] for im in ims)


def test_group_layout_of_one_is_the_single_image(na):
    from noaa_apt_b200 import image
    info, ims = image.png_group_plan(2080, 1, [1800])
    assert ims[0]["stream_offset"] == 0 and ims[0]["out_offset"] == 0
    assert ims[0]["bound"] == image.png_bound(2080, 1800, 1)
    assert info["blocks"] == ims[0]["blocks"] == -(-1800 * 2081 // 65536)


def test_group_layout_argument_errors(na):
    from noaa_apt_b200 import image
    from noaa_apt_b200.err import InvalidInput
    with pytest.raises(InvalidInput):
        image.png_group_plan(2080, 1, [])
    with pytest.raises(InvalidInput):
        image.png_group_plan(2080, 1, [10, 0, 5])
    with pytest.raises(InvalidInput):
        image.png_group_plan(2080, 2, [10])
    with pytest.raises(InvalidInput):
        image.png_group_plan(2080, 1, [10], rgb_from_rgba=True)
