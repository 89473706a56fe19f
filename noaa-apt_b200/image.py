"""noaa_apt::process (noaa_apt.rs:132-240) on the device, the map overlay excepted: contrast bounds (MinMax /
misc::percent / telemetry wedges), map_signal_u8, false colour, grey histogram equalisation and rotation -- the decoded
rows become the finished image before they leave the GPU."""
import ctypes as C

import numpy as np

from . import _lib
from .config import Settings
from .err import InvalidInput, raise_for
from .frequency import _rate_hz

MINMAX, PERCENT, TELEMETRY, HISTOGRAM = (_lib.CONTRAST_MINMAX, _lib.CONTRAST_PERCENT, _lib.CONTRAST_TELEMETRY,
                                         _lib.CONTRAST_HISTOGRAM)


def load_palette(path):
    """A false-colour palette image as (256, 256, 3) u8 RGB: the image crate's into_rgb8 drops alpha, and any size but
    256x256 is InvalidInput (processing.rs:110-116)."""
    from PIL import Image
    with Image.open(path) as im:
        rgb = np.asarray(im.convert("RGB"), dtype=np.uint8)
    if rgb.shape != (256, 256, 3):
        raise InvalidInput(_lib.ERR_BAD_ARG, "Invalid palette image dimensions")
    return np.ascontiguousarray(rgb)


def process_settings(contrast, percent=0.98, rotate=False, palette=None, tune=(0, 0, 0, 0), rgba=None):
    """(apt_process_settings, bytes per pixel, palette array to keep alive).  rgba=None: RGBA with a palette, else grey."""
    pal = None
    if palette is not None:
        pal = np.ascontiguousarray(palette, dtype=np.uint8)
        if pal.shape != (256, 256, 3):
            raise InvalidInput(_lib.ERR_BAD_ARG, "Invalid palette image dimensions")
    if rgba is None:
        rgba = pal is not None
    ps = _lib.CProcessSettings()
    ps.contrast = int(contrast)
    ps.percent = float(percent)
    ps.rotate = int(bool(rotate))
    ps.palette = pal.ctypes.data if pal is not None else None
    ps.tune = (C.c_float * 4)(*[float(t) for t in tune])
    ps.rgba = int(bool(rgba))
    return ps, (4 if rgba else 1), pal


def _shape(flat, bpp):
    return flat.reshape(-1, 2080, 4) if bpp == 4 else flat.reshape(-1, 2080)


def process(rows, contrast, percent=0.98, rotate=False, palette=None, tune=(0, 0, 0, 0), rgba=None):
    """The image process() returns for decode()'s rows (noaa_apt.rs:140-240 without the map): (rows, 2080) u8 grey or
    (rows, 2080, 4) u8 RGBA, plus the contrast info."""
    x = np.ascontiguousarray(rows, dtype=np.float32).ravel()
    ps, bpp, _pal = process_settings(contrast, percent, rotate, palette, tune, rgba)
    out = np.empty(max(x.size * bpp, 1), dtype=np.uint8)
    n = C.c_uint64(0)
    ci = _lib.CImageInfo()
    raise_for(_lib.load().apt_process(x.ctypes.data, x.size, C.byref(ps), out.ctypes.data, out.size, C.byref(n), C.byref(ci)))
    return _shape(out[: n.value], bpp), _info(ci)


def decode_image(context, settings, signal, input_rate, sync=True, contrast=MINMAX, percent=0.98, rotate=False,
                 palette=None, tune=(0, 0, 0, 0), rgba=None):
    """decode() + process() in one call -> (image of shape (rows, 2080) or (rows, 2080, 4), info)."""
    lib = _lib.load()
    x = np.ascontiguousarray(signal)
    fmt = _lib.PCM16 if x.dtype == np.int16 else _lib.F32
    if fmt == _lib.F32:
        x = np.ascontiguousarray(x, dtype=np.float32)
    ps, bpp, _pal = process_settings(contrast, percent, rotate, palette, tune, rgba)
    s = (settings or Settings()).to_c()
    rate = _rate_hz(input_rate)
    bound = C.c_uint64(0)
    raise_for(lib.apt_decode_len_bound(x.size, rate, C.byref(s), C.byref(bound)))
    out = np.empty(max(bound.value * bpp, 1), dtype=np.uint8)
    n = C.c_uint64(0)
    ci = _lib.CImageInfo()

    def _cb(progress, desc, _user):
        if context is not None:
            context.status(progress, desc.decode())

    cb = _lib.STATUS_CB(_cb)
    raise_for(lib.apt_decode_image(x.ctypes.data, fmt, x.size, rate, C.byref(s), int(bool(sync)), C.byref(ps),
                                   out.ctypes.data, out.size, C.byref(n), C.byref(ci), cb, None))
    return _shape(out[: n.value].copy(), bpp), _info(ci)


def png_settings(filter=-1, matches=True, block_bytes=65536, rgb_from_rgba=False):
    """apt_png_settings (DESIGN.md §11): filter -1 adaptive or 0..4 fixed; matches False gives Huffman-only deflate;
    block_bytes a power of two in [4096, 65536]; rgb_from_rgba writes RGBA pixels (alpha all 255) as RGB."""
    ps = _lib.CPngSettings()
    ps.filter = int(filter)
    ps.matches = int(bool(matches))
    ps.block_bytes = int(block_bytes)
    ps.rgb_from_rgba = int(bool(rgb_from_rgba))
    return ps


def _channels(shape):
    if len(shape) == 2:
        return 1
    if len(shape) == 3 and shape[2] in (1, 3, 4):
        return shape[2]
    raise InvalidInput(_lib.ERR_BAD_ARG, f"pixels must be (h, w) or (h, w, 1 / 3 / 4), got {shape}")


def png_bound(width, height, channels, filter=-1, matches=True, block_bytes=65536, rgb_from_rgba=False):
    """Upper bound of encode_png's output size in bytes (host arithmetic, no device)."""
    ps = png_settings(filter, matches, block_bytes, rgb_from_rgba)
    b = C.c_uint64(0)
    raise_for(_lib.load().apt_png_bound(int(width), int(height), int(channels), C.byref(ps), C.byref(b)))
    return b.value


def output_bytes(pixels, bpp, png=None):
    """Bytes the image of `pixels` decoded pixels leaves as: pixels * bpp, or with png (png_settings) the PNG bound of
    max(pixels // 2080, 1) rows (host arithmetic, no device)."""
    if png is None:
        return pixels * bpp
    b = C.c_uint64(0)
    raise_for(_lib.load().apt_png_bound(2080, max(pixels // 2080, 1), int(bpp), C.byref(png), C.byref(b)))
    return b.value


def encode_png(pixels, filter=-1, matches=True, block_bytes=65536, rgb_from_rgba=False):
    """PNG file bytes of u8 pixels (h, w) grey, (h, w, 3) RGB or (h, w, 4) RGBA, encoded on the device."""
    x = np.ascontiguousarray(pixels, dtype=np.uint8)
    ch = _channels(x.shape)
    if x.ndim != 2 and x.ndim != 3:
        raise InvalidInput(_lib.ERR_BAD_ARG, "pixels must be 2-D or 3-D")
    h, w = x.shape[0], x.shape[1]
    ps = png_settings(filter, matches, block_bytes, rgb_from_rgba)
    lib = _lib.load()
    b = C.c_uint64(0)
    raise_for(lib.apt_png_bound(w, h, ch, C.byref(ps), C.byref(b)))
    out = np.empty(max(b.value, 1), dtype=np.uint8)
    n = C.c_uint64(0)
    raise_for(lib.apt_png_encode(x.ctypes.data, w, h, ch, C.byref(ps), out.ctypes.data, out.size, C.byref(n)))
    return out[: n.value].tobytes()


def encode_png_batch(images, filter=-1, matches=True, block_bytes=65536, rgb_from_rgba=False):
    """encode_png of several images of one width and channel count (heights may differ) in one batched encode on the
    device -> list of PNG bytes, each equal to encode_png of that image alone."""
    xs = [np.ascontiguousarray(x, dtype=np.uint8) for x in images]
    if not xs:
        return []
    ch = _channels(xs[0].shape)
    w = xs[0].shape[1]
    if any(x.ndim != xs[0].ndim or _channels(x.shape) != ch or x.shape[1] != w for x in xs):
        raise InvalidInput(_lib.ERR_BAD_ARG, "the images of a batch must share width and channels")
    ps = png_settings(filter, matches, block_bytes, rgb_from_rgba)
    lib = _lib.load()
    n = len(xs)
    outs = [np.empty(max(png_bound(w, x.shape[0], ch, filter, matches, block_bytes, rgb_from_rgba), 1), dtype=np.uint8)
            for x in xs]
    nouts = (C.c_uint64 * n)()
    raise_for(lib.apt_png_encode_batch((C.c_void_p * n)(*[x.ctypes.data for x in xs]), (C.c_uint32 * n)(*[x.shape[0] for x in xs]),
                                       n, w, ch, C.byref(ps), (C.c_void_p * n)(*[o.ctypes.data for o in outs]),
                                       (C.c_uint64 * n)(*[o.size for o in outs]), nouts))
    return [o[: nouts[k]].tobytes() for k, o in enumerate(outs)]


def decode_png(context, settings, signal, input_rate, sync=True, contrast=MINMAX, percent=0.98, rotate=False, palette=None,
               tune=(0, 0, 0, 0), rgba=None, filter=-1, matches=True, block_bytes=65536, rgb_from_rgba=False):
    """decode() + process() + PNG encoding in one call; only the PNG bytes leave the GPU -> (bytes, info)."""
    lib = _lib.load()
    x = np.ascontiguousarray(signal)
    fmt = _lib.PCM16 if x.dtype == np.int16 else _lib.F32
    if fmt == _lib.F32:
        x = np.ascontiguousarray(x, dtype=np.float32)
    ps, bpp, _pal = process_settings(contrast, percent, rotate, palette, tune, rgba)
    png = png_settings(filter, matches, block_bytes, rgb_from_rgba)
    s = (settings or Settings()).to_c()
    rate = _rate_hz(input_rate)
    bound = C.c_uint64(0)
    raise_for(lib.apt_decode_len_bound(x.size, rate, C.byref(s), C.byref(bound)))
    out = np.empty(output_bytes(bound.value, bpp, png), dtype=np.uint8)
    n = C.c_uint64(0)
    ci = _lib.CImageInfo()

    def _cb(progress, desc, _user):
        if context is not None:
            context.status(progress, desc.decode())

    cb = _lib.STATUS_CB(_cb)
    raise_for(lib.apt_decode_png(x.ctypes.data, fmt, x.size, rate, C.byref(s), int(bool(sync)), C.byref(ps), C.byref(png),
                                 out.ctypes.data, out.size, C.byref(n), C.byref(ci), cb, None))
    return out[: n.value].tobytes(), _info(ci)


def decode_batch_png(signals, input_rate, settings=None, sync=True, contrast=MINMAX, percent=0.98, rotate=False,
                     palette=None, tune=(0, 0, 0, 0), rgba=None, png=True, filter=-1, matches=True, block_bytes=65536,
                     rgb_from_rgba=False, devices=None, streams_per_device=4):
    """decode_batch ending each recording in its PNG file (png=True) or its processed image (png=False), sharded as
    decode_batch.  With PNG output the images of each device are encoded in groups, one launch sequence per group.
    Returns (list of bytes or pixel arrays or None, list of infos or None, list of status codes); raises when nothing
    decoded at all."""
    from .decode import _fmt_of, decode_len_bound
    lib = _lib.load()
    s = (settings or Settings()).to_c()
    rate = _rate_hz(input_rate)
    xs = [np.ascontiguousarray(x) for x in signals]
    if not xs:
        return [], [], []
    fmt = _fmt_of(xs[0])
    if any(_fmt_of(x) != fmt for x in xs):
        raise TypeError("all recordings of a batch must share one sample format")
    ps, bpp, _pal = process_settings(contrast, percent, rotate, palette, tune, rgba)
    pngs = png_settings(filter, matches, block_bytes, rgb_from_rgba) if png else None
    count = len(xs)
    caps_list = [output_bytes(decode_len_bound(x.size, rate, settings), bpp, pngs) for x in xs]
    outs = [np.empty(max(c, 1), dtype=np.uint8) for c in caps_list]
    sig_ptrs = (C.c_void_p * count)(*[x.ctypes.data for x in xs])
    out_ptrs = (C.c_void_p * count)(*[o.ctypes.data for o in outs])
    lens = (C.c_uint64 * count)(*[x.size for x in xs])
    caps = (C.c_uint64 * count)(*[o.size for o in outs])
    nouts = (C.c_uint64 * count)()
    infos = (_lib.CImageInfo * count)()
    statuses = (C.c_int * count)(*([-1] * count))   # -1: not written (never "ok" unless the library says so)
    devs = list(devices) if devices else [0]
    dev_arr = (C.c_int * len(devs))(*devs)
    rc = lib.apt_decode_batch_image(sig_ptrs, fmt, lens, count, rate,
                                    C.byref(s), int(bool(sync)), C.byref(ps), C.byref(pngs) if pngs is not None else None,
                                    out_ptrs, caps, nouts, infos, statuses, dev_arr, len(devs), int(streams_per_device))
    if rc != _lib.OK and all(int(v) in (rc, -1) for v in statuses):
        raise_for(rc)   # nothing decoded at all (argument errors, no device, ...): an error, not a result
    res, inf = [], []
    for i in range(count):
        if statuses[i] != _lib.OK:
            res.append(None)
            inf.append(None)
            continue
        got = outs[i][: nouts[i]]
        res.append(got.tobytes() if png else _shape(got.copy(), bpp))
        inf.append(_info(infos[i]))
    return res, inf, [int(v) for v in statuses]


def png_group_plan(width, channels, heights, filter=-1, matches=True, block_bytes=65536, rgb_from_rgba=False):
    """The layout of one batched PNG encode of images of these heights (host arithmetic, no device) ->
    (dict of the shared buffer and grid sizes, list of dicts of each image's regions)."""
    ps = png_settings(filter, matches, block_bytes, rgb_from_rgba)
    hs = (C.c_uint32 * max(len(heights), 1))(*[int(h) for h in heights])
    gi = _lib.CPngGroupInfo()
    ims = (_lib.CPngGroupImage * max(len(heights), 1))()
    raise_for(_lib.load().apt_png_group_plan(int(width), int(channels), C.byref(ps), hs, len(heights), C.byref(gi), ims,
                                             len(heights)))
    info = {n: int(getattr(gi, n)) for n, _ in _lib.CPngGroupInfo._fields_}
    return info, [{n: int(getattr(im, n)) for n, _ in _lib.CPngGroupImage._fields_ if n != "pad"} for im in ims[: len(heights)]]


def decode_wav_png(input_path, output_path, settings=None, sync=True, contrast=MINMAX, percent=0.98, rotate=False,
                   palette=None, tune=(0, 0, 0, 0), rgba=None, filter=-1, matches=True, block_bytes=65536,
                   rgb_from_rgba=False):
    """The reference CLI's job: WAV file in, PNG file out (decode, process and encode on the device) -> info."""
    ps, _bpp, _pal = process_settings(contrast, percent, rotate, palette, tune, rgba)
    png = png_settings(filter, matches, block_bytes, rgb_from_rgba)
    s = (settings or Settings()).to_c()
    ci = _lib.CImageInfo()
    raise_for(_lib.load().apt_decode_wav_png(str(input_path).encode(), str(output_path).encode(), C.byref(s),
                                             int(bool(sync)), C.byref(ps), C.byref(png), C.byref(ci)))
    return _info(ci)


def _info(ci):
    return {"low": ci.low, "high": ci.high, "rows": int(ci.rows), "telemetry_row": int(ci.telemetry_row),
            "wedges_a": np.array(ci.wedges_a[:], dtype=np.float32), "wedges_b": np.array(ci.wedges_b[:], dtype=np.float32)}


def map_signal_u8(signal, low, high):
    """noaa_apt.rs:249-259"""
    x = np.ascontiguousarray(signal, dtype=np.float32)
    out = np.empty(x.size, dtype=np.uint8)
    raise_for(_lib.load().apt_map_signal_u8(x.ctypes.data, x.size, low, high, out.ctypes.data))
    return out


def contrast_bounds(signal, contrast, percent=0.98):
    """(low, high, info): MinMax (dsp.rs:20-54), misc::percent (misc.rs:119-175) or telemetry wedges 9 / 8."""
    x = np.ascontiguousarray(signal, dtype=np.float32)
    ci = _lib.CImageInfo()
    raise_for(_lib.load().apt_contrast_bounds(x.ctypes.data, x.size, int(contrast), float(percent), C.byref(ci)))
    info = _info(ci)
    return info["low"], info["high"], info


def telemetry_rows(signal):
    """telemetry.rs:147-170 -> (mean_a, mean_b, variance) per image row"""
    x = np.ascontiguousarray(signal, dtype=np.float32)
    rows = x.size // 2080
    a, b, v = (np.empty(rows, dtype=np.float32) for _ in range(3))
    raise_for(_lib.load().apt_telemetry_rows(x.ctypes.data, x.size, a.ctypes.data, b.ctypes.data, v.ctypes.data))
    return a, b, v


def decode_image_u8(context, settings, signal, input_rate, sync=True, contrast=MINMAX, percent=0.98):
    """decode() + contrast + map_signal_u8 in one call -> (u8 image of shape (rows, 2080), info)."""
    lib = _lib.load()
    x = np.ascontiguousarray(signal)
    fmt = _lib.PCM16 if x.dtype == np.int16 else _lib.F32
    if fmt == _lib.F32:
        x = np.ascontiguousarray(x, dtype=np.float32)
    s = (settings or Settings()).to_c()
    rate = _rate_hz(input_rate)
    bound = C.c_uint64(0)
    raise_for(lib.apt_decode_len_bound(x.size, rate, C.byref(s), C.byref(bound)))
    out = np.empty(max(bound.value, 1), dtype=np.uint8)
    n = C.c_uint64(0)
    ci = _lib.CImageInfo()

    def _cb(progress, desc, _user):
        if context is not None:
            context.status(progress, desc.decode())

    cb = _lib.STATUS_CB(_cb)
    raise_for(lib.apt_decode_image_u8(x.ctypes.data, fmt, x.size, rate, C.byref(s), int(bool(sync)), int(contrast),
                                      float(percent), out.ctypes.data, out.size, C.byref(n), C.byref(ci), cb, None))
    return out[: n.value].reshape(-1, 2080).copy(), _info(ci)
