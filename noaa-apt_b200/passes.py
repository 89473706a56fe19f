"""Finding the satellite passes in a long recording (DESIGN.md §12) and decoding each one from a single upload.

    with Recording(pcm, 96000) as rec:              # the samples cross PCIe once and stay on the device
        q = rec.quality()                           # q[w]: correlation of image row w with row w + 1 of the envelope
        found = rec.find_passes()                   # [Pass(start, end, first_window, windows, mean_quality, peak_quality)]
        pngs, infos, statuses = rec.decode_png(found, contrast=image.TELEMETRY)

    for p, png, info in decode_passes_png(pcm, 96000):   # the same in one call
        ...

A pass is a run of windows with q >= exit (gaps shorter than max_gap_s joined) that reaches q >= enter somewhere and
lasts at least min_length_s.  Each decoded pass equals apt_decode / decode_image / decode_png of the host slice
signal[p.start:p.end] with the same arguments, bit for bit.
"""
import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import _lib, image
from .config import Settings
from .decode import PX_PER_ROW, _fmt_of, decode_len_bound
from .err import raise_for
from .frequency import _rate_hz

ENTER, EXIT, MAX_GAP_S, MIN_LENGTH_S = 0.30, 0.15, 30.0, 60.0


@dataclass
class Pass:
    """apt_pass: input samples [start, end) and windows [first_window, first_window + windows)."""
    start: int
    end: int
    first_window: int = 0
    windows: int = 0
    mean_quality: float = 0.0
    peak_quality: float = 0.0

    @classmethod
    def from_c(cls, c):
        return cls(int(c.start), int(c.end), int(c.first_window), int(c.windows), float(c.mean_quality),
                   float(c.peak_quality))


def _search(enter=ENTER, exit=EXIT, max_gap_s=MAX_GAP_S, min_length_s=MIN_LENGTH_S):
    return _lib.CPassSearch(float(enter), float(exit), float(max_gap_s), float(min_length_s))


def _ranges(passes):
    ps = [p if isinstance(p, Pass) else Pass(int(p[0]), int(p[1])) for p in passes]
    arr = (_lib.CPass * max(len(ps), 1))()
    for i, p in enumerate(ps):
        arr[i].start, arr[i].end = p.start, p.end
    return ps, arr


def find_passes_quality(q, n, input_rate, enter=ENTER, exit=EXIT, max_gap_s=MAX_GAP_S, min_length_s=MIN_LENGTH_S,
                        max_passes=1024):
    """The pass rule on a quality array (host only): the passes of a recording of n samples at input_rate."""
    x = np.ascontiguousarray(q, dtype=np.float32)
    ps = _search(enter, exit, max_gap_s, min_length_s)
    out = (_lib.CPass * max(int(max_passes), 1))()
    count = C.c_uint32(0)
    raise_for(_lib.load().apt_find_passes_quality(x.ctypes.data if x.size else None, x.size, int(n), _rate_hz(input_rate),
                                                  C.byref(ps), out, len(out), C.byref(count)))
    return [Pass.from_c(out[i]) for i in range(count.value)]


class Recording:
    """apt_recording: a recording (float32 Signal or int16 PCM) uploaded once and kept in device memory."""

    def __init__(self, signal, input_rate, settings=None, device=0):
        self._lib = _lib.load()
        x = np.ascontiguousarray(signal)
        self.format = _fmt_of(x)
        self.settings = settings or Settings()
        self.input_rate = _rate_hz(input_rate)
        self.n = x.size
        s = self.settings.to_c()
        h = C.c_void_p(None)
        raise_for(self._lib.apt_recording_create(int(device), x.ctypes.data if x.size else None, self.format, x.size,
                                                 self.input_rate, C.byref(s), C.byref(h)))
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            self._lib.apt_recording_destroy(self._h)
            self._h = None

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def info(self):
        ci = _lib.CRecordingInfo()
        raise_for(self._lib.apt_recording_get_info(self._h, C.byref(ci)))
        return {n: int(getattr(ci, n)) for n, _ in _lib.CRecordingInfo._fields_}

    @property
    def device_bytes(self):
        return self.info()["device_bytes"]

    def quality(self):
        """q, one float32 per window of the envelope (W = floor(N_w / R) - 1 of them)."""
        nq = C.c_uint64(0)
        raise_for(self._lib.apt_recording_quality(self._h, None, 0, C.byref(nq)))
        q = np.empty(nq.value, dtype=np.float32)
        if nq.value:
            raise_for(self._lib.apt_recording_quality(self._h, q.ctypes.data, q.size, C.byref(nq)))
        return q

    def find_passes(self, enter=ENTER, exit=EXIT, max_gap_s=MAX_GAP_S, min_length_s=MIN_LENGTH_S, max_passes=1024):
        return find_passes_quality(self.quality(), self.n, self.input_rate, enter, exit, max_gap_s, min_length_s, max_passes)

    def _decode(self, passes, sync, ps, bpp, png):
        ranges, arr = _ranges(passes)
        k = len(ranges)
        if k == 0:
            return [], [], []
        caps_list = []
        for p in ranges:
            bound = decode_len_bound(max(p.end - p.start, 0), self.input_rate, self.settings)
            if png is not None:
                caps_list.append(image.png_bound(PX_PER_ROW, max(bound // PX_PER_ROW, 1), bpp, png.filter, bool(png.matches),
                                                 png.block_bytes, bool(png.rgb_from_rgba)))
            else:
                caps_list.append(bound * (bpp or 1))
        dt = np.uint8 if bpp else np.float32
        outs = [np.empty(max(c, 1), dtype=dt) for c in caps_list]
        nouts = (C.c_uint64 * k)()
        infos = (_lib.CImageInfo * k)()
        sts = (C.c_int * k)(*([-1] * k))
        rc = self._lib.apt_recording_decode(self._h, arr, k, int(bool(sync)), C.byref(ps) if ps is not None else None,
                                            C.byref(png) if png is not None else None,
                                            (C.c_void_p * k)(*[o.ctypes.data for o in outs]),
                                            (C.c_uint64 * k)(*[o.size for o in outs]), nouts, infos, sts)
        if rc != _lib.OK and all(int(v) in (rc, -1) for v in sts) and rc in (_lib.ERR_BAD_ARG, _lib.ERR_CUDA, _lib.ERR_NOMEM):
            raise_for(rc)   # nothing was decoded: an error, not a result
        res, inf = [], []
        for i in range(k):
            if sts[i] != _lib.OK:
                res.append(None)
                inf.append(None)
                continue
            got = outs[i][: nouts[i]]
            if png is not None:
                res.append(got.tobytes())
            elif bpp:
                res.append(image._shape(got.copy(), bpp))
            else:
                res.append(got.copy())
            inf.append(image._info(infos[i]) if bpp else None)
        return res, inf, [int(v) for v in sts]

    def decode(self, passes, sync=True):
        """The f32 rows of each pass, as decode() of the host slice: (rows or None per pass, statuses)."""
        rows, _inf, sts = self._decode(passes, sync, None, None, None)
        return rows, sts

    def decode_image(self, passes, sync=True, contrast=image.MINMAX, percent=0.98, rotate=False, palette=None,
                     tune=(0, 0, 0, 0), rgba=None):
        """The processed image of each pass, as image.decode_image of the host slice: (images, infos, statuses)."""
        ps, bpp, _pal = image.process_settings(contrast, percent, rotate, palette, tune, rgba)
        return self._decode(passes, sync, ps, bpp, None)

    def decode_png(self, passes, sync=True, contrast=image.MINMAX, percent=0.98, rotate=False, palette=None,
                   tune=(0, 0, 0, 0), rgba=None, filter=-1, matches=True, block_bytes=65536, rgb_from_rgba=False):
        """The PNG file of each pass, as image.decode_png of the host slice: (bytes, infos, statuses)."""
        ps, bpp, _pal = image.process_settings(contrast, percent, rotate, palette, tune, rgba)
        png = image.png_settings(filter, matches, block_bytes, rgb_from_rgba)
        return self._decode(passes, sync, ps, bpp, png)


def decode_passes_png(signal, input_rate, settings=None, sync=True, device=0, search=None, **process):
    """Find the passes of a recording and decode each one to a PNG file, the samples uploaded once:
    [(Pass, png bytes or None, info or None)].  search: keyword arguments of find_passes; process: those of decode_png."""
    with Recording(signal, input_rate, settings, device) as rec:
        found = rec.find_passes(**(search or {}))
        pngs, infos, _sts = rec.decode_png(found, sync, **process)
    return list(zip(found, pngs, infos))
