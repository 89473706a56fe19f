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
from .iq import _offsets, iq_format
from .config import Settings
from .decode import _fmt_of, decode_len_bound
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
            caps_list.append(image.output_bytes(bound, bpp, png) if bpp else bound)
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


@dataclass
class PassEvent:
    """apt_pass_event: kind "aos", "los" or "segment", the window whose evaluation fired it, and the pass.  From a Watch,
    also the pass number, and for an LOS the decode's status, row count, image info and data (f32 rows, pixels or PNG
    bytes; None when the decode failed)."""
    kind: str
    window: int
    pass_: Pass
    index: int = 0
    status: int = 0
    rows: int = 0
    info: dict = None
    data: object = None


_KINDS = {_lib.PASS_AOS: "aos", _lib.PASS_LOS: "los", _lib.PASS_SEGMENT: "segment"}


def _event(ce):
    return PassEvent(_KINDS[int(ce.kind)], int(ce.window), Pass.from_c(ce.pass_))


class PassTracker:
    """apt_pass_tracker: the pass rule fed q window by window (host only).  feed(q) and finish(n) return the events."""

    def __init__(self, input_rate, enter=ENTER, exit=EXIT, max_gap_s=MAX_GAP_S, min_length_s=MIN_LENGTH_S):
        self._lib = _lib.load()
        ps = _search(enter, exit, max_gap_s, min_length_s)
        h = C.c_void_p(None)
        raise_for(self._lib.apt_pass_tracker_create(_rate_hz(input_rate), C.byref(ps), C.byref(h)))
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            self._lib.apt_pass_tracker_destroy(self._h)
            self._h = None

    __del__ = close

    def feed(self, q):
        x = np.ascontiguousarray(q, dtype=np.float32)
        evs = (_lib.CPassEvent * max(2 * x.size, 1))()
        n = C.c_uint64(0)
        raise_for(self._lib.apt_pass_tracker_feed(self._h, x.ctypes.data if x.size else None, x.size, evs, 2 * x.size,
                                                  C.byref(n)))
        return [_event(evs[i]) for i in range(n.value)]

    def finish(self, n):
        evs = (_lib.CPassEvent * 1)()
        k = C.c_uint64(0)
        raise_for(self._lib.apt_pass_tracker_finish(self._h, int(n), evs, 1, C.byref(k)))
        return [_event(evs[i]) for i in range(k.value)]


def watch_settings(sync=True, search=None, ps=None, png=None, max_rows=0, max_push=0):
    """apt_watch_settings; search: keyword arguments of find_passes_quality's rule (enter, exit, max_gap_s, min_length_s)."""
    ws = _lib.CWatchSettings()
    ws.sync = int(bool(sync))
    ws.search = _search(**(search or {}))
    ws.ps = C.addressof(ps) if ps is not None else None
    ws.png = C.addressof(png) if png is not None else None
    ws.max_rows, ws.max_push = int(max_rows), int(max_push)
    return ws


def _image_args(image_out, process):
    """(apt_process_settings or None, bytes per pixel or None, apt_png_settings or None) for image_out None / "image" / "png"."""
    if image_out is None:
        return None, None, None
    png_kw = {k: process.pop(k) for k in ("filter", "matches", "block_bytes", "rgb_from_rgba") if k in process}
    process.setdefault("contrast", image.MINMAX)
    ps, bpp, pal = image.process_settings(**process)
    png = image.png_settings(**png_kw) if image_out == "png" else None
    return (ps, pal), bpp, png


def _watch_event(e, bpp, png):
    """A PassEvent copied out of an apt_watch_event (during the callback: its data is valid only then)."""
    ev = _event(e.ev)
    ev.index, ev.status, ev.rows = int(e.index), int(e.status), int(e.rows)
    if ev.kind == "los":
        if bpp:
            ev.info = image._info(e.info)
        if e.data and e.bytes:
            raw = C.string_at(e.data, int(e.bytes))
            if png is not None:
                ev.data = raw
            elif bpp:
                ev.data = image._shape(np.frombuffer(raw, dtype=np.uint8).copy(), bpp)
            else:
                ev.data = np.frombuffer(raw, dtype=np.float32).copy()
    return ev


class Watch:
    """apt_watch (DESIGN.md §13): a continuous feed watched for satellite passes, each finished as its rows, image or PNG file.

        with Watch(48000, image_out="png", contrast=image.TELEMETRY, rgba=True) as w:
            for block in feed:                       # any sizes, float32 or int16
                q, events = w.push(block)
                for e in events:
                    if e.kind == "los" and e.status == 0:
                        open(f"pass{e.index}.png", "wb").write(e.data)
            q, events = w.finish()

    image_out None: each pass ends in its f32 rows; "image": its pixels; "png": its PNG file.  process: the keyword
    arguments of image.decode_image / decode_png.  Events are copied out during the callback."""

    def __init__(self, input_rate, settings=None, sync=True, search=None, image_out=None, max_rows=0, max_push=0, device=0,
                 **process):
        self._lib = _lib.load()
        self.input_rate = _rate_hz(input_rate)
        self.settings = settings or Settings()
        self._ps, self._bpp, self._png = _image_args(image_out, dict(process))
        self._ws = watch_settings(sync, search, self._ps[0] if self._ps else None, self._png, max_rows, max_push)
        self._events = []
        self._cb = _lib.WATCH_CB(self._on_event)
        s = self.settings.to_c()
        h = C.c_void_p(None)
        raise_for(self._lib.apt_watch_create(int(device), self.input_rate, C.byref(s), C.byref(self._ws), self._cb, None,
                                             C.byref(h)))
        self._h = h

    def _on_event(self, pev, _user):
        self._events.append(_watch_event(pev.contents, self._bpp, self._png))

    def close(self):
        if getattr(self, "_h", None):
            self._lib.apt_watch_destroy(self._h)
            self._h = None

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def _take(self):
        ev, self._events = self._events, []
        return ev

    def push(self, samples):
        """(q of the windows that became final, [PassEvent])."""
        x = np.ascontiguousarray(samples)
        fmt = _fmt_of(x)
        cap = C.c_uint64(0)
        raise_for(self._lib.apt_watch_push_bound(self._h, x.size, C.byref(cap)))
        q = np.empty(max(cap.value, 1), dtype=np.float32)
        nq = C.c_uint64(0)
        rc = self._lib.apt_watch_push(self._h, x.ctypes.data if x.size else None, fmt, x.size, q.ctypes.data, q.size,
                                      C.byref(nq))
        ev = self._take()
        raise_for(rc)
        return q[: nq.value].copy(), ev

    def finish(self):
        cap = C.c_uint64(0)
        raise_for(self._lib.apt_watch_push_bound(self._h, 0, C.byref(cap)))
        q = np.empty(max(cap.value, 1), dtype=np.float32)
        nq = C.c_uint64(0)
        rc = self._lib.apt_watch_finish(self._h, q.ctypes.data, q.size, C.byref(nq))
        ev = self._take()
        raise_for(rc)
        return q[: nq.value].copy(), ev

    def reset(self):
        raise_for(self._lib.apt_watch_reset(self._h))
        self._events = []

    def info(self):
        ci = _lib.CWatchInfo()
        raise_for(self._lib.apt_watch_get_info(self._h, C.byref(ci)))
        return {n: int(getattr(ci, n)) for n, _ in _lib.CWatchInfo._fields_}

    @property
    def device_bytes(self):
        return self.info()["device_bytes"]


def watch_geometry(input_rate, settings=None, sync=True, search=None, image_out=None, max_rows=0, max_push=0, **process):
    """apt_watch_geometry (host only): the device_bytes, max_push and latency_windows a Watch with these arguments has."""
    ps, _bpp, png = _image_args(image_out, dict(process))
    ws = watch_settings(sync, search, ps[0] if ps else None, png, max_rows, max_push)
    s = (settings or Settings()).to_c()
    ci = _lib.CWatchInfo()
    raise_for(_lib.load().apt_watch_geometry(_rate_hz(input_rate), C.byref(s), C.byref(ws), C.byref(ci)))
    return {n: int(getattr(ci, n)) for n, _ in _lib.CWatchInfo._fields_}


def _iq_watch_args(iq_settings, offsets):
    qs = iq_settings.to_c()
    qs.offset_hz = 0   # ignored: the channels are `offsets`
    offs, c_offs = _offsets(offsets)
    return qs, offs, c_offs


class IqWatch:
    """apt_watch_iq (DESIGN.md §14): one SDR's I/Q feed watched for passes on several channels at once (1..8 offsets, Hz
    from the tuned centre; iq_settings.offset_hz is ignored).  Channel c behaves as a Watch at iq_settings.audio_rate fed
    fm_demod(feed, offset_hz = offsets[c]); every step demodulates all channels in one kernel launch.

        s = iq.IqSettings(2_400_000)
        with IqWatch(s, [-400_000, 120_000, 412_500], image_out="png") as w:
            for block in feed:                       # uint8 (cu8), int16 (cs16) or complex64 / float32 (cf32)
                qs, events = w.push(block)           # qs[c]: channel c's new q
                for c, e in events:
                    if e.kind == "los" and e.status == 0:
                        open(f"ch{c}_pass{e.index}.png", "wb").write(e.data)
            qs, events = w.finish()

    Samples in events are audio samples of the channel; multiply by iq_settings.decimation for I/Q samples.  max_push
    counts I/Q samples.  The other arguments are Watch's."""

    def __init__(self, iq_settings, offsets, settings=None, sync=True, search=None, image_out=None, max_rows=0, max_push=0,
                 device=0, **process):
        self._lib = _lib.load()
        self.iq_settings = iq_settings
        self.settings = settings or Settings()
        qs, self.offsets, c_offs = _iq_watch_args(iq_settings, offsets)
        self._ps, self._bpp, self._png = _image_args(image_out, dict(process))
        self._ws = watch_settings(sync, search, self._ps[0] if self._ps else None, self._png, max_rows, max_push)
        self._events = []
        self._cb = _lib.WATCH_IQ_CB(self._on_event)
        s = self.settings.to_c()
        h = C.c_void_p(None)
        raise_for(self._lib.apt_watch_iq_create(int(device), C.byref(qs), c_offs, len(self.offsets), C.byref(s),
                                                C.byref(self._ws), self._cb, None, C.byref(h)))
        self._h = h

    @property
    def channels(self):
        return len(self.offsets)

    def _on_event(self, channel, pev, _user):
        self._events.append((int(channel), _watch_event(pev.contents, self._bpp, self._png)))

    def close(self):
        if getattr(self, "_h", None):
            self._lib.apt_watch_iq_destroy(self._h)
            self._h = None

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def _take(self):
        ev, self._events = self._events, []
        return ev

    def _q_buffers(self, n):
        cap = C.c_uint64(0)
        raise_for(self._lib.apt_watch_iq_push_bound(self._h, int(n), C.byref(cap)))
        cap = max(cap.value, 1)
        return np.empty((self.channels, cap), dtype=np.float32), cap, (C.c_uint64 * self.channels)()

    def push(self, iq):
        """([q of channel c's windows that became final], [(channel, PassEvent)])."""
        x, fmt, n = iq_format(iq)
        q, cap, nq = self._q_buffers(n)
        rc = self._lib.apt_watch_iq_push(self._h, x.ctypes.data if n else None, fmt, n, q.ctypes.data, cap, nq)
        ev = self._take()
        raise_for(rc)
        return [q[c, : nq[c]].copy() for c in range(self.channels)], ev

    def finish(self):
        q, cap, nq = self._q_buffers(0)
        rc = self._lib.apt_watch_iq_finish(self._h, q.ctypes.data, cap, nq)
        ev = self._take()
        raise_for(rc)
        return [q[c, : nq[c]].copy() for c in range(self.channels)], ev

    def reset(self):
        raise_for(self._lib.apt_watch_iq_reset(self._h))
        self._events = []

    def info(self, channel=0):
        ci = _lib.CWatchInfo()
        raise_for(self._lib.apt_watch_iq_get_info(self._h, int(channel), C.byref(ci)))
        return {n: int(getattr(ci, n)) for n, _ in _lib.CWatchInfo._fields_}

    @property
    def device_bytes(self):
        return self.info()["device_bytes"]


def watch_iq_geometry(iq_settings, offsets, settings=None, sync=True, search=None, image_out=None, max_rows=0, max_push=0,
                      **process):
    """apt_watch_iq_geometry (host only): the device_bytes, max_push (I/Q samples) and latency_windows an IqWatch with these
    arguments has."""
    qs, offs, c_offs = _iq_watch_args(iq_settings, offsets)
    ps, _bpp, png = _image_args(image_out, dict(process))
    ws = watch_settings(sync, search, ps[0] if ps else None, png, max_rows, max_push)
    s = (settings or Settings()).to_c()
    ci = _lib.CWatchInfo()
    raise_for(_lib.load().apt_watch_iq_geometry(C.byref(qs), c_offs, len(offs), C.byref(s), C.byref(ws), C.byref(ci)))
    return {n: int(getattr(ci, n)) for n, _ in _lib.CWatchInfo._fields_}
