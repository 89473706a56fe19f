"""CPU restatement of the rest of noaa_apt::process (noaa_apt.rs:140-240), the map overlay excepted, for the tests of
image.process / decode_image.  Test infrastructure only.

The contrast bounds and map_signal_u8 come from the C oracle (oracle/); this module restates what follows on the u8
image, step by step as the reference writes it.  numpy float32 arithmetic rounds every operation on its own and never
contracts to FMA, like the Rust code; integer -> f32 conversions round to nearest, like `as f32`.

Column layout (decode.rs:16-35): channel A is x in [0, 1040), B is x in [1040, 2080); the image data of A is x in
[86, 995), of B x in [1126, 2035)."""
import numpy as np

import oracle

PX_PER_ROW, PX_PER_CHANNEL = 2080, 1040
IMG_X0, IMG_X1 = 86, 995                      # PX_SYNC_FRAME + PX_SPACE_DATA, + PX_CHANNEL_IMAGE_DATA
MINMAX, PERCENT, TELEMETRY, HISTOGRAM = 0, 1, 2, 3


def _as_u8(v):
    """f32 `as u8` / `as u32` for values the reference clamps to [0, 255]: truncation, NaN -> 0."""
    v = np.asarray(v, dtype=np.float32)
    return np.where(np.isnan(v), np.float32(0), np.clip(np.trunc(v), 0, 255)).astype(np.uint8)


def equalize_lut(half):
    """imageext.rs:23-46, :95-119 on one channel half: the cumulative u32 histogram, total = hist[255] as f32,
    value v -> (255.0 * (hist[v] as f32 / total)) as u8.  Returns the 256-entry table."""
    hist = np.cumsum(np.bincount(half.ravel(), minlength=256)).astype(np.uint32)
    total = np.float32(hist[255])
    fraction = hist.astype(np.float32) / total
    return _as_u8(np.float32(255.0) * fraction)


def equalize(grey):
    """processing.rs:87-103 with has_color = false: each 1040-px channel half over all rows separately."""
    out = np.empty_like(grey)
    for c in (0, 1):
        half = grey[:, c * PX_PER_CHANNEL:(c + 1) * PX_PER_CHANNEL]
        out[:, c * PX_PER_CHANNEL:(c + 1) * PX_PER_CHANNEL] = equalize_lut(half)[half]
    return out


def tune_values(v, start, end):
    """processing.rs:125-140 tune_input_values for one channel: (v * ((1 + e) - s) - s * 255).clamp(0, 255) as u32,
    s = start * 0.3, e = end * 0.3."""
    factor = np.float32(0.3)
    s = np.float32(start) * factor
    e = np.float32(end) * factor
    out = np.asarray(v, dtype=np.uint8).astype(np.float32) * ((np.float32(1.0) + e) - s) - s * np.float32(255.0)
    return _as_u8(out).astype(np.uint32)


def false_color(rgba, palette, tune):
    """processing.rs:108-157 in place on the RGBA image: channel A's image columns become palette[val_b][val_a]."""
    a = rgba[:, IMG_X0:IMG_X1, 0]
    b = rgba[:, IMG_X0 + PX_PER_CHANNEL:IMG_X1 + PX_PER_CHANNEL, 0]     # never written: no read-after-write hazard
    va = tune_values(a, tune[0], tune[1])
    vb = tune_values(b, tune[2], tune[3])
    rgba[:, IMG_X0:IMG_X1, :3] = palette[vb, va]
    rgba[:, IMG_X0:IMG_X1, 3] = 255


def rotate(img):
    """processing.rs:21-37: rotate180_in_place on the two 909-px image rectangles, all rows.  Works on (rows, 2080)
    and (rows, 2080, 4) images; returns a new array."""
    out = img.copy()
    for x0 in (IMG_X0, IMG_X0 + PX_PER_CHANNEL):
        x1 = x0 + (IMG_X1 - IMG_X0)
        out[:, x0:x1] = img[::-1, x0:x1][:, ::-1]
    return out


def bounds(rows, contrast, percent=0.98):
    """(low, high) of noaa_apt.rs:140-163; Contrast::Histogram takes MinMax."""
    if contrast in (MINMAX, HISTOGRAM):
        return oracle.minmax(rows)
    if contrast == PERCENT:
        return oracle.percent(rows, percent)
    wa, wb, _ = oracle.read_telemetry(rows)
    low = float((np.float32(wa[8]) + np.float32(wb[8])) / np.float32(2))
    high = float((np.float32(wa[7]) + np.float32(wb[7])) / np.float32(2))
    return low, high


def process_grey(grey, contrast, rotate_=False, palette=None, tune=(0, 0, 0, 0), rgba=None):
    """Steps after map_signal_u8 on a (rows, 2080) u8 image, in process()'s order: into_rgba8 -> false colour ->
    histogram equalisation -> rotation.  rgba=None: RGBA with a palette, else grey."""
    if rgba is None:
        rgba = palette is not None
    if palette is not None and not rgba:
        raise ValueError("false colour needs RGBA output")
    if palette is not None and contrast == HISTOGRAM:
        raise ValueError("colour histogram equalisation is not available")
    grey = np.asarray(grey, dtype=np.uint8).reshape(-1, PX_PER_ROW)
    if contrast == HISTOGRAM:
        grey = equalize(grey)     # R = G = B: the R histogram applied to all three (imageext.rs:23-46)
    if rgba:
        img = np.empty(grey.shape + (4,), dtype=np.uint8)
        img[..., :3] = grey[..., None]
        img[..., 3] = 255
        if palette is not None:
            false_color(img, np.asarray(palette, dtype=np.uint8), tune)
    else:
        img = grey.copy()
    return rotate(img) if rotate_ else img


def process(rows, contrast, percent=0.98, rotate_=False, palette=None, tune=(0, 0, 0, 0), rgba=None):
    """noaa_apt::process without the map on f32 rows -> (image, (low, high))."""
    rows = np.ascontiguousarray(rows, dtype=np.float32).ravel()
    low, high = bounds(rows, contrast, percent)
    grey = oracle.map_signal_u8(rows, low, high).reshape(-1, PX_PER_ROW)
    return process_grey(grey, contrast, rotate_, palette, tune, rgba), (low, high)
