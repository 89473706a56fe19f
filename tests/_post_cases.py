"""Edge inputs of the image stage's min / max (dsp::get_min / get_max, dsp.rs:20-54), shared by the CPU check of the C
oracle (test_post_oracle_cpu.py) and the device comparison (test_gpu_post_exact.py).  Test infrastructure only.

Each case is (name, f32 values, old_rule_differs): old_rule_differs says whether an unordered min / max over a
monotone float -> u32 key (NaN ordered above +Inf or below -Inf, -0.0 below +0.0) gives other bits than the
reference's walk from x[0] with strict `<` / `>`.  Those cases are the ones that tell the two rules apart."""
import numpy as np


def f32_bits(u):
    return np.array([u], dtype=np.uint32).view(np.float32)[0]


NAN = f32_bits(0x7FC00000)
NEG_NAN = f32_bits(0xFFC00000)
NAN_PAYLOAD = f32_bits(0x7FC12345)
NEG_NAN_PAYLOAD = f32_bits(0xFFD00001)
INF = np.float32(np.inf)
SUB = f32_bits(0x00000001)                      # smallest subnormal
SUB_MAX = f32_bits(0x007FFFFF)                  # largest subnormal
Z, NZ = np.float32(0.0), np.float32(-0.0)


def _a(*v):
    return np.array(v, dtype=np.float32)


MINMAX_CASES = [
    ("nan_middle", _a(0.2, 0.5, NAN, 0.9, 0.1), True),
    ("nan_first", _a(NAN, 0.5, 0.9, 0.1), True),
    ("neg_nan_middle", _a(0.2, NEG_NAN, 0.9), True),
    ("nan_last", _a(0.3, -0.5, 0.25, NAN_PAYLOAD), True),
    ("nan_payload_first", _a(NAN_PAYLOAD, -4.0, 7.0), True),
    ("neg_nan_payload_first", _a(NEG_NAN_PAYLOAD, -4.0, 7.0), True),
    ("all_nan_two_payloads", _a(NAN, NAN_PAYLOAD, NEG_NAN), True),
    ("max_neg_zero_then_pos_zero", _a(NZ, -1.0, Z, -2.0), True),
    ("min_pos_zero_then_neg_zero", _a(1.0, Z, NZ, 2.0), True),
    ("min_zero_first_pos", _a(Z, 1.0, NZ), True),
    ("max_zero_first_neg", _a(-1.0, NZ, -3.0, Z), True),
    ("zeros_neg_first", _a(NZ, Z), True),
    ("zeros_pos_first", _a(Z, NZ), True),
    ("min_neg_zero_then_pos_zero", _a(3.0, NZ, 5.0, Z), False),
    ("max_pos_zero_then_neg_zero", _a(-1.0, Z, NZ, -3.0), False),
    ("infinities", _a(1.0, INF, -INF, 2.0), False),
    ("inf_and_nan", _a(-INF, NAN, INF), True),
    ("subnormal_extremes", _a(0.0, SUB, -SUB, SUB_MAX, -SUB_MAX), False),
    ("subnormal_and_zeros", _a(SUB, NZ, Z, -SUB), False),
    ("constant", _a(0.75, 0.75, 0.75), False),
    ("one_pixel", _a(-3.5), False),
    ("one_nan_pixel", _a(NEG_NAN_PAYLOAD), False),
]


def old_rule_minmax(x):
    """min / max over the ordered-int key as an unordered atomic reduction takes them (the rule the device used before it
    followed dsp::get_min / get_max): -> (min, max) as f32."""
    b = np.asarray(x, dtype=np.float32).view(np.uint32)
    key = np.where(b & 0x80000000, ~b, b | 0x80000000).astype(np.uint32)

    def back(k):
        k = np.uint32(k)
        return f32_bits((k & 0x7FFFFFFF) if k & 0x80000000 else ~k)
    return back(key.min()), back(key.max())


def preimages(targets, low, high, scale):
    """For each target t, the f32 values x near low + t * (high - low) / scale whose f32 computation
    (x - low) / (high - low) * scale is exactly t, and those where it is one ulp below t -> (exact, below) arrays."""
    low, high, scale = np.float32(low), np.float32(high), np.float32(scale)
    rng = high - low
    exact, below = [], []
    with np.errstate(all="ignore"):
        for t in np.asarray(targets, dtype=np.float32):
            x0 = np.float32(float(low) + float(t) * float(rng) / float(scale))
            xs = (x0.view(np.int32) + np.arange(-64, 65, dtype=np.int32)).view(np.float32)
            v = (xs - low) / rng * scale
            e = xs[v == t]
            b = xs[v == np.nextafter(t, np.float32(-np.inf))]
            if e.size:
                exact.append(e[0])
            if b.size:
                below.append(b[-1])
    return np.array(exact, np.float32), np.array(below, np.float32)


def telemetry_image(rows, seed=0, nan_row=None, zero_var=None, negative=False, period=None):
    """(rows * 2080,) f32 rows with telemetry-like bands (wedges of 8 rows, noise across the band): nan_row puts a NaN in
    channel A's band of that row; zero_var = (r0, r1) makes the bands of those rows constant (variance exactly 0, so
    quality +Inf where a whole frame lies inside); negative makes every band mean, so every quality, negative; period
    repeats the rows with that period, so equal qualities recur every `period` rows."""
    r = np.random.default_rng(seed)
    n = period or rows
    x = r.random((n, 2080), dtype=np.float32)
    wedge = np.array([31, 63, 95, 127, 159, 191, 224, 255, 0] + [0] * 7, np.float32) / np.float32(255)
    per_row = np.tile(np.repeat(wedge, 8), n // 128 + 1)[:n] * np.float32(0.8) + r.random(n, dtype=np.float32) * np.float32(0.2)
    for c0 in (994, 2034):
        x[:, c0:c0 + 44] = per_row[:, None] + r.random((n, 44), dtype=np.float32) * np.float32(0.05)
        if zero_var is not None:                                   # multiples of 2^-8: the band mean is exact, variance 0
            lo, hi = zero_var
            x[lo:hi, c0:c0 + 44] = (np.round(per_row[lo:hi] * 256) / 256 + np.float32(1 / 64))[:, None]
    if period:
        x = np.tile(x, (rows // period + 1, 1))[:rows]
    if negative:
        x = -x - np.float32(1)
    if nan_row is not None:
        x[nan_row, 1000] = NAN
    return x.ravel()
