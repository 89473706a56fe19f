"""CPU restatement of the project's PNG encoder (DESIGN.md §11), for the tests of image.encode_png / decode_png and the
GPU encoder.  Test infrastructure only.

The output bytes are a pure function of the pixels and the settings; every step below is the definition written out in
numpy and plain Python, in the order of DESIGN.md §11:

  1. filter     -- per row the five PNG filters, lowest sum of min(r, 256 - r) wins, ties to the lower type
  2. blocks     -- the filtered stream F cut into block_bytes pieces, one dynamic-Huffman deflate block each
  3. matches    -- m(i): last earlier position with the same 15-bit zlib hash within 32 KiB; l(i): common run capped at
                   min(258, end of i's block - i); a match needs l(i) >= 4
  4. parse      -- greedy, restarting at every block start
  5. lengths    -- package-merge (15 / 15 / 7 bits), ties: leaves before packages, lower symbols first; < 2 used symbols
                   completed with symbol 0 (or 1)
  6. header     -- HLIT / HDIST / HCLEN trimmed, the lengths run-length coded as one sequence (18 / 17 / 16 rules)
  7. container  -- zlib 78 9C + deflate + Adler-32; PNG signature, IHDR, one IDAT, IEND
"""
import zlib

import numpy as np

WINDOW = 32768
MAX_MATCH = 258
MIN_MATCH = 4
LIT_LIMIT, DIST_LIMIT, CL_LIMIT = 15, 15, 7
CL_ORDER = (16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15)
PNG_SIGNATURE = b"\x89PNG\r\n\x1a\n"
FRAMING = 57                    # signature 8 + IHDR 25 + IDAT length/type/CRC 12 + IEND 12
ZLIB_FRAMING = 6                # 78 9C + Adler-32

# RFC 1951 §3.2.5
LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0] + [k for k in range(1, 14) for _ in (0, 1)]


def _len_table():
    sym = np.zeros(MAX_MATCH + 1, dtype=np.int64)
    for c in range(29):
        hi = LEN_BASE[c + 1] if c < 28 else 259
        if c == 27:
            hi = 258                                  # 258 has its own code 285
        sym[LEN_BASE[c]:hi] = c
    return sym


LEN_SYM = _len_table()


def dist_sym(d):
    d = np.asarray(d, dtype=np.int64)
    return np.searchsorted(np.asarray(DIST_BASE), d, side="right") - 1


class Settings:
    def __init__(self, filter=-1, matches=1, block_bytes=65536, rgb_from_rgba=0):
        self.filter, self.matches, self.block_bytes, self.rgb_from_rgba = filter, matches, block_bytes, rgb_from_rgba


def check_settings(s):
    if not -1 <= s.filter <= 4:
        raise ValueError("filter")
    bb = s.block_bytes
    if bb < 4096 or bb > 65536 or bb & (bb - 1):
        raise ValueError("block_bytes")


# ---------------------------------------------------------------------------------------------------------- 1. filter

def paeth(a, b, c):
    a, b, c = (np.asarray(v, dtype=np.int16) for v in (a, b, c))
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c)).astype(np.uint8)


def residuals(img, bpp):
    """(5, rows, row_bytes) u8: the residuals of filter types 0..4 for every row of img (rows, row_bytes)."""
    x = img.astype(np.int16)
    a = np.zeros_like(x)
    a[:, bpp:] = x[:, :-bpp]
    b = np.zeros_like(x)
    b[1:] = x[:-1]
    c = np.zeros_like(x)
    c[1:, bpp:] = x[:-1, :-bpp]
    out = np.empty((5,) + x.shape, dtype=np.uint8)
    out[0] = img
    out[1] = (x - a) & 0xFF
    out[2] = (x - b) & 0xFF
    out[3] = (x - ((a + b) >> 1)) & 0xFF
    out[4] = (x - paeth(a, b, c)) & 0xFF
    return out


def filter_types(img, bpp, fixed=-1):
    rows = img.shape[0]
    if fixed >= 0:
        return np.full(rows, fixed, dtype=np.uint8)
    r = residuals(img, bpp).astype(np.int32)
    score = np.minimum(r, 256 - r).sum(axis=2)          # (5, rows)
    return np.argmin(score, axis=0).astype(np.uint8)   # first minimum: ties go to the lower type


def filtered_stream(pixels, channels, filter=-1, rgb_from_rgba=0):
    """The filtered stream F (u8) and the per-row filter types of a (height, width, channels) image."""
    img = np.ascontiguousarray(pixels, dtype=np.uint8)
    if img.ndim == 2:
        img = img[:, :, None]
    if rgb_from_rgba:
        img = img[:, :, :3]
    bpp = img.shape[2]
    img = img.reshape(img.shape[0], -1)
    types = filter_types(img, bpp, filter)
    res = residuals(img, bpp)
    rows = res[types, np.arange(img.shape[0])]
    f = np.concatenate([types[:, None], rows], axis=1).ravel()
    return np.ascontiguousarray(f), types


# --------------------------------------------------------------------------------------------------------- 3. matches

def hashes(f):
    f = f.astype(np.int64)
    return ((f[:-2] << 10) ^ (f[1:-1] << 5) ^ f[2:]) & 0x7FFF


def match_candidates(f, block_bytes):
    """(m, l) for every position: m = -1 where no earlier position has the hash within the window; l = 0 where no match
    (l < 4 counts as none)."""
    n = f.size
    m = np.full(n, -1, dtype=np.int64)
    ell = np.zeros(n, dtype=np.int64)
    if n < 3:
        return m, ell
    h = hashes(f)
    order = np.argsort(h, kind="stable")
    same = h[order[1:]] == h[order[:-1]]
    prev = np.full(h.size, -1, dtype=np.int64)
    prev[order[1:][same]] = order[:-1][same]
    pos = np.arange(h.size)
    ok = (prev >= 0) & (prev >= pos - WINDOW)
    m[:h.size] = np.where(ok, prev, -1)
    cap = np.minimum(MAX_MATCH, (pos // block_bytes + 1) * block_bytes - pos)
    cap = np.minimum(cap, n - pos)
    act = np.nonzero(ok)[0]
    # common runs compared eight bytes at a time: an unaligned little-endian u64 at every byte offset of F (padded)
    fp = np.zeros(n + 16 + MAX_MATCH, dtype=np.uint8)
    fp[:n] = f
    w64 = np.ndarray(shape=(n + MAX_MATCH,), dtype="<u8", buffer=fp, strides=(1,))
    run = np.zeros(act.size, dtype=np.int64)
    idx = np.arange(act.size)
    for t in range(0, MAX_MATCH, 8):
        if idx.size == 0:
            break
        i, j = act[idx], prev[act[idx]]
        x = w64[j + t] ^ w64[i + t]
        eq = x == 0
        run[idx[eq]] += 8
        ne = ~eq
        low = x[ne] & (~x[ne] + np.uint64(1))
        run[idx[ne]] += np.log2(low.astype(np.float64)).astype(np.int64) // 8
        idx = idx[eq]
    run = np.minimum(run, cap[act])
    ell[act] = np.where(run >= MIN_MATCH, run, 0)
    m[ell == 0] = -1
    return m, ell


# ----------------------------------------------------------------------------------------------------------- 4. parse

def parse_block(f, start, end, m, ell):
    """Greedy parse of F[start:end] -> (positions, lengths, distances) of its tokens; length 0 marks a literal."""
    ml = ell[start:end].tolist()
    pos = []
    p, n = 0, end - start
    while p < n:
        pos.append(p)
        p += ml[p] or 1
    pos = np.asarray(pos, dtype=np.int64) + start
    lens = ell[pos]
    dists = np.where(lens > 0, pos - m[pos], 0)
    return pos, lens, dists


# ---------------------------------------------------------------------------------------------------------- 5. lengths

def package_merge(freqs, limit):
    """Length-limited optimal code lengths.  Ties: leaves before packages, lower symbols before higher."""
    freqs = [int(v) for v in freqs]
    n = len(freqs)
    lengths = [0] * n
    used = [s for s in range(n) if freqs[s] > 0]
    if len(used) < 2:
        for s in used:
            lengths[s] = 1
        extra = 0 if not used or used[0] != 0 else 1
        lengths[extra] = 1
        if not used:
            lengths[1] = 1
        return lengths
    leaves = sorted(used, key=lambda s: (freqs[s], s))
    lw = [freqs[s] for s in leaves]
    levels = []
    prev = [(w, True) for w in lw]
    levels.append(prev)
    for _ in range(limit - 1):
        pk = [prev[2 * k][0] + prev[2 * k + 1][0] for k in range(len(prev) // 2)]
        merged, a, b = [], 0, 0
        while a < len(lw) or b < len(pk):
            if b >= len(pk) or (a < len(lw) and lw[a] <= pk[b]):
                merged.append((lw[a], True))
                a += 1
            else:
                merged.append((pk[b], False))
                b += 1
        levels.append(merged)
        prev = merged
    c = 2 * len(leaves) - 2
    depth = [0] * len(leaves)
    for lvl in reversed(levels):
        nleaf = sum(1 for w, leaf in lvl[:c] if leaf)
        for r in range(nleaf):
            depth[r] += 1
        c = 2 * (c - nleaf)
    for r, s in enumerate(leaves):
        lengths[s] = depth[r]
    return lengths


def canonical_codes(lengths):
    """RFC 1951 §3.2.2 codes, returned bit-reversed (ready for LSB-first packing)."""
    lengths = list(lengths)
    maxl = max(lengths) if lengths else 0
    bl = [0] * (maxl + 2)
    for L in lengths:
        if L:
            bl[L] += 1
    code, nxt = 0, [0] * (maxl + 2)
    for bits in range(1, maxl + 1):
        code = (code + bl[bits - 1]) << 1
        nxt[bits] = code
    out = [0] * len(lengths)
    for s, L in enumerate(lengths):
        if L:
            c = nxt[L]
            nxt[L] += 1
            out[s] = int(format(c, f"0{L}b")[::-1], 2)
    return out


def kraft_ok(lengths, limit):
    used = [L for L in lengths if L]
    return all(L <= limit for L in used) and sum(2.0 ** -L for L in used) == 1.0


# ----------------------------------------------------------------------------------------------------------- 6. header

def rle_lengths(lengths):
    """[(symbol, extra value, extra bits)] of the run-length coded code-length sequence."""
    out, i, n = [], 0, len(lengths)
    while i < n:
        v = lengths[i]
        run = 1
        while i + run < n and lengths[i + run] == v:
            run += 1
        if v == 0:
            r = run
            while r >= 11:
                k = min(r, 138)
                out.append((18, k - 11, 7))
                r -= k
            if r >= 3:
                out.append((17, r - 3, 3))
                r = 0
            out.extend([(0, 0, 0)] * r)
        else:
            out.append((v, 0, 0))
            r = run - 1
            while r >= 3:
                k = min(r, 6)
                out.append((16, k - 3, 2))
                r -= k
            out.extend([(v, 0, 0)] * r)
        i += run
    return out


class BitWriter:
    """LSB-first bit packing (RFC 1951 §3.1.1) of (value, bit count) pieces; counts of 0 write nothing."""

    def __init__(self):
        self.vals, self.lens = [], []

    def put(self, v, n):
        self.put_many([v], [n])

    def put_many(self, vals, lens):
        self.vals.append(np.asarray(vals, dtype=np.int64).ravel())
        self.lens.append(np.asarray(lens, dtype=np.int64).ravel())

    def bits(self):
        return int(sum(int(L.sum()) for L in self.lens))

    def to_bytes(self):
        if not self.vals:
            return b""
        v = np.concatenate(self.vals)
        L = np.concatenate(self.lens)
        mat = (v[:, None] >> np.arange(16)) & 1
        keep = np.arange(16)[None, :] < L[:, None]
        return np.packbits(mat[keep].astype(np.uint8), bitorder="little").tobytes()


def block_bits(f, toks, final, w):
    """Appends one dynamic-Huffman block to BitWriter w; returns (lit lengths, dist lengths, cl lengths)."""
    pos, lens, dists = toks
    lit = lens == 0
    lsym = np.where(lit, f[pos].astype(np.int64), 257 + LEN_SYM[lens])
    dsym = np.where(lit, 0, dist_sym(np.maximum(dists, 1)))
    lf = np.bincount(lsym, minlength=286).tolist()
    lf[256] += 1
    df = np.bincount(dsym[~lit], minlength=30).tolist()
    ll = package_merge(lf, LIT_LIMIT)
    dl = package_merge(df, DIST_LIMIT)
    hlit = max(257, max((s + 1 for s in range(286) if ll[s]), default=0))
    hdist = max(1, max((s + 1 for s in range(30) if dl[s]), default=0))
    seq = rle_lengths(ll[:hlit] + dl[:hdist])
    cf = [0] * 19
    for s, _, _ in seq:
        cf[s] += 1
    cl = package_merge(cf, CL_LIMIT)
    hclen = 19
    while hclen > 4 and cl[CL_ORDER[hclen - 1]] == 0:
        hclen -= 1
    w.put_many([1 if final else 0, 2, hlit - 257, hdist - 1, hclen - 4], [1, 2, 5, 5, 4])
    w.put_many([cl[CL_ORDER[k]] for k in range(hclen)], [3] * hclen)
    cc = canonical_codes(cl)
    hv, hl = [], []
    for s, ev, eb in seq:
        hv += [cc[s], ev]
        hl += [cl[s], eb]
    w.put_many(hv, hl)
    lc = np.asarray(canonical_codes(ll), dtype=np.int64)
    dc = np.asarray(canonical_codes(dl), dtype=np.int64)
    lla, dla = np.asarray(ll, dtype=np.int64), np.asarray(dl, dtype=np.int64)
    ls = np.maximum(lsym - 257, 0)
    vals = np.stack([lc[lsym], np.where(lit, 0, lens - np.asarray(LEN_BASE)[ls]), dc[dsym],
                     np.where(lit, 0, dists - np.asarray(DIST_BASE)[dsym])], axis=1)
    nbits = np.stack([lla[lsym], np.where(lit, 0, np.asarray(LEN_EXTRA)[ls]), np.where(lit, 0, dla[dsym]),
                      np.where(lit, 0, np.asarray(DIST_EXTRA)[dsym])], axis=1)
    w.put_many(vals, nbits)
    w.put(lc[256], ll[256])
    return ll, dl, cl


# -------------------------------------------------------------------------------------------------------- 7. container

def adler32(f):
    """zlib's Adler-32, from the closed form s1 = 1 + sum F, s2 = N + sum (N - i) F[i] (mod 65521)."""
    f = np.asarray(f, dtype=np.uint64)
    n = f.size
    s1 = (1 + int(f.sum(dtype=np.uint64))) % 65521
    w = (np.uint64(n) - np.arange(n, dtype=np.uint64)) % np.uint64(65521)
    s2 = (n + int(((f * w) % np.uint64(65521)).sum(dtype=np.uint64))) % 65521
    return (s2 << 16) | s1


_CRC_TABLE = None


def crc32(data, crc=0):
    """Table-driven CRC-32 (reflected 0xEDB88320), byte at a time -- the restatement zlib.crc32 is checked against."""
    global _CRC_TABLE
    if _CRC_TABLE is None:
        t = []
        for k in range(256):
            c = k
            for _ in range(8):
                c = (c >> 1) ^ 0xEDB88320 if c & 1 else c >> 1
            t.append(c)
        _CRC_TABLE = t
    c = crc ^ 0xFFFFFFFF
    for b in bytes(data):
        c = _CRC_TABLE[(c ^ b) & 0xFF] ^ (c >> 8)
    return c ^ 0xFFFFFFFF


def deflate(f, block_bytes=65536, matches=1, info=None):
    n = f.size
    if matches:
        m, ell = match_candidates(f, block_bytes)
    else:
        m, ell = np.full(n, -1, np.int64), np.zeros(n, np.int64)
    w = BitWriter()
    nb = (n + block_bytes - 1) // block_bytes
    for b in range(nb):
        s, e = b * block_bytes, min(n, (b + 1) * block_bytes)
        toks = parse_block(f, s, e, m, ell)
        ll, dl, cl = block_bits(f, toks, b == nb - 1, w)
        if info is not None:
            info.setdefault("trees", []).append((ll, dl, cl))
            info.setdefault("tokens", []).append(len(toks[0]))
    if info is not None:
        info["deflate_bits"] = w.bits()
    return w.to_bytes()


def zlib_stream(f, block_bytes=65536, matches=1, info=None):
    return b"\x78\x9c" + deflate(f, block_bytes, matches, info) + int(adler32(f)).to_bytes(4, "big")


def _chunk(kind, data, crc=zlib.crc32):
    return len(data).to_bytes(4, "big") + kind + data + crc(kind + data).to_bytes(4, "big")


def bound(width, height, channels, block_bytes=65536, rgb_from_rgba=0):
    c = 3 if (channels == 4 and rgb_from_rgba) else channels
    n = height * (1 + width * c)
    nb = (n + block_bytes - 1) // block_bytes
    bits = 9 * n + nb * (9 + 2400)
    return FRAMING + ZLIB_FRAMING + (bits + 7) // 8


def encode(pixels, filter=-1, matches=1, block_bytes=65536, rgb_from_rgba=0, info=None, crc=zlib.crc32):
    """PNG bytes of (height, width[, channels]) u8 pixels, channels 1 / 3 / 4."""
    img = np.asarray(pixels, dtype=np.uint8)
    if img.ndim == 2:
        img = img[:, :, None]
    h, wd, ch = img.shape
    if rgb_from_rgba and (ch != 4 or np.any(img[:, :, 3] != 255)):
        raise ValueError("rgb_from_rgba needs RGBA pixels with alpha 255")
    f, types = filtered_stream(img, ch, filter, rgb_from_rgba)
    if info is not None:
        info["filter_types"] = types
        info["F"] = f
    z = zlib_stream(f, block_bytes, matches, info)
    out_ch = 3 if rgb_from_rgba else ch
    ctype = {1: 0, 3: 2, 4: 6}[out_ch]
    ihdr = wd.to_bytes(4, "big") + h.to_bytes(4, "big") + bytes([8, ctype, 0, 0, 0])
    return PNG_SIGNATURE + _chunk(b"IHDR", ihdr, crc) + _chunk(b"IDAT", z, crc) + _chunk(b"IEND", b"", crc)
