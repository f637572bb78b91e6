"""PNGs of every colour type, bit depth and interlace method, written here with chosen filters, zlib modes and chunk
cuts, and a numpy model of the general decode (http_master.parse_png_general's filtered stream -> u8 RGB, as the
installed Pillow's convert("RGB") gives it)."""
import struct
import zlib

import numpy as np

from __graft_entry__ import load_package

load_package()
from comfyui_distributed_b200 import http_master as hm  # noqa: E402

SIGNATURE = b"\x89PNG\r\n\x1a\n"
MODES = [(c, d) for c, ds in sorted(hm.GENERAL_DEPTHS.items()) for d in ds]     # every legal (colour type, depth)


def chunk(ctype: bytes, data: bytes) -> bytes:
    return struct.pack(">I", len(data)) + ctype + data + struct.pack(">I", zlib.crc32(ctype + data))


def _passes(W, H, interlace):
    for x0, y0, dx, dy in (hm.ADAM7 if interlace else ((0, 0, 1, 1),)):
        pw, ph = max(0, (W - x0 + dx - 1) // dx), max(0, (H - y0 + dy - 1) // dy)
        if pw and ph:
            yield x0, y0, dx, dy, pw, ph


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def filter_row(f: int, cur: np.ndarray, prev: np.ndarray, bpp: int) -> np.ndarray:
    """PNG filter `f` of the raw row `cur` (int32) over the raw row `prev` (zeros above a pass's first row)."""
    a = np.concatenate([np.zeros(bpp, np.int32), cur[:-bpp]]) if len(cur) > bpp else np.zeros_like(cur)
    c = np.concatenate([np.zeros(bpp, np.int32), prev[:-bpp]]) if len(prev) > bpp else np.zeros_like(prev)
    pred = [np.zeros_like(cur), a, prev, (a + prev) >> 1, _paeth(a, prev, c)][f]
    return ((cur - pred) & 0xFF).astype(np.uint8)


def raw_rows(rng, color, depth, W, H, interlace):
    """Random raw (unfiltered) rows per pass; 16-bit rows are sometimes small values (16-bit grey's clip at 255)."""
    out = []
    for x0, y0, dx, dy, pw, ph in _passes(W, H, interlace):
        n = (pw * depth * hm.GENERAL_CHANNELS[color] + 7) // 8
        rows = rng.integers(0, 256, (ph, n), dtype=np.int32)
        if depth == 16:
            for r in range(ph):
                if rng.random() < 0.5:
                    rows[r, 0::2] = rng.integers(0, 2, n // 2)
        out.append(rows)
    return out


def make_png(rng, color, depth, W, H, interlace, level=6, idat_cuts=3, plte_entries=None, trns=None, filters=None,
             comp=0, raw=None):
    """A PNG with the given IHDR, random pixels (or `raw`, per pass), row r of pass p filtered with
    filters(p, r) (default: cycling through all five), zlib `level` (0: stored blocks), the stream cut into
    `idat_cuts` IDAT chunks at random points, a PLTE of `plte_entries` entries (colour type 3) and a tRNS chunk."""
    C = hm.GENERAL_CHANNELS[color]
    bpp = max(1, depth * C // 8)
    raw = raw if raw is not None else raw_rows(rng, color, depth, W, H, interlace)
    off = int(rng.integers(0, 5))
    filters = filters or (lambda p, r: (off + p + r) % 5)
    R = bytearray()
    for p, rows in enumerate(raw):
        prev = np.zeros(rows.shape[1], np.int32)
        for r in range(rows.shape[0]):
            f = filters(p, r)
            R.append(f)
            R += filter_row(f, rows[r], prev, bpp).tobytes()
            prev = rows[r]
    z = zlib.compress(bytes(R), level)
    cuts = sorted(set(int(v) for v in rng.integers(1, max(2, len(z)), max(0, idat_cuts - 1))))
    pieces = [z[a:b] for a, b in zip([0] + cuts, cuts + [len(z)])]
    out = SIGNATURE + chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, depth, color, comp, 0, interlace))
    if color == 3:
        k = plte_entries if plte_entries is not None else 1 << depth
        out += chunk(b"PLTE", rng.integers(0, 256, 3 * k, dtype=np.uint8).tobytes())
    if trns is not None:
        out += chunk(b"tRNS", trns)
    for piece in pieces:
        out += chunk(b"IDAT", piece)
    return out + chunk(b"IEND", b"")


def trns_for(rng, color, depth):
    if color == 0:
        return struct.pack(">H", int(rng.integers(0, 1 << depth)))
    if color == 2:
        return struct.pack(">HHH", *(int(v) for v in rng.integers(0, 1 << depth, 3)))
    if color == 3:
        return rng.integers(0, 256, int(rng.integers(1, 1 << depth)), dtype=np.uint8).tobytes()
    return None


def corpus(seed=0):
    """[(name, PNG bytes)]: every (colour type, depth) with interlace 0 and 1; widths 1..17 against heights cycling
    1..9, plus wider odd shapes; every filter on some row of each pass; stored and compressed streams cut into several
    IDAT chunks; short PLTEs; tRNS on grey, RGB and palette files."""
    rng = np.random.default_rng(seed)
    shapes = [(w, 1 + (w * 5) % 9) for w in range(1, 18)] + [(31, 9), (33, 8), (67, 5), (129, 3), (255, 11)]
    out = []
    for color, depth in MODES:
        for interlace in (0, 1):
            for i, (W, H) in enumerate(shapes):
                level = (0, 6, 9)[i % 3]
                plte = None
                if color == 3:
                    plte = [1 << depth, max(1, (1 << depth) // 2 - 1), 1][i % 3]
                trns = trns_for(rng, color, depth) if i % 4 == 1 else None
                name = f"c{color}d{depth}i{interlace}_{W}x{H}_z{level}"
                out.append((name, make_png(rng, color, depth, W, H, interlace, level, 1 + i % 4, plte, trns,
                                           filters=lambda p, r, i=i: (i + p + r) % 5)))
    return out


def unfilter(R: np.ndarray, ph: int, n: int, bpp: int) -> np.ndarray:
    """The pass's filtered rows ([ph, 1 + n] of R) -> raw rows [ph, n] (int32)."""
    rows = R.reshape(ph, 1 + n)
    out = np.zeros((ph, n), np.int32)
    prev = np.zeros(n, np.int32)
    for r in range(ph):
        f, row = int(rows[r, 0]), rows[r, 1:].astype(np.int32)
        if f == 0:
            cur = row
        elif f == 2:
            cur = (row + prev) & 0xFF
        else:
            cur = np.zeros(n, np.int32)
            for x in range(n):
                a = int(cur[x - bpp]) if x >= bpp else 0
                b = int(prev[x])
                c = int(prev[x - bpp]) if x >= bpp else 0
                pred = a if f == 1 else (a + b) >> 1 if f == 3 else int(_paeth(np.int32(a), np.int32(b), np.int32(c)))
                cur[x] = (int(row[x]) + pred) & 0xFF
        out[r] = cur
        prev = cur
    return out


def to_rgb(info, raw: np.ndarray, pw: int) -> np.ndarray:
    """Raw rows [ph, n] of a pass -> u8 RGB [ph, pw, 3] as PIL's convert("RGB")."""
    C, depth, ph = info.C, info.depth, raw.shape[0]
    if depth < 8:
        bits = np.unpackbits(raw.astype(np.uint8), axis=1).reshape(ph, -1, depth)
        s = (bits * (1 << np.arange(depth - 1, -1, -1))).sum(2)[:, :pw * C].reshape(ph, pw, C)
    elif depth == 8:
        s = raw.reshape(ph, pw, C)
    else:
        s = (raw[:, 0::2] * 256 + raw[:, 1::2]).reshape(ph, pw, C)
    if info.color == 3:
        pal = np.frombuffer(info.palette, np.uint8).reshape(256, 3)
        return pal[s[..., 0]]
    if info.color == 0:
        g = s[..., 0] * (255 // ((1 << depth) - 1)) if depth < 8 else np.minimum(s[..., 0], 255) if depth == 16 \
            else s[..., 0]
        return np.repeat(g[..., None], 3, 2).astype(np.uint8)
    hi = s >> 8 if depth == 16 else s
    return (np.repeat(hi[..., :1], 3, 2) if C < 3 else hi[..., :3]).astype(np.uint8)


def decode_model(info) -> np.ndarray:
    """PngGeneral -> u8 [H, W, 3]: each pass un-filtered on units of info.bpp bytes, converted, and scattered."""
    out = np.zeros((info.H, info.W, 3), np.uint8)
    R = np.frombuffer(info.inflated, np.uint8)
    for x0, y0, dx, dy, pw, ph, at in info.passes():
        n = info.row_bytes(pw)
        raw = unfilter(R[at: at + ph * (1 + n)], ph, n, info.bpp)
        out[y0::dy, x0::dx][:ph, :pw] = to_rgb(info, raw, pw)
    return out


def pack_passes(samples: np.ndarray, depth: int, interlace: int):
    """Samples [H, W, C] (grey, palette indices or colour values at `depth` bits) -> the raw rows of each pass, as
    make_png's `raw` takes them."""
    H, W, C = samples.shape
    out = []
    for x0, y0, dx, dy, pw, ph in _passes(W, H, interlace):
        s = samples[y0::dy, x0::dx][:ph, :pw].astype(np.uint32).reshape(ph, pw * C)
        if depth == 16:
            b = np.stack([s >> 8, s & 0xFF], 2).reshape(ph, -1)
        elif depth == 8:
            b = s
        else:
            bits = ((s[..., None] >> np.arange(depth - 1, -1, -1)) & 1).astype(np.uint8).reshape(ph, -1)
            b = np.packbits(bits, axis=1)
        out.append(b.astype(np.int32))
    return out


def encode_as(rng, rgb: np.ndarray, fmt: str, level=6, idat_cuts=2) -> bytes:
    """A PNG in format `fmt` whose convert("RGB") is the u8 image `rgb` [H, W, 3]: "rgb16" / "rgba16" / "la16" (the
    pixels in the high bytes, random low bytes), "grey16" (grey pixels as values below 256), "grey1/2/4" (grey levels
    the depth holds), "pal1/2/4/8" (at most 2^depth colours), each with "_i" for Adam7."""
    base, _, il = fmt.partition("_")
    interlace = int(il == "i")
    H, W, _ = rgb.shape
    if base in ("rgb16", "rgba16", "la16"):
        C = {"rgb16": 3, "rgba16": 4, "la16": 2}[base]
        hi = rgb[..., :3] if C >= 3 else rgb[..., :1]
        if C in (2, 4):
            hi = np.concatenate([hi, rng.integers(0, 256, (H, W, 1))], 2)
        s = hi.astype(np.uint32) * 256 + rng.integers(0, 256, hi.shape)
        color = {3: 2, 4: 6, 2: 4}[C]
        return make_png(rng, color, 16, W, H, interlace, level, idat_cuts, raw=pack_passes(s, 16, interlace))
    if base == "grey16":
        return make_png(rng, 0, 16, W, H, interlace, level, idat_cuts, raw=pack_passes(rgb[..., :1], 16, interlace))
    if base.startswith("grey"):
        d = int(base[4:])
        s = rgb[..., :1] // (255 // ((1 << d) - 1))
        return make_png(rng, 0, d, W, H, interlace, level, idat_cuts, raw=pack_passes(s, d, interlace))
    if base.startswith("pal"):
        d = int(base[3:])
        colours, idx = np.unique(rgb.reshape(-1, 3), axis=0, return_inverse=True)
        assert len(colours) <= 1 << d, "too many colours for the palette"
        out = SIGNATURE + chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, d, 3, 0, 0, interlace))
        out += chunk(b"PLTE", colours.astype(np.uint8).tobytes())
        body = make_png(rng, 3, d, W, H, interlace, level, idat_cuts, plte_entries=0,
                        raw=pack_passes(idx.reshape(H, W, 1), d, interlace))
        return out + body[body.index(b"IDAT") - 4:]
    raise ValueError(fmt)


def palette_image(rng, H, W, colours: int) -> np.ndarray:
    """A u8 RGB image of at most `colours` colours."""
    pal = rng.integers(0, 256, (colours, 3), dtype=np.uint8)
    return pal[rng.integers(0, colours, (H, W))]


def grey_image(rng, H, W, depth: int = 8) -> np.ndarray:
    """A u8 grey image (replicated to RGB) whose levels a `depth`-bit grey PNG holds."""
    step = 255 // ((1 << depth) - 1)
    return np.repeat((rng.integers(0, 1 << depth, (H, W, 1)) * step).astype(np.uint8), 3, 2)
