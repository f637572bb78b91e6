"""numpy restatement of the baseline JPEG decode's device stages (csrc/usdu_jpeg_decode.cu), and a small baseline
encoder that writes arbitrary quantised coefficients (4:4:0, RGB-coded files, IDCT overflow and range-limit cases no
real encoder produces).

model_decode(info, quant, coefs) takes the library's host parse and Huffman decode (_native.jpeg_parse,
jpeg_decode_coefs) and returns the [H, W, 3] u8 frame PIL's open().convert("RGB") gives."""
from __future__ import annotations

import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
                   6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45,
                   38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])
F298, F390, F541, F765, F899, F1175 = 2446, 3196, 4433, 6270, 7373, 9633
F1501, F1847, F1961, F2053, F2562, F3072 = 12299, 15137, 16069, 16819, 20995, 25172


def w16(x):
    return ((x + 32768) & 0xFFFF) - 32768


def w32(x):
    return ((x + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


def sat(x, lo, hi):
    return np.clip(x, lo, hi)


def idct8(x):
    """One pass over 8 int64 arrays of 16-bit values -> 8 arrays, exact before the 32-bit wrap (applied by the
    caller before its shift: every step is an add, subtract or multiply, so wrapping once is the same)."""
    tmp2 = x[2] * F541 + x[6] * (F541 - F1847)
    tmp3 = x[2] * (F541 + F765) + x[6] * F541
    tmp0 = w16(x[0] + x[4]) << 13
    tmp1 = w16(x[0] - x[4]) << 13
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    a0, a1, a2, a3 = x[7], x[5], x[3], x[1]
    z3, z4 = w16(a0 + a2), w16(a1 + a3)
    z3p = z3 * (F1175 - F1961) + z4 * F1175
    z4p = z3 * F1175 + z4 * (F1175 - F390)
    o0 = a0 * (F298 - F899) - a3 * F899 + z3p
    o3 = -a0 * F899 + a3 * (F1501 - F899) + z4p
    o1 = a1 * (F2053 - F2562) - a2 * F2562 + z4p
    o2 = -a1 * F2562 + a2 * (F3072 - F2562) + z3p
    return [t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3]


def idct_blocks(coef: np.ndarray, q: np.ndarray) -> np.ndarray:
    """coef int16 [N, 64] natural order, q [64] -> [N, 8, 8] u8: libjpeg-turbo's x86 SIMD islow."""
    c = coef.astype(np.int64).reshape(-1, 8, 8)
    d = w16(c * q.astype(np.int64).reshape(8, 8))
    p1 = idct8([d[:, r, :] for r in range(8)])                         # per column, over rows
    ws = np.stack([sat(w32(v + (1 << 10)) >> 11, -32768, 32767) for v in p1], 1)      # [N, row, col]
    dc_only = ~np.any(c[:, 1:, :] != 0, axis=(1, 2))
    ws[dc_only] = w16(d[dc_only, 0, :] * 4)[:, None, :]
    p2 = idct8([ws[:, :, k] for k in range(8)])                        # per row, over columns
    out = np.stack([sat(sat(w32(v + (1 << 17)) >> 18, -32768, 32767), -128, 127) + 128 for v in p2], 2)
    return out.astype(np.uint8)


def plane(coefs: np.ndarray, q: np.ndarray, bw: int, bh: int) -> np.ndarray:
    b = idct_blocks(coefs.reshape(-1, 64), q).reshape(bh, bw, 8, 8)
    return b.transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8)


def upsample(c: np.ndarray, h: int, v: int, W: int, H: int) -> np.ndarray:
    """A chroma plane (its real dh x dw samples) -> H x W, as jdsample.c: fancy h2v1 / h1v2 / h2v2 with clamped edges,
    replication for h2 when dw <= 2."""
    c = c.astype(np.int32)
    dh, dw = c.shape
    y, x = np.arange(H)[:, None], np.arange(W)[None, :]
    rc, cc = y // v, x // h
    if h == 2 and dw <= 2 or (h == 1 and v == 1):
        return c[rc, cc]
    odd_x, odd_y = x & 1, y & 1
    ncol = np.where(odd_x == 1, np.minimum(cc + 1, dw - 1), np.maximum(cc - 1, 0))
    nrow = np.where(odd_y == 1, np.minimum(rc + 1, dh - 1), np.maximum(rc - 1, 0))
    if v == 1:
        return (3 * c[rc, cc] + c[rc, ncol] + np.where(odd_x == 1, 2, 1)) >> 2
    if h == 1:
        return (3 * c[rc, cc] + c[nrow, cc] + np.where(odd_y == 1, 2, 1)) >> 2
    s0 = 3 * c[rc, cc] + c[nrow, cc]
    s1 = 3 * c[rc, ncol] + c[nrow, ncol]
    return (3 * s0 + s1 + np.where(odd_x == 1, 7, 8)) >> 4


def model_decode(info: np.ndarray, quant: np.ndarray, coefs: np.ndarray) -> np.ndarray:
    W, H, nc, h0, v0, colour = (int(info[i]) for i in range(6))
    mcux, mcuy = int(info[7]), int(info[8])
    at = 0
    planes = []
    for c in range(nc):
        bw, bh = mcux * (h0 if c == 0 else 1), mcuy * (v0 if c == 0 else 1)
        planes.append(plane(coefs[at: at + bw * bh * 64], quant[c], bw, bh))
        at += bw * bh * 64
    Y = planes[0][:H, :W].astype(np.int32)
    if nc == 1:
        return np.repeat(Y[:, :, None], 3, 2).astype(np.uint8)
    dw, dh = -(-W // h0), -(-H // v0)
    cb, cr = (upsample(p[:dh, :dw], h0, v0, W, H) for p in planes[1:])
    if colour == 2:
        return np.stack([Y, cb, cr], 2).astype(np.uint8)
    cb, cr = cb - 128, cr - 128
    r = Y + ((91881 * cr + 32768) >> 16)
    g = Y + ((-46802 * cr - 22554 * cb + 32768) >> 16)
    b = Y + ((116130 * cb + 32768) >> 16)
    return np.clip(np.stack([r, g, b], 2), 0, 255).astype(np.uint8)


# --------------------------------------------------------------------------------------
# a baseline encoder of given quantised coefficients
# --------------------------------------------------------------------------------------
class _Bits:
    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def put(self, value: int, length: int):
        for i in range(length - 1, -1, -1):
            self.acc = (self.acc << 1) | ((value >> i) & 1)
            self.n += 1
            if self.n == 8:
                self.out.append(self.acc)
                if self.acc == 0xFF:
                    self.out.append(0)
                self.acc, self.n = 0, 0

    def flush(self):
        if self.n:
            self.put((1 << (8 - self.n)) - 1, 8 - self.n)


def _category(v: int) -> int:
    return int(abs(v)).bit_length()


def _table(symbols):
    """A fixed-length canonical table over the symbols used: (counts[16], values, {symbol: (code, length)})."""
    syms = sorted(set(symbols)) or [0]
    L = max(1, len(syms).bit_length())
    counts = [0] * 16
    counts[L - 1] = len(syms)
    return counts, syms, {s: (i, L) for i, s in enumerate(syms)}


def encode(blocks, quant, W: int, H: int, h0: int = 1, v0: int = 1, ids=(1, 2, 3), jfif: bool = True,
           adobe=None, restart: int = 0, q16: bool = False) -> bytes:
    """blocks: per component an int array [bh, bw, 64] of quantised coefficients in natural order over the
    MCU-padded component (the layout usdu_jpeg_decode_coefs writes); quant: per component 64 values, natural order.
    -> a baseline JPEG (SOF0, one interleaved scan, fixed-length Huffman tables per component)."""
    nc = len(blocks)
    hs = [h0 if c == 0 else 1 for c in range(nc)] if nc > 1 else [1]
    vs = [v0 if c == 0 else 1 for c in range(nc)] if nc > 1 else [1]
    mcuy, mcux = blocks[0].shape[0] // vs[0], blocks[0].shape[1] // hs[0]
    order = []                                         # (component, block) in scan order, with restarts
    for m in range(mcux * mcuy):
        my, mx = divmod(m, mcux)
        for c in range(nc):
            for yy in range(vs[c]):
                for xx in range(hs[c]):
                    order.append((m, c, blocks[c][my * vs[c] + yy, mx * hs[c] + xx]))
    # symbols per component
    dcs, acs = [[] for _ in range(nc)], [[] for _ in range(nc)]
    coded = []
    last, cur = [0] * nc, -1
    for m, c, blk in order:
        if m != cur:
            cur = m
            if restart and m % restart == 0:
                last = [0] * nc
        zz = [int(blk[ZIGZAG[k]]) for k in range(64)]
        diff = zz[0] - last[c]
        last[c] = zz[0]
        s = _category(diff)
        syms = [(0, s, diff)]
        run = 0
        for k in range(1, 64):
            if zz[k] == 0:
                run += 1
                continue
            while run > 15:
                syms.append((1, 0xF0, None))
                run -= 16
            syms.append((1, (run << 4) | _category(zz[k]), zz[k]))
            run = 0
        if run:
            syms.append((1, 0x00, None))
        for cls, sym, _ in syms:
            (dcs if cls == 0 else acs)[c].append(sym)
        coded.append((m, c, syms))
    tabs = [(_table(dcs[c]), _table(acs[c])) for c in range(nc)]
    bits = _Bits()
    scan = bytearray()
    prev_m, rst = 0, 0
    for m, c, syms in coded:
        if restart and m != prev_m and m % restart == 0:
            bits.flush()
            scan += bits.out + bytes([0xFF, 0xD0 + rst])
            rst = (rst + 1) & 7
            bits = _Bits()
        prev_m = m
        for cls, sym, val in syms:
            code, length = tabs[c][cls][2][sym]
            bits.put(code, length)
            s = sym & 15 if cls else sym
            if s:
                bits.put(val if val >= 0 else val + (1 << s) - 1, s)
    bits.flush()
    scan += bits.out

    def seg(marker, body):
        return bytes([0xFF, marker]) + (len(body) + 2).to_bytes(2, "big") + bytes(body)

    out = bytearray(b"\xFF\xD8")
    if jfif:
        out += seg(0xE0, b"JFIF\0\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    if adobe is not None:
        out += seg(0xEE, b"Adobe\x00\x64\x00\x00\x00\x00" + bytes([adobe]))
    for c in range(nc):
        qz = [int(quant[c][ZIGZAG[k]]) for k in range(64)]
        out += seg(0xDB, bytes([(0x10 if q16 else 0) | c]) +
                   (b"".join(v.to_bytes(2, "big") for v in qz) if q16 else bytes(qz)))
    sof = bytearray([8]) + H.to_bytes(2, "big") + W.to_bytes(2, "big") + bytes([nc])
    for c in range(nc):
        sof += bytes([ids[c], (hs[c] << 4) | vs[c], c])
    out += seg(0xC0, sof)
    for c in range(nc):
        for cls in (0, 1):
            counts, vals, _ = tabs[c][cls]
            out += seg(0xC4, bytes([(cls << 4) | c] + counts + vals))
    if restart:
        out += seg(0xDD, restart.to_bytes(2, "big"))
    sos = bytearray([nc])
    for c in range(nc):
        sos += bytes([ids[c], (c << 4) | c])
    out += seg(0xDA, sos + b"\x00\x3F\x00")
    out += scan + b"\xFF\xD9"
    return bytes(out)


def random_blocks(rng, W: int, H: int, nc: int, h0: int, v0: int, scale: float, dc_range=(-60, 60)):
    """Random quantised coefficients for a W x H frame: smooth-ish (decaying AC) by default; scale sets the AC size."""
    hs, vs = (h0, 1, 1), (v0, 1, 1)
    if nc == 1:
        hs, vs = (1,), (1,)
    mcux, mcuy = -(-W // (8 * hs[0])), -(-H // (8 * vs[0]))
    out = []
    decay = np.exp(-np.add.outer(np.arange(8), np.arange(8)).reshape(64) / 3.0)
    for c in range(nc):
        shape = (mcuy * vs[c], mcux * hs[c], 64)
        b = np.rint(rng.standard_normal(shape) * scale * decay).astype(np.int64)
        b[..., 0] = rng.integers(dc_range[0], dc_range[1] + 1, shape[:2])
        out.append(b)
    return out
