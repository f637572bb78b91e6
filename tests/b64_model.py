"""numpy models of the collector master's device checks (csrc/usdu_b64.cu, usdu_b64_png_check): the base64 verdict and
decode, and the table the walk, block-sum and finish passes leave; plus the base64 corpus the tests run them on."""
import base64
import binascii
import io
import zlib

import numpy as np
from PIL import Image

from __graft_entry__ import load_package

load_package()
from comfyui_distributed_b200 import _native as nat  # noqa: E402
from comfyui_distributed_b200 import http_collector as hc  # noqa: E402

ALPHABET = b"ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/"
LUT = np.full(256, 65, np.int64)
LUT[np.frombuffer(ALPHABET, np.uint8)] = np.arange(64)
LUT[ord("=")] = 64
CB = nat.B64_HEAD_WORDS
BB = CB + 4 * nat.B64_MAX_CHUNKS
PB = BB + 4 * nat.B64_MAX_BLOCKS
ADLER = 65521


def interpreter(text):
    """What this interpreter's b64decode(validate=True) makes of `text`: the bytes, or None when it refuses."""
    try:
        return base64.b64decode(text, validate=True)
    except (binascii.Error, ValueError):
        return None


def b64_words(t: bytes):
    """-> (a byte outside the alphabet, first '=' index or n, index after the last other byte or 0, every quad decoded
    with '=' and refused bytes as 0): pass 1's reductions and output."""
    a = LUT[np.frombuffer(t, np.uint8)]
    n = a.size
    eq, data = np.flatnonzero(a == 64), np.flatnonzero(a < 64)
    first = int(eq[0]) if eq.size else n
    end = int(data[-1]) + 1 if data.size else 0
    v = np.zeros((n + 3) // 4 * 4, np.int64)
    v[:n] = np.where(a < 64, a, 0)
    t24 = (v[0::4] << 18) | (v[1::4] << 12) | (v[2::4] << 6) | v[3::4]
    out = np.stack([t24 >> 16, (t24 >> 8) & 255, t24 & 255], 1).astype(np.uint8).reshape(-1)
    return bool((a == 65).any()), first, end, out


def b64_length(n: int, bad: bool, first_pad: int, data_end: int) -> int:
    """The decoded length of an n-byte text that Python 3.12's b64decode(validate=True) accepts, else -1, from three
    facts about the text: a byte outside [A-Za-z0-9+/=], the index of the first '=' (n if none), the index after the
    last other byte (0 if none).  Accepted: no '=' first and none followed by data, and d = first_pad data characters
    with p = n - d pads where d % 4 == 0 (any p), or d % 4 == 2 and p == 2, or d % 4 == 3 and p == 1.  The device
    computes the same ([3] of usdu_b64_png_check's table, walk_kernel)."""
    q, p = first_pad % 4, n - first_pad
    if bad or data_end > first_pad or (n > 0 and first_pad == 0):
        return -1
    if q == 0 or (q == 2 and p == 2) or (q == 3 and p == 1):
        return 3 * (first_pad // 4) + (q - 1 if q else 0)
    return -1


def b64_model(text):
    """The model's verdict and bytes for a str or bytes text: None when refused."""
    if isinstance(text, str):
        try:
            text = text.encode("ascii")
        except UnicodeEncodeError:
            return None
    bad, first, end, out = b64_words(text)
    m = b64_length(len(text), bad, first, end)
    return None if m < 0 else out[:m].tobytes()


def table_model(text: bytes):
    """-> (the table usdu_b64_png_check leaves for `text`, its decoded bytes), every word the passes write (the other
    words of the chunk and block areas stay 0 here; on the device they are not written)."""
    n = len(text)
    bad, first, end, out = b64_words(text)
    tab = np.zeros(nat.B64_TABLE_WORDS, np.int64)
    head = tab[:CB]
    m = b64_length(n, bad, first, end)
    head[:4] = [int(bad), first, end, m]
    head[[6, 7, 11, 12, 13]] = -1
    png = out[:max(m, 0)].tobytes()
    np_ = min(max(m, 0), nat.B64_PREFIX_BYTES)
    tab[PB:].view(np.uint8)[:np_] = np.frombuffer(png[:np_], np.uint8)
    if m < 8:
        return tab, png
    be = lambda p: int.from_bytes(png[p:p + 4], "big")
    ch = tab[CB:BB].reshape(-1, 4)
    pos, stream, nc, idat0, nidat, code = 8, 0, 0, -1, 0, nat.B64_CHUNKS_FULL
    while nc < nat.B64_MAX_CHUNKS:
        if pos + 8 > m:
            code = nat.B64_CHUNKS_SHORT
            break
        ln, ty = be(pos), be(pos + 4)
        ch[nc] = [pos, ln, ty, -1]
        nc += 1
        body = pos + 8
        if ln > 0x7FFFFFFF or body + ln + 4 > m:
            code = nat.B64_CHUNKS_PAST_END
            break
        if nc == 1 and ty == 0x49484452 and ln == 13:
            W, H, depth, color = be(body), be(body + 4), png[body + 8], png[body + 9]
            C = {0: 1, 2: 3, 4: 2, 6: 4}.get(color, 0)
            if depth == 8 and C and W >= 1 and H >= 1 and W * C <= nat.PNG_MAX_ROW_BYTES:
                head[6] = H * (1 + W * C)
        if ty == 0x49444154:
            idat0 = nc - 1 if idat0 < 0 else idat0
            ch[nc - 1, 3] = stream
            stream += ln
            nidat += 1
        elif nidat:
            code = nat.B64_CHUNKS_AFTER_IDAT
            break
        elif ty == 0x49454E44:
            code = nat.B64_CHUNKS_IEND
            break
        pos = body + ln + 4
    head[4], head[5], head[8], head[16], head[17] = nc, code, stream, idat0, nidat
    if code != nat.B64_CHUNKS_AFTER_IDAT:
        return tab, png
    pieces = ch[idat0: idat0 + nidat]
    S = b"".join(png[p + 8: p + 8 + ln] for p, ln, _, _ in pieces.tolist())
    bl = tab[BB:PB].reshape(-1, 4)
    nb, raw, bcode = 0, 0, nat.B64_BLOCKS_FULL
    spans = []                                   # (stream offset, length) of each block's data
    if stream < 2:
        bcode = nat.B64_BLOCKS_SHORT
    else:
        cmf, flg = S[0], S[1]
        head[7] = cmf | (flg << 8)
        if (cmf & 0x0F) != 8 or (cmf >> 4) > 7 or (cmf * 256 + flg) % 31 != 0 or (flg & 0x20):
            bcode = nat.B64_BLOCKS_ZLIB
        else:
            s = 2
            while nb < nat.B64_MAX_BLOCKS:
                if s + 1 > stream:
                    bcode = nat.B64_BLOCKS_SHORT
                    break
                hb = S[s]
                bl[nb] = [s, hb, raw, 0]
                if (hb >> 1) & 3:
                    nb += 1
                    bcode = nat.B64_BLOCKS_COMPRESSED
                    break
                if s + 5 > stream:
                    bcode = nat.B64_BLOCKS_SHORT
                    break
                ln, nln = S[s + 1] | (S[s + 2] << 8), S[s + 3] | (S[s + 4] << 8)
                bl[nb, 1] = hb | (ln << 8) | (nln << 24)
                nb += 1
                if ln ^ nln != 0xFFFF:
                    bcode = nat.B64_BLOCKS_LEN
                    break
                s += 5
                if s + ln > stream:
                    bcode = nat.B64_BLOCKS_SHORT
                    break
                spans.append((s, ln))
                raw += ln
                s += ln
                if hb & 1:
                    bcode = nat.B64_BLOCKS_FINAL
                    head[15] = s
                    if s + 4 <= stream:
                        head[11] = int.from_bytes(S[s:s + 4], "big")
                    break
    head[9], head[10], head[14] = nb, bcode, raw
    if bcode != nat.B64_BLOCKS_FINAL:
        return tab, png
    for b, (s, ln) in enumerate(spans):
        d = np.frombuffer(S[s:s + ln], np.uint8).astype(np.int64)
        s1 = int(d.sum()) % ADLER
        s2 = int(((ln - np.arange(ln)) * d).sum()) % ADLER
        bl[b, 3] = s1 | (s2 << 32)
    D = b"".join(S[s:s + ln] for s, ln in spans)
    head[12] = zlib.adler32(D)
    if head[6] > 0 and raw >= head[6]:
        W, H, color = be(16), be(20), png[25]
        rowlen = 1 + W * {0: 1, 2: 3, 4: 2, 6: 4}[color]
        head[13] = int(np.frombuffer(D, np.uint8)[: H * rowlen: rowlen].max())
    return tab, png


def used_words(tab: np.ndarray) -> np.ndarray:
    """The words of a table that the passes write for its text (head, recorded entries, prefix)."""
    head = tab[:CB]
    nc, nb, m = int(head[4]), int(head[9]), int(head[3])
    pre = tab[PB:].view(np.uint8)[:min(max(m, 0), nat.B64_PREFIX_BYTES)]
    return np.concatenate([head, tab[CB: CB + 4 * nc], tab[BB: BB + 4 * nb], pre.astype(np.int64)])


def check_model(text: bytes):
    """The split parse_png, modelled: the device table, then the host walk.  -> (PNG bytes, PngInfo) or ValueError
    with png_of_payload's message; HostParse falls back to parse_png as the route does."""
    tab, png = table_model(text)
    m = int(tab[3])
    if m < 0:
        raise ValueError(hc.NOT_BASE64)
    if m == 0:
        raise ValueError(hc.EMPTY_PNG)
    try:
        return png, hc.check_png_tables(tab, m)
    except hc.HostParse:
        try:
            return png, hc.parse_png(png)
        except Exception as exc:
            raise ValueError(f"{hc.PNG_FAILED}{exc}") from exc
    except Exception as exc:
        raise ValueError(f"{hc.PNG_FAILED}{exc}") from exc


# --------------------------------------------------------------------------------------
# the base64 corpus
# --------------------------------------------------------------------------------------
def corpus():
    """(name, text) -- str or bytes: every data length mod 4 with 0..3 '=', '=' at every position of the last two
    quads, each byte value at the start, middle and end of a valid text, non-ASCII str, empty text, whitespace, valid
    texts of assorted lengths."""
    rng = np.random.default_rng(0)
    out = [("empty", ""), ("empty_bytes", b"")]
    for n in range(0, 13):
        d = "".join(chr(ALPHABET[i]) for i in rng.integers(0, 64, n))
        for k in range(4):
            out.append((f"len{n}_pad{k}", d + "=" * k))
    for n in (6, 7, 8, 9):                       # 8, 12 characters with 0, 1 or 2 pads
        t = base64.b64encode(bytes(rng.integers(0, 256, n).tolist())).decode()
        for i in range(max(0, len(t) - 8), len(t)):
            out.append((f"eq_at_{n}_{i}", t[:i] + "=" + t[i + 1:]))
            out.append((f"eq_ins_{n}_{i}", t[:i] + "=" + t[i:]))
        out.append((f"eq_tail_{n}", t + "="))
        out.append((f"eq_tail3_{n}", t + "==="))
    good = base64.b64encode(bytes(rng.integers(0, 256, 30).tolist()))
    for v in range(256):
        for where, i in (("start", 0), ("mid", len(good) // 2), ("end", len(good))):
            out.append((f"byte{v}_{where}", good[:i] + bytes([v]) + good[i:]))
    out += [("non_ascii", good.decode()[:8] + "é" + good.decode()[8:]), ("non_ascii_end", good.decode() + "€"),
            ("space_inside", good.decode()[:8] + " " + good.decode()[8:]),
            ("newline_inside", good.decode()[:12] + "\n" + good.decode()[12:]), ("tab", "\t" + good.decode()),
            ("leading_pad", "=QUJD"), ("gap_pad", "QU=D"), ("short_pad", "QQ="), ("short", "QUI"), ("excess", "QQ==="),
            ("after_quad", "QUJD="), ("after_quad3", "QUJD==="), ("trailing_bits", "QR=="), ("all_pad", "===="),
            ("pad_then_data", "QUJD=QUJD")]
    for n in (1, 2, 3, 47, 48, 49, 1000, 4099, 65537):
        t = base64.b64encode(bytes(rng.integers(0, 256, n).tolist()))
        out.append((f"valid_{n}", t))
        out.append((f"valid_{n}_trailing_bits", t[:-3] + b"B==" if t.endswith(b"==") else t))
    return out


def png_of(arr: np.ndarray, level: int) -> bytes:
    bio = io.BytesIO()
    Image.fromarray(arr).save(bio, format="PNG", compress_level=level)
    return bio.getvalue()
