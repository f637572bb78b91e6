"""The HTTP tile worker's PNG, stated in numpy -- TEST INFRASTRUCTURE ONLY, the byte-exact reference of the GPU encoder
(usdu_png_encode_u8, include/usdu_b200.h).  Pillow's level-0 PNG of an RGB frame is its framing (a function of the shape
alone, http_worker.png_layout) filled with the filtered stream R and the checksums.  R is per row one filter byte and the
filtered row; the filter follows Pillow's choice without `optimize`: for None (0), Up (2), Sub (1), Paeth (4) in that
order, the sum over the filtered bytes v of min(v, 256 - v), the previous row being the previous RAW row (zeros above
the first); the first candidate with the smallest sum wins."""
from __future__ import annotations

import zlib

import numpy as np

ORDER = (0, 2, 1, 4)          # the order Pillow tries the filters in


def _paeth(a: np.ndarray, b: np.ndarray, c: np.ndarray) -> np.ndarray:
    a, b, c = (x.astype(np.int32) for x in (a, b, c))
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c)).astype(np.uint8)


def filter_candidates(frame_u8: np.ndarray) -> dict:
    """{filter type: [H, W*C] u8 filtered rows} for the four filters Pillow tries."""
    H, W, C = frame_u8.shape
    x = np.ascontiguousarray(frame_u8, dtype=np.uint8).reshape(H, W * C)
    up = np.zeros_like(x)
    up[1:] = x[:-1]
    left = np.zeros_like(x)
    left[:, C:] = x[:, :-C]
    upleft = np.zeros_like(x)
    upleft[:, C:] = up[:, :-C]
    return {0: x, 2: x - up, 1: x - left, 4: x - _paeth(left, up, upleft)}


def filter_choice(frame_u8: np.ndarray) -> np.ndarray:
    """[H] filter type Pillow writes for each row."""
    cand = filter_candidates(frame_u8)
    cost = np.stack([np.minimum(cand[f], 256 - cand[f].astype(np.int32)).sum(1, dtype=np.int64) for f in ORDER])
    return np.asarray(ORDER, np.uint8)[np.argmin(cost, 0)]      # argmin: the first of equal sums


def filtered_stream(frame_u8: np.ndarray) -> bytes:
    """R: per row the chosen filter byte, then the filtered row."""
    cand = filter_candidates(frame_u8)
    choice = filter_choice(frame_u8)
    rows = np.stack([cand[int(f)][r] for r, f in enumerate(choice)]) if len(choice) else np.zeros((0, 0), np.uint8)
    return np.concatenate([choice[:, None], rows], 1).tobytes()


def host_encode(frame_u8: np.ndarray, layout) -> bytes:
    """The whole encoder on the host from the tables the kernel consumes: the template, R spliced in by the runs, the
    Adler-32 of R at its four offsets, then every IDAT chunk's CRC-32 over its type and data."""
    raw = filtered_stream(frame_u8)
    out = bytearray(layout.template)
    for f, s, n in layout.runs.tolist():
        out[f: f + n] = raw[s: s + n]
    for i, p in enumerate(layout.adler_at):
        out[p] = zlib.adler32(raw).to_bytes(4, "big")[i]
    for off, n in layout.chunks.tolist():
        out[off + 8 + n: off + 12 + n] = zlib.crc32(bytes(out[off + 4: off + 8 + n])).to_bytes(4, "big")
    return bytes(out)


def rechunk(data: bytes, cuts) -> bytes:
    """The same PNG with its zlib stream re-cut into IDAT chunks at the stream offsets `cuts` (one chunk when empty):
    a valid file whose chunk boundaries fall where Pillow's never do -- inside the Adler trailer, inside a stored-block
    header, or chunks longer than one CRC span of the kernel."""
    pos, stream, head, tail = 8, b"", None, None
    while pos < len(data):
        n, kind = int.from_bytes(data[pos:pos + 4], "big"), data[pos + 4:pos + 8]
        if kind == b"IDAT":
            head = pos if head is None else head
            stream += data[pos + 8:pos + 8 + n]
        elif head is not None and tail is None:
            tail = pos
        pos += 12 + n
    edges = [0] + sorted(c for c in cuts if 0 < c < len(stream)) + [len(stream)]
    body = b"".join(len(stream[a:b]).to_bytes(4, "big") + b"IDAT" + stream[a:b]
                    + zlib.crc32(b"IDAT" + stream[a:b]).to_bytes(4, "big") for a, b in zip(edges, edges[1:]))
    return data[:head] + body + data[tail:]


def split_cuts(data: bytes):
    """Stream offsets that cut the Adler trailer in two and every stored-block header after its first two bytes."""
    pos, stream = 8, b""
    while pos < len(data):
        n, kind = int.from_bytes(data[pos:pos + 4], "big"), data[pos + 4:pos + 8]
        if kind == b"IDAT":
            stream += data[pos + 8:pos + 8 + n]
        pos += 12 + n
    cuts, p = [len(stream) - 2], 2
    while True:
        cuts.append(p + 2)
        final, ln = stream[p] & 1, int.from_bytes(stream[p + 1:p + 3], "little")
        p += 5 + ln
        if final:
            return cuts
