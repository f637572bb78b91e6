"""The collector worker's PNG, stated in numpy -- TEST INFRASTRUCTURE ONLY, the byte-exact reference of the GPU encoder
(usdu_png_base64_u8, include/usdu_b200.h).  A stored (deflate level 0), filter-None PNG with a fixed layout; the
checksums come from zlib.crc32 / zlib.adler32."""
from __future__ import annotations

import base64
import zlib

import numpy as np

PNG_STORED_BLOCK = 65535
PNG_COLOUR_TYPE = {2: 4, 3: 2, 4: 6}     # LA, RGB, RGBA: the modes Image.fromarray gives (utils/image.py:8-10)


def _png_chunk(kind: bytes, data: bytes) -> bytes:
    return len(data).to_bytes(4, "big") + kind + data + zlib.crc32(kind + data).to_bytes(4, "big")


def png_raw_stream(frame_u8: np.ndarray) -> bytes:
    """R: per row a filter byte 0, then the row's W*C bytes."""
    H = frame_u8.shape[0]
    rows = np.ascontiguousarray(frame_u8, dtype=np.uint8).reshape(H, -1)
    return np.concatenate([np.zeros((H, 1), np.uint8), rows], 1).tobytes()


def png_stored(frame_u8: np.ndarray) -> bytes:
    """The PNG bytes of one u8 frame [H, W, C], C in {2, 3, 4}: signature, IHDR, R cut into stored deflate blocks of
    65535 bytes with block k alone in IDAT chunk k (chunk 0 starts with the zlib header 78 01), one IDAT chunk holding
    the big-endian Adler-32 of R, IEND.  C = 1 or any other C raises TypeError, as Image.fromarray does."""
    if frame_u8.ndim != 3 or frame_u8.shape[2] not in PNG_COLOUR_TYPE:
        raise TypeError(f"cannot write a PNG of a frame of shape {tuple(frame_u8.shape)}")
    H, W, C = frame_u8.shape
    raw = png_raw_stream(frame_u8)
    out = [b"\x89PNG\r\n\x1a\n",
           _png_chunk(b"IHDR", W.to_bytes(4, "big") + H.to_bytes(4, "big") + bytes([8, PNG_COLOUR_TYPE[C], 0, 0, 0]))]
    nblk = -(-len(raw) // PNG_STORED_BLOCK)
    for k in range(nblk):
        block = raw[k * PNG_STORED_BLOCK:(k + 1) * PNG_STORED_BLOCK]
        L = len(block)
        head = (b"\x78\x01" if k == 0 else b"") + bytes([1 if k == nblk - 1 else 0])
        out.append(_png_chunk(b"IDAT", head + L.to_bytes(2, "little") + (L ^ 0xFFFF).to_bytes(2, "little") + block))
    out.append(_png_chunk(b"IDAT", zlib.adler32(raw).to_bytes(4, "big")))
    out.append(_png_chunk(b"IEND", b""))
    return b"".join(out)


def png_stored_b64(frame_u8: np.ndarray) -> bytes:
    """base64 (standard alphabet, '=' padding, no line breaks) of png_stored(frame_u8), as ASCII bytes."""
    return base64.b64encode(png_stored(frame_u8))


# --------------------------------------------------------------------------------------
# the T0 test denoiser (BASELINE.md section 3): same callable on both sides of a parity test
# --------------------------------------------------------------------------------------
def t0_noise(seed: int, shape: Tuple[int, ...]) -> np.ndarray:
    """Seeded uniform noise; torch's CPU generator so that it is identical everywhere."""
    import torch
    g = torch.Generator().manual_seed(int(seed))
    return torch.rand(shape, generator=g, dtype=torch.float32).numpy()


def make_t0_denoiser(seed: int, denoise: float) -> DenoiseFn:
    """x' = clamp(x*(1-d) + noise*d, 0, 1); every step individually rounded in fp32 so
    that CPU and GPU agree bit-for-bit.  The same seed is used for every tile
    (upscale/tile_ops.py:430-431, single_gpu.py:53-55)."""
    d = np.float32(denoise)
    omd = np.float32(1.0) - d
    cache = {}

    def fn(tile: np.ndarray, t: TilePlan) -> np.ndarray:
        if tile.shape not in cache:
            cache[tile.shape] = t0_noise(seed, tile.shape)
        y = tile.astype(np.float32) * omd + cache[tile.shape] * d
        return np.clip(y, np.float32(0), np.float32(1))

    return fn
