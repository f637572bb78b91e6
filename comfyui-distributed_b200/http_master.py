"""Master side of the reference's static-mode HTTP protocol: its five USDU routes (api/usdu_routes.py:16-228), its tile
queue and time-outs (upscale/job_store.py, job_state.py, job_timeout.py), and the master's own share of the tiles plus
the final composite (upscale/modes/static.py:371-570) on this GPU.

The routes and the job store live on ComfyUI's server event loop, as in the reference; the master's prompt thread
reaches them with `run_coroutine_threadsafe`.  A route handler never decodes pixels: it validates each posted PNG on the
host (`parse_png`, which refuses what PIL's open().convert("RGB") refuses) and keeps the raw bytes, the segment table of
the filtered stream inside them and the tile's metadata.  A palette, 1/2/4/16-bit or interlaced PNG, which parse_png
refuses, is validated and inflated by `parse_png_general` instead, and its filtered stream kept; a baseline JPEG is
parsed and Huffman-decoded by `parse_jpeg` (csrc/usdu_jpeg.cpp), and its coefficients kept.  The master uploads each
drained batch of tiles and decodes it on a side stream (csrc/usdu_png_decode.cu) while it waits for more, and
composites all kept worker tiles in the reference's order with the existing blend kernels.

Differences from the reference (INTEGRATION.md, "A master for HTTP workers"):
* no "busy" probe of a timed-out worker (job_timeout.py:82-105 reads the orchestrator's gpu_config.json): a worker whose
  heartbeat is older than COMFYUI_HEARTBEAT_TIMEOUT has its incomplete tiles re-queued;
* PNGs with filtered rows over PNG_MAX_ROW_BYTES answer 400;
* x, y, extracted_width and extracted_height must equal the plan's window of tile_idx, and the PNG must be at the tile's
  processing size, else 400;
* a job is cleaned up in a `finally` around the whole master run, including an interrupt before the collect phase.
"""
from __future__ import annotations

import asyncio
import io
import json
import os
import struct
import time
import warnings
import zlib
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np

from ._native import PNG_MAX_ROW_BYTES

PNG_SIGNATURE = b"\x89PNG\r\n\x1a\n"
CHANNELS = {0: 1, 2: 3, 4: 2, 6: 4}          # PNG colour type -> samples per pixel (8-bit)
REQUEST_WAIT = 0.1                            # request_image's wait on an empty queue (usdu_routes.py:195)
MASTER_EMPTY_POLLS = 2                        # static.py:404
COLLECT_POLL = 0.1                            # static.py:366


def max_payload_size() -> int:
    return int(os.environ.get("COMFYUI_MAX_PAYLOAD_SIZE", str(50 * 1024 * 1024)))


def heartbeat_timeout() -> float:
    return float(os.environ.get("COMFYUI_HEARTBEAT_TIMEOUT", "60"))


def heartbeat_interval() -> float:
    return float(os.environ.get("COMFYUI_HEARTBEAT_INTERVAL", "10"))


# --------------------------------------------------------------------------------------
# PNG validation and the segment table of the filtered stream
# --------------------------------------------------------------------------------------
class PngInfo:
    """A validated 8-bit, non-interlaced PNG.  The filtered stream R (per row a filter byte, then W*C bytes) is the
    concatenation, in order, of data[src:src + length] for (src, raw start) in `segs` (each runs to the next raw start,
    the last to |R|), or, when the stream had compressed blocks, `inflated` itself (segs = [(0, 0)]).  `idat` lists the
    (file offset, data length) of every IDAT chunk, `trailer` the file offsets of the four Adler-32 bytes (stored blocks
    only, else None): the framing http_worker.png_layout reads."""
    __slots__ = ("W", "H", "C", "segs", "inflated", "idat", "trailer")

    def __init__(self, W, H, C, segs, inflated=None, idat=(), trailer=None):
        self.W, self.H, self.C, self.segs, self.inflated = W, H, C, segs, inflated
        self.idat, self.trailer = list(idat), trailer

    @property
    def raw_len(self) -> int:
        return self.H * (1 + self.W * self.C)


class UnsupportedPng(ValueError):
    """parse_png's refusal of a bit depth, colour type or interlace method it does not take: parse_png_general decides
    such a file."""


def parse_png(data: bytes) -> PngInfo:
    """Validate `data` as PIL's open().convert("RGB") would read it and return its segment table.  ValueError with the
    reason otherwise (UnsupportedPng for the IHDR's depth, colour type or interlace).  Checks: signature; IHDR (8-bit,
    colour type 0/2/4/6, no interlace); chunk bounds; the CRC-32 of every chunk before the first IDAT (PIL checks those,
    not IDAT's or later ones); the zlib header; the stored-block LEN/NLEN chain (any compressed block: the stream is
    inflated with zlib); the Adler-32; the IDAT length against the image size; every filter byte <= 4; rows of at most
    PNG_MAX_ROW_BYTES (what the decode kernel takes)."""
    (W, H, C), idat, _ = _walk_chunks(data, _ihdr_8bit)
    raw_len = H * (1 + W * C)
    stream = _IdatStream(data, idat)
    segs, inflated, trailer = _stored_segments(stream, raw_len)
    info = PngInfo(W, H, C, segs, inflated, [(off - 8, ln) for off, ln in idat], trailer)
    _check_filters(info, data)
    return info


def _ihdr_8bit(W, H, depth, color, comp, filt, interlace):
    if depth != 8 or color not in CHANNELS:
        raise UnsupportedPng(f"unsupported PNG: bit depth {depth}, colour type {color}")
    if comp != 0 or filt != 0:
        raise ValueError("unknown compression or filter method")
    if interlace != 0:
        raise UnsupportedPng("unsupported PNG: interlaced")
    if W * CHANNELS[color] > PNG_MAX_ROW_BYTES:
        raise ValueError(f"unsupported PNG: rows of {W * CHANNELS[color]} bytes (at most {PNG_MAX_ROW_BYTES})")
    return W, H, CHANNELS[color]


def _walk_chunks(data: bytes, on_ihdr, keep=()):
    """The chunk walk both parses share: signature, chunk bounds, IHDR first (its fields go to `on_ihdr`, which raises
    or returns what the caller keeps of them), the CRC-32 of every chunk before the first IDAT, consecutive IDATs, a
    chunk after them.  -> (on_ihdr's result, (data offset, length) of every IDAT chunk, [(type, data)] of the chunks
    before the first IDAT whose type is in `keep`, in file order)."""
    mv = memoryview(data)
    n = len(data)
    if n < 8 or data[:8] != PNG_SIGNATURE:
        raise ValueError("not a PNG file")
    pos = 8
    ihdr = None
    idat: List[Tuple[int, int]] = []             # (file offset, length) of every IDAT chunk's data
    kept = []
    while True:
        if pos + 8 > n:
            raise ValueError("truncated PNG (chunk header)")
        length, ctype = struct.unpack_from(">I4s", data, pos)
        body = pos + 8
        if length > 0x7FFFFFFF or body + length + 4 > n:
            raise ValueError(f"truncated PNG ({ctype!r} chunk runs past the end)")
        if ihdr is None:
            if ctype != b"IHDR" or length != 13:
                raise ValueError("first chunk is not IHDR")
        if not idat and ctype != b"IDAT":
            crc, = struct.unpack_from(">I", data, body + length)
            if zlib.crc32(mv[pos + 4: body + length]) != crc:
                raise ValueError(f"bad CRC in {ctype.decode('latin-1')}")
        if ctype == b"IHDR":
            if ihdr is not None:
                raise ValueError("second IHDR")
            W, H, depth, color, comp, filt, interlace = struct.unpack_from(">IIBBBBB", data, body)
            if W == 0 or H == 0 or W > 0x7FFFFFFF or H > 0x7FFFFFFF:
                raise ValueError("bad image size")
            ihdr = on_ihdr(W, H, depth, color, comp, filt, interlace)
        elif ctype == b"IDAT":
            if idat and idat[-1][0] + idat[-1][1] + 4 != pos:
                raise ValueError("IDAT chunks are not consecutive")
            idat.append((body, length))
        elif idat:
            break                                 # the image data ends at the first chunk after the IDATs
        elif ctype == b"IEND":
            raise ValueError("no IDAT chunk")
        elif ctype in keep:
            kept.append((ctype, bytes(mv[body: body + length])))
        pos = body + length + 4
    return ihdr, idat, kept


# --------------------------------------------------------------------------------------
# every other PNG PIL opens: palette, 1/2/4/16-bit, Adam7 (csrc/usdu_png_decode.cu, general entry)
# --------------------------------------------------------------------------------------
GENERAL_CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}             # colour type -> samples per pixel
GENERAL_DEPTHS = {0: (1, 2, 4, 8, 16), 2: (8, 16), 3: (1, 2, 4, 8), 4: (8, 16), 6: (8, 16)}
ADAM7 = ((0, 0, 8, 8), (4, 0, 8, 8), (0, 4, 4, 8), (2, 0, 4, 4), (0, 2, 2, 4), (1, 0, 2, 2), (0, 1, 1, 2))


class PngGeneral:
    """A validated PNG of any colour type and bit depth, interlaced or not.  `inflated` is its filtered stream R: per
    pass (one, or Adam7's seven back to back; a pass with no columns or rows has no bytes), per row a filter byte and
    row_bytes(pass width) bytes.  `palette`: 768 bytes (PLTE's entries, then zeros) for colour type 3, else None."""
    __slots__ = ("W", "H", "color", "depth", "interlace", "palette", "inflated")

    def __init__(self, W, H, color, depth, interlace, palette=None, inflated=b""):
        self.W, self.H, self.color, self.depth, self.interlace = W, H, color, depth, interlace
        self.palette, self.inflated = palette, inflated

    @property
    def C(self) -> int:
        return GENERAL_CHANNELS[self.color]

    @property
    def bpp(self) -> int:
        """Bytes of a PNG filter unit: max(1, depth * C / 8)."""
        return max(1, self.depth * self.C // 8)

    def row_bytes(self, w: int) -> int:
        return (w * self.depth * self.C + 7) // 8

    def passes(self) -> List[Tuple[int, int, int, int, int, int, int]]:
        """-> (x0, y0, dx, dy, pass width, pass height, offset in R) of every non-empty pass."""
        out, at = [], 0
        for x0, y0, dx, dy in (ADAM7 if self.interlace else ((0, 0, 1, 1),)):
            pw, ph = max(0, (self.W - x0 + dx - 1) // dx), max(0, (self.H - y0 + dy - 1) // dy)
            if pw and ph:
                out.append((x0, y0, dx, dy, pw, ph, at))
                at += ph * (1 + self.row_bytes(pw))
        return out

    @property
    def raw_len(self) -> int:
        return sum(ph * (1 + self.row_bytes(pw)) for _, _, _, _, pw, ph, _ in self.passes())


def _ihdr_general(W, H, depth, color, comp, filt, interlace):
    # PIL reads no compression method and takes any non-zero interlace byte as Adam7
    if depth not in GENERAL_DEPTHS.get(color, ()):
        raise ValueError(f"unsupported PNG: bit depth {depth}, colour type {color}")
    if filt != 0:
        raise ValueError("unknown filter method")
    n = (W * depth * GENERAL_CHANNELS[color] + 7) // 8
    if n > PNG_MAX_ROW_BYTES:
        raise ValueError(f"unsupported PNG: rows of {n} bytes (at most {PNG_MAX_ROW_BYTES})")
    return W, H, depth, color, int(interlace != 0)


def parse_png_general(data: bytes) -> PngGeneral:
    """Validate `data` as PIL's open().convert("RGB") reads any PNG and return it with its inflated filtered stream:
    parse_png's chunk walk and CRC rule; every (colour type, depth) the PNG spec allows; PLTE (at most 256 entries, any
    length) and tRNS (grey needs 2 bytes, RGB 6) as PIL reads them; the zlib stream inflated to its end, its Adler-32
    included; every filter byte <= 4; filtered rows of at most PNG_MAX_ROW_BYTES.  ValueError with the reason
    otherwise.  As with parse_png, a stream that ends before the image does, or a bad Adler-32 after a later IDAT
    chunk, is refused although PIL, which stops reading once the last row is decoded, may take some such files."""
    (W, H, depth, color, interlace), idat, kept = _walk_chunks(data, _ihdr_general, (b"PLTE", b"tRNS"))
    palette = None
    for ctype, body in kept:
        if ctype == b"PLTE" and color == 3:
            if len(body) // 3 > 256:
                raise ValueError("invalid palette size")
            palette = body[:len(body) // 3 * 3]
        elif ctype == b"tRNS" and len(body) < {0: 2, 2: 6}.get(color, 0):
            raise ValueError("tRNS chunk too short")
    if color == 3:
        palette = (palette or b"").ljust(768, b"\0")
    info = PngGeneral(W, H, color, depth, interlace, palette)
    st = _IdatStream(data, idat)
    hdr = st.read(0, 2)
    cmf, flg = hdr[0], hdr[1]
    if (cmf & 0x0F) != 8 or (cmf >> 4) > 7 or (cmf * 256 + flg) % 31 != 0 or (flg & 0x20):
        raise ValueError("bad zlib header")
    d = zlib.decompressobj()
    try:
        out = d.decompress(st.joined(), info.raw_len)
        while not d.eof:                          # the rest up to the stream's end, its Adler-32 included
            if not d.decompress(d.unconsumed_tail, 1 << 20) and not d.unconsumed_tail:
                break
    except zlib.error as e:
        raise ValueError(f"broken deflate stream: {e}") from None
    if not d.eof:
        raise ValueError("image data is truncated")
    if len(out) < info.raw_len:
        # as parse_png: PIL takes some streams that end early on a row's end, depending on how IDAT is cut; not these
        raise ValueError("image data is truncated")
    info.inflated = out
    R = np.frombuffer(info.inflated, np.uint8)
    for _, _, _, _, pw, ph, at in info.passes():
        if int(R[at: at + ph * (1 + info.row_bytes(pw)): 1 + info.row_bytes(pw)].max()) > 4:
            raise ValueError("unrecognized data stream contents (filter type > 4)")
    return info


def parse_png_any(data: bytes):
    """parse_png, or parse_png_general for a file parse_png refuses only for its depth, colour type or interlace.
    -> PngInfo (the 8-bit fast path) or PngGeneral."""
    try:
        return parse_png(data)
    except UnsupportedPng:
        return parse_png_general(data)


# --------------------------------------------------------------------------------------
# baseline JPEG (csrc/usdu_jpeg.cpp on the host, csrc/usdu_jpeg_decode.cu on the device)
# --------------------------------------------------------------------------------------
JPEG_SOI = b"\xff\xd8\xff"


class JpegInfo:
    """A baseline JPEG the library takes (usdu_jpeg_parse): `info` its JPEG_INFO_WORDS words, `quant` int32 [3, 64]
    tables, `coefs` the int16 coefficient blocks of its Huffman decode."""
    __slots__ = ("W", "H", "info", "quant", "coefs", "__weakref__")

    def __init__(self, info, quant, coefs):
        from . import _native as nat
        self.info, self.quant, self.coefs = info, quant, coefs
        self.W, self.H = int(info[nat.JI_W]), int(info[nat.JI_H])


def _pil_header_opens(data: bytes, W: int, H: int) -> bool:
    """PIL's own verdict on the header: Image.open parses the markers up to SOS in Python (APPn contents, Exif for the
    DPI, an MPF index) before libjpeg sees the file, and raises on some it cannot read.  Reads no pixels."""
    try:
        from PIL import Image
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            with Image.open(io.BytesIO(data)) as im:
                return im.format == "JPEG" and im.size == (W, H)
    except Exception:
        return False


def parse_jpeg(data: bytes) -> JpegInfo:
    """The marker parse and Huffman decode of a baseline JPEG, or ValueError with the reason for every file it does not
    take: the library's (include/usdu_b200.h, usdu_jpeg_parse), or a header PIL's Image.open refuses."""
    from . import _native as nat
    info, quant = nat.jpeg_parse(data)
    if not _pil_header_opens(data, int(info[nat.JI_W]), int(info[nat.JI_H])):
        raise ValueError("JPEG: PIL does not open its header")
    coefs = np.empty(int(info[nat.JI_BLOCKS]) * 64, np.int16)
    nat.jpeg_decode_coefs(data, coefs)
    return JpegInfo(info, quant, coefs)


def parse_image_any(data: bytes):
    """parse_jpeg for bytes that start with the JPEG SOI, else parse_png_any.  A JPEG parse_jpeg refuses gets
    parse_png_any's answer, the refusal any JPEG had before this path existed.  -> JpegInfo, PngInfo or PngGeneral."""
    if data[:3] == JPEG_SOI:
        try:
            return parse_jpeg(data)
        except ValueError:
            pass
    return parse_png_any(data)


class _IdatStream:
    """The concatenated data of the IDAT chunks, addressed by stream position."""

    def __init__(self, data: bytes, idat: List[Tuple[int, int]]):
        self.data = data
        self.pieces = idat
        self.starts = np.cumsum([0] + [ln for _, ln in idat]).tolist()
        self.size = self.starts[-1]

    def read(self, pos: int, k: int) -> bytes:
        if pos + k > self.size:
            raise ValueError("truncated deflate stream")
        out = b""
        i = int(np.searchsorted(self.starts, pos, side="right")) - 1
        while k > 0:
            off, ln = self.pieces[i]
            take = min(k, self.starts[i] + ln - pos)
            out += self.data[off + pos - self.starts[i]: off + pos - self.starts[i] + take]
            pos, k, i = pos + take, k - take, i + 1
        return out

    def ranges(self, pos: int, k: int):
        """(file offset, length) runs of stream bytes [pos, pos + k)."""
        i = int(np.searchsorted(self.starts, pos, side="right")) - 1
        while k > 0:
            off, ln = self.pieces[i]
            take = min(k, self.starts[i] + ln - pos)
            if take > 0:
                yield off + pos - self.starts[i], take
            pos, k, i = pos + take, k - take, i + 1

    def joined(self) -> bytes:
        return b"".join(self.data[o: o + ln] for o, ln in self.pieces)


def _stored_segments(st: _IdatStream, raw_len: int):
    """-> (segments, None, file offsets of the Adler-32 bytes) for a zlib stream of stored blocks, or ([(0, 0)], R, None)
    after inflating any other stream."""
    hdr = st.read(0, 2)
    cmf, flg = hdr[0], hdr[1]
    if (cmf & 0x0F) != 8 or (cmf >> 4) > 7 or (cmf * 256 + flg) % 31 != 0 or (flg & 0x20):
        raise ValueError("bad zlib header")
    pos, raw, segs, adler = 2, 0, [], 1
    while True:
        head = st.read(pos, 1)[0]
        if (head >> 1) & 3 != 0:                  # a compressed block: let zlib do the whole stream
            return _inflated(st, raw_len)
        ln, nln = struct.unpack("<HH", st.read(pos + 1, 4))
        if ln ^ nln != 0xFFFF:
            raise ValueError("stored block LEN/NLEN mismatch")
        pos += 5
        if pos + ln > st.size:
            raise ValueError("truncated deflate stream")
        for off, k in st.ranges(pos, ln):
            use = min(k, raw_len - raw)
            if use > 0:
                segs.append((off, raw))
            raw += use
            adler = zlib.adler32(memoryview(st.data)[off: off + k], adler)
        pos += ln
        if head & 1:
            break
    if raw < raw_len:
        raise ValueError("image data is truncated")
    if struct.unpack(">I", st.read(pos, 4))[0] != adler:
        raise ValueError("bad Adler-32 of the image data")
    trailer = [off + i for off, k in st.ranges(pos, 4) for i in range(k)]
    return segs, None, trailer


def _inflated(st: _IdatStream, raw_len: int):
    d = zlib.decompressobj()
    try:
        out = d.decompress(st.joined())
    except zlib.error as e:
        raise ValueError(f"broken deflate stream: {e}") from None
    if not d.eof:
        raise ValueError("image data is truncated")
    if len(out) < raw_len:
        raise ValueError("image data is truncated")
    return [(0, 0)], out[:raw_len], None


def filtered_stream(info: PngInfo, data: bytes) -> bytes:
    """R itself, gathered from the segments (tests and the filter-byte check)."""
    if info.inflated is not None:
        return info.inflated
    parts = []
    for i, (off, start) in enumerate(info.segs):
        end = info.segs[i + 1][1] if i + 1 < len(info.segs) else info.raw_len
        parts.append(data[off: off + end - start])
    return b"".join(parts)


def _check_filters(info: PngInfo, data: bytes):
    rowlen = 1 + info.W * info.C
    if info.inflated is not None:
        filt = np.frombuffer(info.inflated, np.uint8)[::rowlen]
    else:
        pos = np.arange(info.H, dtype=np.int64) * rowlen
        starts = np.array([s for _, s in info.segs], np.int64)
        offs = np.array([o for o, _ in info.segs], np.int64)
        k = np.searchsorted(starts, pos, side="right") - 1
        filt = np.frombuffer(data, np.uint8)[offs[k] + pos - starts[k]]
    if filt.size and int(filt.max()) > 4:
        raise ValueError("unrecognized data stream contents (filter type > 4)")


def unfilter_model(info: PngInfo, data: bytes) -> np.ndarray:
    """The un-filter and convert("RGB") in numpy, row by row: the reference the decode kernel is tested against."""
    W, H, C = info.W, info.H, info.C
    R = np.frombuffer(filtered_stream(info, data), np.uint8).reshape(H, 1 + W * C)
    out = np.zeros((H, W * C), np.int32)
    prev = np.zeros(W * C, np.int32)
    for r in range(H):
        f, row = int(R[r, 0]), R[r, 1:].astype(np.int32)
        if f == 0:
            cur = row
        elif f == 1:
            cur = row.reshape(W, C).cumsum(0).reshape(-1) & 0xFF
        elif f == 2:
            cur = (row + prev) & 0xFF
        else:
            cur = np.zeros_like(row)
            for x in range(W * C):
                a = int(cur[x - C]) if x >= C else 0
                b = int(prev[x])
                c = int(prev[x - C]) if x >= C else 0
                if f == 3:
                    pred = (a + b) >> 1
                else:
                    p = a + b - c
                    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
                    pred = a if (pa <= pb and pa <= pc) else (b if pb <= pc else c)
                cur[x] = (int(row[x]) + pred) & 0xFF
        out[r] = cur
        prev = cur
    px = out.reshape(H, W, C).astype(np.uint8)
    return np.repeat(px[:, :, :1], 3, 2) if C < 3 else np.ascontiguousarray(px[:, :, :3])


# --------------------------------------------------------------------------------------
# job store (upscale/job_store.py, job_timeout.py)
# --------------------------------------------------------------------------------------
class TileJob:
    """One static-mode job: `pending` tile ids 0..T-1 (batched_static), the workers' result queue, worker_status
    (last heartbeat), assigned_to_workers, and completed_tasks keyed by global_idx = b*T + tile.  geometry[t] =
    (x1, y1, ew, eh, pw, ph) of tile t, for the metadata and size checks of submitted tiles."""

    def __init__(self, multi_job_id: str, batch_size: int, geometry: Sequence[Tuple[int, ...]],
                 enabled_workers: Sequence[str], now: float):
        self.multi_job_id = multi_job_id
        self.batch_size = int(batch_size)
        self.num_tiles_per_image = len(geometry)
        self.geometry = [tuple(int(v) for v in g) for g in geometry]
        self.batched_static = True
        self.mode = "static"
        self.pending: asyncio.Queue = asyncio.Queue()
        for i in range(self.num_tiles_per_image):
            self.pending.put_nowait(i)
        self.queue: asyncio.Queue = asyncio.Queue()
        self.worker_status: Dict[str, float] = {str(w): now for w in enabled_workers}
        self.assigned_to_workers: Dict[str, List[int]] = {str(w): [] for w in enabled_workers}
        self.completed_tasks: Dict[int, dict] = {}


class JobStore:
    """The jobs of one server, touched only on its event loop.  `clock` gives the wall time of heartbeats."""

    def __init__(self, clock: Callable[[], float] = time.time):
        self.jobs: Dict[str, TileJob] = {}
        self.clock = clock
        self._lock: Optional[asyncio.Lock] = None

    @property
    def lock(self) -> asyncio.Lock:
        if self._lock is None:
            self._lock = asyncio.Lock()
        return self._lock

    async def init_job(self, multi_job_id, batch_size, geometry, enabled_workers):
        async with self.lock:
            if multi_job_id not in self.jobs:            # job_store.py:46-48
                self.jobs[multi_job_id] = TileJob(multi_job_id, batch_size, geometry, enabled_workers, self.clock())

    async def next_tile(self, multi_job_id, timeout: float = REQUEST_WAIT) -> Optional[int]:
        """The master's pull (job_state.py:42-57)."""
        async with self.lock:
            job = self.jobs.get(multi_job_id)
        if job is None:
            return None
        try:
            return await asyncio.wait_for(job.pending.get(), timeout=timeout)
        except asyncio.TimeoutError:
            return None

    async def mark_completed(self, multi_job_id, task_id: int, result: dict):
        """The master's own mark (job_store.py:165-171): overwrites."""
        async with self.lock:
            job = self.jobs.get(multi_job_id)
            if job is not None:
                job.completed_tasks[task_id] = result

    async def drain(self, multi_job_id) -> List[Tuple[int, dict]]:
        """Move the workers' posted results into completed_tasks (job_store.py:117-152): an entry is kept only if its
        global_idx is absent; is_last removes the worker from worker_status.  -> the (global_idx, entry) pairs kept."""
        async with self.lock:
            job = self.jobs.get(multi_job_id)
            if job is None:
                return []
            kept = []
            while True:
                try:
                    result = job.queue.get_nowait()
                except asyncio.QueueEmpty:
                    break
                for tile in result.get("tiles", ()):
                    key = tile.get("global_idx", tile["tile_idx"])
                    if key not in job.completed_tasks:
                        tile["worker_id"] = result["worker_id"]
                        job.completed_tasks[key] = tile
                        kept.append((key, tile))
                if result.get("is_last", False):
                    job.worker_status.pop(result["worker_id"], None)
            return kept

    async def status(self, multi_job_id) -> Tuple[int, int, int]:
        """-> (completed tasks, pending tile ids, active workers)."""
        async with self.lock:
            job = self.jobs.get(multi_job_id)
            if job is None:
                return 0, 0, 0
            return len(job.completed_tasks), job.pending.qsize(), len(job.worker_status)

    async def snapshot(self, multi_job_id) -> Dict[int, dict]:
        async with self.lock:
            job = self.jobs.get(multi_job_id)
            return dict(job.completed_tasks) if job is not None else {}

    async def requeue_timed_out(self, multi_job_id) -> int:
        """job_timeout.py:17-150 without the config-file probe: every worker whose last heartbeat is older than
        COMFYUI_HEARTBEAT_TIMEOUT gets its tile ids with any frame still missing put back on the queue, and leaves
        worker_status; its assignment list is emptied.  -> tile ids re-queued."""
        limit = heartbeat_timeout()
        async with self.lock:
            job = self.jobs.get(multi_job_id)
            if job is None:
                return 0
            now = self.clock()
            T, B = job.num_tiles_per_image or 1, job.batch_size or 1
            count = 0
            for worker, seen in list(job.worker_status.items()):
                if now - float(seen) <= limit:
                    continue
                for tid in list(job.assigned_to_workers.get(worker, [])):
                    if any(b * T + tid not in job.completed_tasks for b in range(B)):
                        job.pending.put_nowait(tid)
                        count += 1
                job.worker_status.pop(worker, None)
                if worker in job.assigned_to_workers:
                    job.assigned_to_workers[worker] = []
            return count

    async def cleanup(self, multi_job_id):
        async with self.lock:
            self.jobs.pop(multi_job_id, None)


# --------------------------------------------------------------------------------------
# routes (api/usdu_routes.py)
# --------------------------------------------------------------------------------------
def _error(message, status):
    from aiohttp import web
    return web.json_response({"error": str(message)}, status=status)


def parse_tiles_from_form(data) -> List[dict]:
    """_parse_tiles_from_form (payload_parsers.py:7-64) with the PNG validated and kept as bytes, not decoded."""
    try:
        padding = int(data.get("padding", 0)) if data.get("padding") is not None else 0
    except Exception:
        padding = 0
    meta_raw = data.get("tiles_metadata")
    if meta_raw is None:
        raise ValueError("Missing tiles_metadata")
    try:
        metadata = json.loads(meta_raw)
    except Exception as e:
        raise ValueError(f"Invalid tiles_metadata JSON: {e}")
    if not isinstance(metadata, list):
        raise ValueError("tiles_metadata must be a list")
    tiles = []
    for i, meta in enumerate(metadata):
        field = data.get(f"tile_{i}")
        if field is None or not hasattr(field, "file"):
            raise ValueError(f"Missing tile data for index {i}")
        raw = field.file.read()
        try:
            info = parse_image_any(raw)
        except Exception as e:
            raise ValueError(f"Invalid image data for tile {i}: {e}")
        try:
            tile = {"png": raw, "info": info, "tile_idx": int(meta.get("tile_idx", i)), "x": int(meta.get("x", 0)),
                    "y": int(meta.get("y", 0)), "extracted_width": int(meta.get("extracted_width", info.W)),
                    "extracted_height": int(meta.get("extracted_height", info.H)), "padding": int(padding)}
        except Exception as e:
            raise ValueError(f"Invalid metadata values for tile {i}: {e}")
        for k in ("batch_idx", "global_idx"):
            if k in meta:
                try:
                    tile[k] = int(meta[k])
                except Exception:
                    pass
        tiles.append(tile)
    return tiles


def _check_geometry(job: TileJob, tiles: List[dict]) -> Optional[str]:
    """The checks the reference does not make: the window metadata and the PNG size must be the plan's."""
    for i, t in enumerate(tiles):
        tid = t["tile_idx"]
        if not 0 <= tid < job.num_tiles_per_image:
            return f"Invalid tile_idx {tid} for tile {i}: the job has {job.num_tiles_per_image} tiles"
        x1, y1, ew, eh, pw, ph = job.geometry[tid]
        if (t["x"], t["y"], t["extracted_width"], t["extracted_height"]) != (x1, y1, ew, eh):
            return (f"Tile {i} (tile_idx {tid}): window ({t['x']}, {t['y']}, {t['extracted_width']}, "
                    f"{t['extracted_height']}) differs from the plan's ({x1}, {y1}, {ew}, {eh})")
        if (t["info"].W, t["info"].H) != (pw, ph):
            return f"Tile {i} (tile_idx {tid}): image is {t['info'].W}x{t['info'].H}, processing size is {pw}x{ph}"
    return None


def make_handlers(store: JobStore):
    """The five route handlers over `store` -> {(method, path): handler}."""
    from aiohttp import web

    async def heartbeat(request):
        try:
            data = await request.json()
            worker_id, multi_job_id = data.get("worker_id"), data.get("multi_job_id")
            if not worker_id or not multi_job_id:
                return _error("Missing worker_id or multi_job_id", 400)
            async with store.lock:
                job = store.jobs.get(multi_job_id)
                if job is not None:
                    job.worker_status[worker_id] = store.clock()
                    return web.json_response({"status": "success"})
                return _error("Job not found", 404)
        except Exception as e:
            return _error(e, 500)

    async def submit_tiles(request):
        try:
            content_length = request.headers.get("content-length")
            if content_length and int(content_length) > max_payload_size():
                return _error(f"Payload too large: {content_length} bytes", 413)
            data = await request.post()
            multi_job_id, worker_id = data.get("multi_job_id"), data.get("worker_id")
            is_last = data.get("is_last", "False").lower() == "true"
            if multi_job_id is None or worker_id is None:
                return _error("Missing multi_job_id or worker_id", 400)
            batch_size = int(data.get("batch_size", 0))
            if batch_size == 0 and is_last:
                async with store.lock:
                    job = store.jobs.get(multi_job_id)
                    if job is not None:
                        job.queue.put_nowait({"worker_id": worker_id, "is_last": True, "tiles": []})
                        return web.json_response({"status": "success"})
            try:               # the PNG inflate and the JPEG Huffman decode run off the server loop
                tiles = await asyncio.get_running_loop().run_in_executor(None, parse_tiles_from_form, data)
            except ValueError as e:
                return _error(str(e), 400)
            async with store.lock:
                job = store.jobs.get(multi_job_id)
                if job is None:
                    return _error("Job not found", 404)
                bad = _check_geometry(job, tiles)
                if bad is not None:
                    return _error(bad, 400)
                if batch_size > 0 or tiles:
                    job.queue.put_nowait({"worker_id": worker_id, "tiles": tiles, "is_last": is_last})
                else:
                    job.queue.put_nowait({"worker_id": worker_id, "is_last": True, "tiles": []})
                return web.json_response({"status": "success"})
        except Exception as e:
            return _error(e, 500)

    async def submit_image(request):
        # dynamic mode is unreachable in the reference (its master never creates an image job): every image submission
        # for a known job answers as the reference does for a tile job
        try:
            content_length = request.headers.get("content-length")
            if content_length and int(content_length) > max_payload_size():
                return _error(f"Payload too large: {content_length} bytes", 413)
            data = await request.post()
            multi_job_id, worker_id = data.get("multi_job_id"), data.get("worker_id")
            is_last = data.get("is_last", "False").lower() == "true"
            if multi_job_id is None or worker_id is None:
                return _error("Missing multi_job_id or worker_id", 400)
            if "full_image" in data and "image_idx" in data:
                int(data.get("image_idx"))
                img = data["full_image"].file.read()
                try:
                    await asyncio.get_running_loop().run_in_executor(None, parse_image_any, img)
                except ValueError as e:
                    return _error(e, 500)
            elif not is_last:
                return _error("Missing image data or invalid request", 400)
            async with store.lock:
                if multi_job_id in store.jobs:
                    return _error("Job not configured for image submissions", 400)
            return _error("Job not found", 404)
        except Exception as e:
            return _error(e, 500)

    async def request_image(request):
        try:
            data = await request.json()
            worker_id, multi_job_id = data.get("worker_id"), data.get("multi_job_id")
            if not worker_id or not multi_job_id:
                return _error("Missing worker_id or multi_job_id", 400)
            async with store.lock:
                job = store.jobs.get(multi_job_id)
                if job is None:
                    return _error("Job not found", 404)
                try:            # the wait happens under the lock, as in usdu_routes.py:180-212
                    tid = await asyncio.wait_for(job.pending.get(), timeout=REQUEST_WAIT)
                except asyncio.TimeoutError:
                    return web.json_response({"tile_idx": None})
                job.assigned_to_workers.setdefault(worker_id, []).append(tid)
                job.worker_status[worker_id] = store.clock()
                return web.json_response({"tile_idx": tid, "estimated_remaining": job.pending.qsize(),
                                          "batched_static": job.batched_static})
        except Exception as e:
            return _error(e, 500)

    async def job_status(request):
        multi_job_id = request.query.get("multi_job_id")
        if not multi_job_id:
            return web.json_response({"ready": False})
        async with store.lock:
            return web.json_response({"ready": multi_job_id in store.jobs})

    return {("POST", "/distributed/heartbeat"): heartbeat, ("POST", "/distributed/submit_tiles"): submit_tiles,
            ("POST", "/distributed/submit_image"): submit_image, ("POST", "/distributed/request_image"): request_image,
            ("GET", "/distributed/job_status"): job_status}


# the routes a master needs served by this module for the master role
MASTER_ROUTES = (("GET", "/distributed/job_status"), ("POST", "/distributed/request_image"),
                 ("POST", "/distributed/heartbeat"), ("POST", "/distributed/submit_tiles"))

STORE = JobStore()
_served: set = set()
_loop = None
_warned: set = set()


def register(routes, store: JobStore = STORE, loop=None) -> set:
    """Add the handlers to an aiohttp RouteTableDef (ComfyUI's PromptServer.instance.routes), skipping, with one warning
    each, every path another package already serves.  -> the (method, path) pairs this module serves."""
    global _loop
    taken = {(getattr(r, "method", None), getattr(r, "path", None)) for r in routes}
    served = set()
    for (method, path), fn in make_handlers(store).items():
        if (method, path) in taken:
            if (method, path) not in _warned:
                _warned.add((method, path))
                warnings.warn(f"comfyui-distributed_b200: {method} {path} is already served by another package; "
                              "this package's master role stays off", RuntimeWarning, stacklevel=2)
            continue
        routes.route(method, path)(fn)
        served.add((method, path))
    if store is STORE:
        _served.update(served)
        _loop = loop
    return served


def install_in_comfyui():
    """Register the routes of this module, of http_collector, of the orchestrator and of worker_routes on
    server.PromptServer.instance when imported inside ComfyUI; a no-op elsewhere."""
    try:
        import server
        inst = server.PromptServer.instance
    except Exception:
        return
    if inst is None or getattr(inst, "routes", None) is None:
        return
    if not _served:
        register(inst.routes, STORE, getattr(inst, "loop", None))
    from . import http_collector, orchestrator, worker_routes
    http_collector.install(inst.routes, getattr(inst, "loop", None))
    orchestrator.install(inst)
    worker_routes.install(inst)


def serving() -> bool:
    """This process serves the master's routes (and has the server loop to reach them)."""
    return all(r in _served for r in MASTER_ROUTES) and _server_loop() is not None


def _server_loop():
    if _loop is not None:
        return _loop
    try:
        import server
        return server.PromptServer.instance.loop
    except Exception:
        return None


def reset_for_tests():
    """Forget the registration (test harnesses that start and stop their own server)."""
    global _loop
    _served.clear()
    _loop = None
    STORE.jobs.clear()
    STORE._lock = None


# --------------------------------------------------------------------------------------
# decode on the device as frames arrive (csrc/usdu_png_decode.cu)
# --------------------------------------------------------------------------------------
class PngDecoder:
    """Uploads batches of validated PNGs through pinned memory and decodes each batch with one usdu_png_decode_u8
    launch on a side stream, so the caller can go on waiting for more.  A batch's staging stays alive until
    `release()`; `times()` (after the side stream has finished) sums the upload and decode times of every batch."""

    def __init__(self, device):
        import torch
        self.device = device
        with torch.cuda.device(device):
            self.side = torch.cuda.Stream(device)
        self._events = []
        self._keep_alive = []

    def decode(self, items: Sequence[Tuple[object, bytes, int]], dst) -> int:
        """items: (PngInfo, PngGeneral or JpegInfo, the posted bytes, byte offset of the frame's [H, W, 3] u8 output in
        the device tensor `dst`).  The 8-bit PNGs go to usdu_png_decode_u8, the other PNGs to
        usdu_png_decode_general_u8, the JPEGs to usdu_jpeg_decode_u8, on the side stream.  -> launches made."""
        general = [it for it in items if isinstance(it[0], PngGeneral)]
        jpeg = [it for it in items if isinstance(it[0], JpegInfo)]
        fast = [it for it in items if not isinstance(it[0], (PngGeneral, JpegInfo))]
        self._decode_fast(fast, dst)
        self.decode_general([(info, off) for info, _, off in general], dst)
        self.decode_jpeg([(info, off) for info, _, off in jpeg], dst)
        return int(bool(fast)) + int(bool(general)) + int(bool(jpeg))

    def decode_jpeg(self, items: Sequence[Tuple[JpegInfo, int]], dst):
        """items: (JpegInfo, byte offset of the frame's output in `dst`): each frame's quantisation tables and
        coefficients uploaded through pinned memory, one usdu_jpeg_decode_u8 launch over all of them."""
        import torch
        from . import _native as nat
        if not items:
            return
        blobs, descs, pos, ctas = [], [], 0, 0
        for info, off in items:
            w = info.info
            q_at, c_at = pos, pos + info.quant.nbytes
            blobs += [(q_at, info.quant.view(np.uint8).reshape(-1)), (c_at, info.coefs.view(np.uint8))]
            pos = (c_at + info.coefs.nbytes + 15) // 16 * 16
            descs.append([c_at, q_at, info.W, info.H, w[nat.JI_COMPONENTS], w[nat.JI_H0], w[nat.JI_V0],
                          w[nat.JI_COLOUR], w[nat.JI_MCUX], w[nat.JI_MCUY], off, ctas, 0, 0, 0, 0])
            ctas += int(w[nat.JI_MCUY]) * ((info.W + nat.JPEG_TILE_W - 1) // nat.JPEG_TILE_W)
        tabs = np.asarray(descs, np.int64).reshape(-1)
        host = torch.empty(pos + tabs.nbytes, dtype=torch.uint8, pin_memory=True)
        h = host.numpy()
        for at, blob in blobs:
            h[at: at + blob.size] = blob
        h[pos:] = tabs.view(np.uint8)
        with torch.cuda.device(self.device), torch.cuda.stream(self.side):
            dev = torch.empty(host.numel(), dtype=torch.uint8, device=self.device)
            e_up, e0, e1 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            e_up.record(self.side)
            dev.copy_(host, non_blocking=True)
            e0.record(self.side)
            nat.jpeg_decode_u8(dev.data_ptr(), dev.data_ptr() + pos, len(descs), ctas, dst.data_ptr(),
                               self.side.cuda_stream)
            e1.record(self.side)
        self._events.append((e_up, e0, e1))
        self._keep_alive.append((host, dev, dst))

    def decode_general(self, items: Sequence[Tuple[PngGeneral, int]], dst):
        """items: (PngGeneral, byte offset of the frame's output in `dst`): each frame's R and palette uploaded through
        pinned memory, one CTA per (frame, pass) in one usdu_png_decode_general_u8 launch."""
        import torch
        from . import _native as nat
        if not items:
            return
        blobs, descs, pos, max_row = [], [], 0, 1
        for info, off in items:
            pal = pos
            if info.palette is not None:
                blobs.append(info.palette)
                pos += len(info.palette)
            for x0, y0, dx, dy, pw, ph, at in info.passes():
                descs.append([pos + at, pw, ph, x0, y0, dx, dy, info.W, info.color, info.depth, off, pal, 0, 0, 0, 0])
                max_row = max(max_row, info.row_bytes(pw))
            blobs.append(info.inflated)
            pos += len(info.inflated)
        tabs = np.asarray(descs, np.int64).reshape(-1)
        t0 = (pos + 15) // 16 * 16
        host = torch.empty(t0 + tabs.nbytes, dtype=torch.uint8, pin_memory=True)
        h = host.numpy()
        o = 0
        for blob in blobs:
            h[o: o + len(blob)] = np.frombuffer(blob, np.uint8)
            o += len(blob)
        h[t0:] = tabs.view(np.uint8)
        with torch.cuda.device(self.device), torch.cuda.stream(self.side):
            dev = torch.empty(host.numel(), dtype=torch.uint8, device=self.device)
            e_up, e0, e1 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            e_up.record(self.side)
            dev.copy_(host, non_blocking=True)
            e0.record(self.side)
            nat.png_decode_general_u8(dev.data_ptr(), dev.data_ptr() + t0, len(descs), max_row, dst.data_ptr(),
                                      self.side.cuda_stream)
            e1.record(self.side)
        self._events.append((e_up, e0, e1))
        self._keep_alive.append((host, dev, dst))

    def _decode_fast(self, items: Sequence[Tuple[PngInfo, bytes, int]], dst):
        import torch
        from . import _native as nat
        if not items:
            return
        blobs, segs, descs, pos, max_row = [], [], [], 0, 1
        for info, png, off in items:
            blob = info.inflated if info.inflated is not None else png
            descs.append([len(segs), len(info.segs), info.H, info.W, info.C, off, 0, 0])
            segs.extend((pos + o, r) for o, r in info.segs)
            blobs.append(blob)
            pos += len(blob)
            max_row = max(max_row, info.W * info.C)
        tabs = np.concatenate([np.asarray(segs, np.int64).reshape(-1), np.asarray(descs, np.int64).reshape(-1)])
        nbytes = (pos + 15) // 16 * 16 + tabs.nbytes
        host = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
        h = host.numpy()
        o = 0
        for blob in blobs:
            h[o: o + len(blob)] = np.frombuffer(blob, np.uint8)
            o += len(blob)
        t0 = (pos + 15) // 16 * 16
        h[t0:] = tabs.view(np.uint8)
        with torch.cuda.device(self.device), torch.cuda.stream(self.side):
            dev = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
            e_up, e0, e1 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            e_up.record(self.side)
            dev.copy_(host, non_blocking=True)
            e0.record(self.side)
            nat.png_decode_u8(dev.data_ptr(), dev.data_ptr() + t0, len(segs), dev.data_ptr() + t0 + 16 * len(segs),
                              len(descs), max_row, dst.data_ptr(), self.side.cuda_stream)
            e1.record(self.side)
        self._events.append((e_up, e0, e1))
        self._keep_alive.append((host, dev, dst))

    def decode_device(self, items: Sequence[Tuple[PngInfo, object, int]], dst):
        """items: (info of stored blocks, http_collector.DevicePng on this device, byte offset of the frame's output in
        `dst`): decoded where the PNGs lie, after each one's `ready` event; only the segment table is uploaded."""
        import torch
        from . import _native as nat
        if not items:
            return
        base = min(png.buf.data_ptr() for _, png, _ in items)
        segs, descs, max_row = [], [], 1
        for info, png, off in items:
            descs.append([len(segs), len(info.segs), info.H, info.W, info.C, off, 0, 0])
            at = png.buf.data_ptr() - base
            segs.extend((at + o, r) for o, r in info.segs)
            max_row = max(max_row, info.W * info.C)
        tabs = np.concatenate([np.asarray(segs, np.int64).reshape(-1), np.asarray(descs, np.int64).reshape(-1)])
        host = torch.from_numpy(tabs).pin_memory()
        with torch.cuda.device(self.device), torch.cuda.stream(self.side):
            for _, png, _ in items:
                self.side.wait_event(png.ready)
            dev = torch.empty(tabs.size, dtype=torch.int64, device=self.device)
            e_up, e0, e1 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            e_up.record(self.side)
            dev.copy_(host, non_blocking=True)
            e0.record(self.side)
            nat.png_decode_u8(base, dev.data_ptr(), len(segs), dev.data_ptr() + 16 * len(segs), len(descs), max_row,
                              dst.data_ptr(), self.side.cuda_stream)
            e1.record(self.side)
        self._events.append((e_up, e0, e1))
        self._keep_alive.append((host, dev, dst, [png for _, png, _ in items]))

    def times(self) -> Tuple[float, float]:
        """-> (upload ms, decode ms) over every batch so far; the side stream must have finished."""
        return (sum(a.elapsed_time(b) for a, b, _ in self._events),
                sum(b.elapsed_time(c) for _, b, c in self._events))

    def release(self):
        self._keep_alive.clear()


# --------------------------------------------------------------------------------------
# the master role (static.py:371-570) on the device
# --------------------------------------------------------------------------------------
class HttpStaticMaster:
    """One static-mode job with this process as the master of HTTP workers.  `job` is an engine.WorkerJob (the master's
    own u8 canvas and 1-tile step); worker tiles are decoded into a payload buffer with one [B, ph, pw, 3] slot per
    tile and composited onto the master's canvas at the end."""

    def __init__(self, job, multi_job_id: str, enabled_workers: Sequence[str], store: JobStore = STORE, loop=None):
        import torch
        self.job, self.multi_job_id = job, multi_job_id
        self.workers = [str(w) for w in enabled_workers]
        self.store, self.loop = store, loop if loop is not None else _server_loop()
        if self.loop is None:
            raise RuntimeError("HttpStaticMaster: no server event loop")
        plan, B = job.plan, job.canvas.B
        self.T, self.B = len(plan.tiles), B
        self.geometry = [(t.x1, t.y1, t.ew, t.eh, t.pw, t.ph) for t in plan.tiles]
        self.base, cur = [], 0
        for t in plan.tiles:                      # tile t's frames: payload[base[t] + b * frame bytes]
            self.base.append(cur)
            cur = (cur + B * t.ph * t.pw * 3 + 15) // 16 * 16
        self.device = job.device
        with torch.cuda.device(self.device):
            self.payload = torch.empty(max(cur, 16), dtype=torch.uint8, device=self.device)
        self.decoder = PngDecoder(self.device)
        self.master_ids: List[int] = []
        self.kept: Dict[str, List[int]] = {}
        self.stats = {"bytes_received": 0, "tiles_received": 0, "upload_ms": 0.0, "decode_ms": 0.0,
                      "decode_launches": 0, "blend_ms": 0.0}

    # -- event-loop calls ---------------------------------------------------------------
    def _call(self, coro, timeout: Optional[float] = 5.0):
        return asyncio.run_coroutine_threadsafe(coro, self.loop).result(timeout)

    # -- the master's own tiles ---------------------------------------------------------
    def _process(self, tid: int):
        self.job.step_device(tid)
        self.master_ids.append(tid)
        for b in range(self.B):
            self._call(self.store.mark_completed(self.multi_job_id, b * self.T + tid, {"batch_idx": b, "tile_idx": tid}))

    # -- decode as results arrive ---------------------------------------------------------
    def _decode(self, entries: List[Tuple[int, dict]]):
        """Upload the PNG bytes (or, for a PngGeneral, the filtered stream) of `entries` through pinned memory and
        decode them on the side stream."""
        items = []
        for g, e in entries:
            b = e.get("batch_idx", g // self.T)
            t = e["tile_idx"]
            if b >= self.B or not 0 <= t < self.T:
                continue
            self.kept.setdefault(str(e["worker_id"]), [])
            if t not in self.kept[str(e["worker_id"])]:
                self.kept[str(e["worker_id"])].append(t)
            info = e["info"]
            items.append((info, e["png"], self.base[t] + b * info.H * info.W * 3))
            self.stats["bytes_received"] += len(e["png"])
        if not items:
            return
        self.stats["tiles_received"] += len(items)
        self.stats["decode_launches"] += self.decoder.decode(items, self.payload)

    # -- the job --------------------------------------------------------------------------
    def run(self):
        """-> the result fp32 [B, H, W, 3] on the master's device."""
        import torch
        mm = _comfy_mm()
        job_id, total = self.multi_job_id, self.T * self.B
        self._call(self.store.init_job(job_id, self.B, self.geometry, self.workers), 10.0)
        try:
            processed, empty = 0, 0
            while processed < total:                  # static.py:406-448
                if mm is not None:
                    mm.throw_exception_if_processing_interrupted()
                tid = self._call(self.store.next_tile(job_id))
                if tid is not None:
                    empty = 0
                    self._process(tid)
                    processed += self.B
                else:
                    empty += 1
                    if empty >= MASTER_EMPTY_POLLS:
                        break
                    time.sleep(0.1)
            if processed < total:
                snap = self._collect()
                if len(snap) < total:                 # static.py:470-513: what the timed-out workers left
                    while True:
                        if mm is not None:
                            mm.throw_exception_if_processing_interrupted()
                        tid = self._call(self.store.next_tile(job_id))
                        if tid is None:
                            break
                        self._process(tid)
            else:
                snap = self._call(self.store.snapshot(job_id))
            return self._composite(snap)
        finally:
            self._call(self.store.cleanup(job_id))

    def _collect(self) -> Dict[int, dict]:
        """_async_collect_and_monitor_static (static.py:316-369), with each drained batch decoded on the side stream."""
        mm = _comfy_mm()
        job_id, total = self.multi_job_id, self.T * self.B
        last_check = time.time()
        while True:
            if mm is not None and mm.processing_interrupted():
                raise mm.InterruptProcessingException()
            kept = self._call(self.store.drain(job_id))
            if kept:
                self._decode(kept)
            now = time.time()
            if now - last_check >= heartbeat_interval():
                self._call(self.store.requeue_timed_out(job_id))
                last_check = now
            done, pending, active = self._call(self.store.status(job_id))
            if done >= total or (pending > 0 and active == 0):
                break
            time.sleep(COLLECT_POLL)
        return self._call(self.store.snapshot(job_id))

    def _composite(self, snap: Dict[int, dict]):
        """Blend the kept worker entries onto the master's canvas in (tile_idx, batch_idx, global_idx) order
        (static.py:521-553): one launch over all tiles when every kept tile has all its frames, else one per frame."""
        import torch
        from .engine import Canvas
        T, B = self.T, self.B
        have: Dict[int, set] = {}
        for g, e in snap.items():
            if "png" not in e:
                continue                              # the master's own mark: no image (static.py:529-531)
            b, t = e.get("batch_idx", g // T), e.get("tile_idx", g % T)
            if b < B and 0 <= t < T:
                have.setdefault(t, set()).add(b)
        canvas = self.job.canvas
        with torch.cuda.device(self.device):
            main = torch.cuda.current_stream()
            main.wait_stream(self.decoder.side)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            tiles = sorted(have)
            if tiles and all(len(have[t]) == B for t in tiles):
                canvas.blend(tiles, self.payload, np.array([self.base[t] for t in tiles], np.int64))
            else:
                plan = self.job.plan
                for b in range(B):
                    ids = [t for t in tiles if b in have[t]]
                    if ids:
                        one = Canvas(canvas.dp, 1, canvas.buf[b:b + 1])
                        offs = np.array([self.base[t] + b * plan.tiles[t].ph * plan.tiles[t].pw * 3 for t in ids],
                                        np.int64)
                        one.blend(ids, self.payload, offs)
            e1.record()
            out = canvas.result()
            main.synchronize()
        self.stats["blend_ms"] = e0.elapsed_time(e1)
        self.stats["upload_ms"], self.stats["decode_ms"] = self.decoder.times()
        self.decoder.release()
        return out

    def assignment(self) -> List[List[int]]:
        """The effective assignment: the master's tile ids in processing order, then the tile ids kept from each
        enabled worker (then any other worker), in arrival order."""
        order = self.workers + sorted(w for w in self.kept if w not in self.workers)
        return [list(self.master_ids)] + [list(self.kept.get(w, [])) for w in order]


def _comfy_mm():
    try:
        import comfy.model_management as mm
        return mm
    except ImportError:
        return None
