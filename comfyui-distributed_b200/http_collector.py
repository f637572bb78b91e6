"""Master side of the reference's collector transport: its job_complete and prepare_job routes
(api/job_routes.py:142-157, 273-343) and the master role of DistributedCollector (nodes/collector.py:238-469), with the
workers' images decoded and assembled on this GPU.

The routes and the job state (multi_job_id -> asyncio.Queue, plus a lock) live on ComfyUI's server event loop, as in
the reference; the master's prompt thread reaches them with `run_coroutine_threadsafe`.  The job_complete handler checks
a POST in the reference's order and answers with its status codes and JSON bodies, but never decodes pixels.  With a
CUDA device (DeviceChecks), the image's base64 text is decoded on the device and the decoded PNG's Adler-32 and filter
bytes are checked there (csrc/usdu_b64.cu); the handler awaits the result without holding the loop, replays
http_master.parse_png's structural walk over the chunk and block headers the device read out (check_png_tables), and
queues the PNG as it lies on the device (DevicePng, a lease on a bounded DevicePool), on the device the job's master
decodes on.  Without a device, when the buffers cannot be had (the pool's bound, or device or pinned memory the master's
model holds), or for what the device tables do not settle (compressed blocks, more chunks or blocks than the table
holds), the host path png_of_payload answers as the reference does (`b64decode(validate=True)`, then parse_png).  A
palette, 1/2/4/16-bit or interlaced PNG, which parse_png refuses for its IHDR, is validated and inflated on the host by
http_master.parse_png_general (the device path hands it the decoded bytes) and decoded with usdu_png_decode_general_u8.
A baseline JPEG (base64 text starting "/9j/") always takes the host path, off the event loop: b64decode, then the
library's marker parse and Huffman decode (http_master.parse_jpeg); usdu_jpeg_decode_u8 does the rest on the device.
Both paths give every body the same answer.  The master decodes each drained batch of frames on a side stream (http_master.PngDecoder), from the
device buffers or through a pinned upload, while it waits for more, and assembles the result with one
usdu_gather_unpack_f32 launch that writes every worker frame, as k / 255, straight into the pinned host result in its
final order.

Differences from the reference (INTEGRATION.md, "A master for HTTP workers"):
* images PIL would open but this module refuses answer the reference's decode-failure response (500, "Failed to
  decode PNG image payload: ..."): PNGs with filtered rows over PNG_MAX_ROW_BYTES (16,384 8-bit RGBA pixels), JPEGs
  outside the baseline subset http_master.parse_jpeg takes, and other formats PIL detects (BMP, GIF, ...).  Neither
  worker sends any of them;
* no busy-probe of missing workers (collector.py:374-411 reads the orchestrator's gpu_config.json), and the worker
  timeout is COMFYUI_HEARTBEAT_TIMEOUT (default 60 s), not the config file's setting;
* delegate-only mode comes from the node's hidden input only, not from the config file;
* load_balance is not implemented (the orchestrator's concern), as for the USDU master.
"""
from __future__ import annotations

import asyncio
import base64
import binascii
import os
import struct
import time
import warnings
import weakref
import zlib
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import _native as nat
from .http_master import (CHANNELS, PNG_MAX_ROW_BYTES, PNG_SIGNATURE, JpegInfo, PngInfo, UnsupportedPng, _IdatStream,
                          heartbeat_interval, heartbeat_timeout, parse_image_any, parse_png, parse_png_general)

JOB_INIT_GRACE_PERIOD = 10.0        # utils/constants.py:37: how long a POST waits for its job's queue
GRACE_POLL = 0.05                   # job_routes.py:333
EMPTY_AUDIO_SAMPLE_RATE = 44100


def max_audio_payload_bytes() -> int:
    return int(os.environ.get("COMFYUI_MAX_AUDIO_PAYLOAD_BYTES", str(256 * 1024 * 1024)))


# --------------------------------------------------------------------------------------
# request checks (job_routes.py:104-139, utils/audio_payload.py), messages as the reference's
# --------------------------------------------------------------------------------------
def field_errors(data: dict) -> List[str]:
    job_id, worker_id, batch_idx = data.get("job_id"), data.get("worker_id"), data.get("batch_idx")
    image, audio, is_last = data.get("image"), data.get("audio"), data.get("is_last")
    errors = []
    if not isinstance(job_id, str) or not job_id.strip():
        errors.append("job_id: expected non-empty string")
    if not isinstance(worker_id, str) or not worker_id.strip():
        errors.append("worker_id: expected non-empty string")
    if not isinstance(batch_idx, int) or batch_idx < 0:        # a bool is an int here, as in the reference
        errors.append("batch_idx: expected non-negative integer")
    if not isinstance(image, str) or not image.strip():
        errors.append("image: expected non-empty base64 PNG string")
    if audio is not None and not isinstance(audio, dict):
        errors.append("audio: expected object when provided")
    if not isinstance(is_last, bool):
        errors.append("is_last: expected boolean")
    return errors


NOT_BASE64 = "Field 'image' is not valid base64 PNG data."
EMPTY_PNG = "Field 'image' decoded to empty PNG data."
PNG_FAILED = "Failed to decode PNG image payload: "


def payload_text(image: str) -> str:
    """The image field -> its base64 text (after a data URL's header), or ValueError with the reference's message."""
    text = image.strip()
    if text.startswith("data:"):
        header, sep, body = text.partition(",")
        if not sep:
            raise ValueError("Field 'image' data URL is malformed.")
        if not header.lower().startswith("data:image/png;base64"):
            raise ValueError("Field 'image' must be a PNG data URL when using data:* format.")
        text = body
    return text


def png_of_payload(image: str) -> Tuple[bytes, PngInfo]:
    """The image field -> (image bytes, their validation: PngInfo, PngGeneral for a palette, 1/2/4/16-bit or
    interlaced PNG, JpegInfo for a baseline JPEG), or ValueError with the reference's message: the host path."""
    text = payload_text(image)
    try:
        png = base64.b64decode(text, validate=True)
    except (binascii.Error, ValueError) as exc:
        raise ValueError(NOT_BASE64) from exc
    if not png:
        raise ValueError(EMPTY_PNG)
    try:
        info = parse_image_any(png)
    except Exception as exc:
        raise ValueError(f"{PNG_FAILED}{exc}") from exc
    return png, info


# --------------------------------------------------------------------------------------
# parse_png split: the device tables of usdu_b64_png_check, the structural walk here
# --------------------------------------------------------------------------------------
_CB = nat.B64_HEAD_WORDS
_BB = _CB + 4 * nat.B64_MAX_CHUNKS
_PB = _BB + 4 * nat.B64_MAX_BLOCKS


class HostParse(Exception):
    """The device tables do not settle this file (a compressed block, more chunks or blocks than the table holds, chunks
    before IDAT past the fetched prefix): parse_png decides on the whole file."""


def check_png_tables(tab: np.ndarray, m: int) -> PngInfo:
    """parse_png over the m-byte PNG that usdu_b64_png_check decoded, from its table `tab` (int64): the walk over the
    chunk and stored-block headers here, with parse_png's checks and reasons in its order; the Adler-32 and the largest
    filter byte from the device.  -> the same PngInfo, or ValueError with parse_png's reason (UnsupportedPng where
    parse_png raises it), or HostParse."""
    head = tab[:_CB]
    prefix = tab[_PB:].view(np.uint8)[:min(m, nat.B64_PREFIX_BYTES)].tobytes()
    nc = int(head[4])
    ch = tab[_CB: _CB + 4 * nc].reshape(-1, 4).tolist()
    if m < 8 or prefix[:8] != PNG_SIGNATURE:
        raise ValueError("not a PNG file")
    pos, i = 8, 0
    ihdr = None
    idat: List[Tuple[int, int]] = []
    while True:
        if pos + 8 > m:
            raise ValueError("truncated PNG (chunk header)")
        if i == nc:
            raise HostParse("chunk table full")
        at, length, ctype, _ = ch[i]
        i += 1
        if at != pos:
            raise HostParse("chunk table out of step")
        ctype = int(ctype).to_bytes(4, "big")
        body = pos + 8
        if length > 0x7FFFFFFF or body + length + 4 > m:
            raise ValueError(f"truncated PNG ({ctype!r} chunk runs past the end)")
        if ihdr is None:
            if ctype != b"IHDR" or length != 13:
                raise ValueError("first chunk is not IHDR")
        if not idat and ctype != b"IDAT":
            if body + length + 4 > len(prefix):
                raise HostParse("chunk before IDAT past the prefix")
            crc, = struct.unpack_from(">I", prefix, body + length)
            if zlib.crc32(prefix[pos + 4: body + length]) != crc:
                raise ValueError(f"bad CRC in {ctype.decode('latin-1')}")
        if ctype == b"IHDR":
            if ihdr is not None:
                raise ValueError("second IHDR")
            W, H, depth, color, comp, filt, interlace = struct.unpack_from(">IIBBBBB", prefix, body)
            if W == 0 or H == 0 or W > 0x7FFFFFFF or H > 0x7FFFFFFF:
                raise ValueError("bad image size")
            if depth != 8 or color not in CHANNELS:
                raise UnsupportedPng(f"unsupported PNG: bit depth {depth}, colour type {color}")
            if comp != 0 or filt != 0:
                raise ValueError("unknown compression or filter method")
            if interlace != 0:
                raise UnsupportedPng("unsupported PNG: interlaced")
            if W * CHANNELS[color] > PNG_MAX_ROW_BYTES:
                raise ValueError(f"unsupported PNG: rows of {W * CHANNELS[color]} bytes (at most {PNG_MAX_ROW_BYTES})")
            ihdr = (W, H, CHANNELS[color])
        elif ctype == b"IDAT":
            if idat and idat[-1][0] + idat[-1][1] + 4 != pos:
                raise ValueError("IDAT chunks are not consecutive")
            idat.append((body, length))
        elif idat:
            break
        elif ctype == b"IEND":
            raise ValueError("no IDAT chunk")
        pos = body + length + 4
    W, H, C = ihdr
    raw_len = H * (1 + W * C)
    st = _IdatStream(None, idat)
    if st.size != int(head[8]):
        raise HostParse("stream size out of step")
    # _stored_segments
    if st.size < 2:
        raise ValueError("truncated deflate stream")
    zh = int(head[7])
    cmf, flg = zh & 0xFF, zh >> 8
    if (cmf & 0x0F) != 8 or (cmf >> 4) > 7 or (cmf * 256 + flg) % 31 != 0 or (flg & 0x20):
        raise ValueError("bad zlib header")
    nb, code = int(head[9]), int(head[10])
    bl = tab[_BB: _BB + 4 * nb].reshape(-1, 4).tolist()
    pos, raw, segs, j = 2, 0, [], 0
    while True:
        if j == nb:
            if code == nat.B64_BLOCKS_SHORT:
                raise ValueError("truncated deflate stream")
            raise HostParse("block table full")
        at, packed, _, _ = bl[j]
        j += 1
        if at != pos:
            raise HostParse("block table out of step")
        hb = packed & 0xFF
        if (hb >> 1) & 3 != 0:
            raise HostParse("compressed block")
        ln, nln = (packed >> 8) & 0xFFFF, (packed >> 24) & 0xFFFF
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
        pos += ln
        if hb & 1:
            break
    if raw < raw_len:
        raise ValueError("image data is truncated")
    if pos + 4 > st.size:
        raise ValueError("truncated deflate stream")
    if code != nat.B64_BLOCKS_FINAL or int(head[15]) != pos or int(head[13]) < 0:
        raise HostParse("device checks out of step")
    if int(head[11]) != int(head[12]):
        raise ValueError("bad Adler-32 of the image data")
    trailer = [off + i for off, k in st.ranges(pos, 4) for i in range(k)]
    info = PngInfo(W, H, C, segs, None, [(off - 8, ln) for off, ln in idat], trailer)
    if int(head[13]) > 4:
        raise ValueError("unrecognized data stream contents (filter type > 4)")
    return info


# --------------------------------------------------------------------------------------
# the device path of the image checks
# --------------------------------------------------------------------------------------
POOL_BYTES = 4 << 30        # bytes of decoded PNGs (device) and JPEG coefficients (host) held at once: 81 4K RGB
                            # frames are about 2 GB
JPEG_B64 = "/9j/"           # the base64 text of a body that starts with the JPEG SOI (FF D8 FF)
WAIT_POLL = 0.0005          # s between polls of a CUDA event on the loop


class DevicePool:
    """The device buffers of decoded PNGs waiting in the collector queues, at most `limit` bytes at once.  A buffer
    returns to the pool when its DevicePng is dropped (after the master decoded it, or with its job).  A request that
    would pass the limit takes the host path."""

    def __init__(self, limit: int = POOL_BYTES):
        self.limit, self.used = int(limit), 0

    def take(self, nbytes: int, device, stream):
        import torch
        if self.used + nbytes > self.limit:
            return None
        with torch.cuda.device(device), torch.cuda.stream(stream):
            buf = torch.empty(nbytes, dtype=torch.uint8, device=device)
        self.used += nbytes
        return buf

    def give(self, nbytes: int):
        self.used -= nbytes

    def hold(self, coefs: np.ndarray):
        """Count a JPEG's host coefficient buffer, queued for the master's decode, until it is dropped: it stands in
        for the decoded bytes a PNG keeps on the device, so PNGs that arrive while it waits see the bound sooner."""
        self.used += coefs.nbytes
        weakref.finalize(coefs, self.give, coefs.nbytes)


class DevicePng:
    """A decoded PNG on the device: buf[:size] (uint8), written once `ready` (a CUDA event) has completed.  len() is
    its size; bytes(), slicing and == copy it to the host once (tests, a consumer on another device)."""
    __slots__ = ("buf", "size", "ready", "_host", "__weakref__")

    def __init__(self, buf, size: int, ready):
        self.buf, self.size, self.ready, self._host = buf, int(size), ready, None

    def __len__(self):
        return self.size

    def __bytes__(self):
        if self._host is None:
            self.ready.synchronize()
            self._host = self.buf[:self.size].cpu().numpy().tobytes()
        return self._host

    def __getitem__(self, k):
        return bytes(self)[k]

    def __eq__(self, other):
        if isinstance(other, DevicePng):
            other = bytes(other)
        if isinstance(other, (bytes, bytearray, memoryview)):
            return bytes(self) == bytes(other)
        return NotImplemented

    __hash__ = None


async def device_wait(event):
    """Wait for a CUDA event without holding the event loop."""
    while not event.query():
        await asyncio.sleep(WAIT_POLL)


class DeviceChecks:
    """The image checks of job_complete on one device, on a stream of its own: usdu_b64_png_check, then the
    structural walk on the host (check_png_tables).  One per device and process (device_checks())."""

    def __init__(self, device, pool: Optional[DevicePool] = None):
        import torch
        self.device = torch.device(device)
        with torch.cuda.device(self.device):
            self.stream = torch.cuda.Stream(self.device)
        self.pool = pool if pool is not None else DevicePool()
        self.stats = {"device": 0, "host": 0, "general": 0, "jpeg": 0}

    def _buffers(self, n: int):
        """-> (PNG buffer, pinned text, device table, pinned table) for an n-byte text, or None when they cannot all be
        had: past the pool's bound, or out of device or pinned memory (the model the master runs may hold it)."""
        import torch
        nbytes = max(16, nat.b64_png_bytes(n))
        try:
            buf = self.pool.take(nbytes, self.device, self.stream)
            if buf is None:
                return None
            weakref.finalize(buf, self.pool.give, nbytes)
            pinned = torch.empty((n + 15) // 16 * 16 or 16, dtype=torch.uint8, pin_memory=True)
            tab = torch.empty(nat.B64_TABLE_WORDS, dtype=torch.int64, pin_memory=True)
            with torch.cuda.device(self.device), torch.cuda.stream(self.stream):
                tab_dev = torch.empty(nat.B64_TABLE_WORDS, dtype=torch.int64, device=self.device)
        except RuntimeError:                            # torch.OutOfMemoryError, or a failed pinned allocation
            return None
        return buf, pinned, tab_dev, tab

    async def png_of_payload(self, image: str):
        """png_of_payload with the base64 decode and the PNG's O(bytes) checks on the device: the same answer for
        every field.  What the device cannot take (no buffers, a text of 2^31 bytes or more) or the tables do not
        settle (HostParse) gets the host path's answer from png_of_payload itself.  -> (DevicePng or bytes, PngInfo)."""
        import torch
        text = payload_text(image)
        if text.startswith(JPEG_B64):
            # a JPEG body: the host b64decode and Huffman decode, off the event loop; the device check is PNG-only
            self.stats["jpeg"] += 1
            png, info = await asyncio.get_running_loop().run_in_executor(None, png_of_payload, image)
            if isinstance(info, JpegInfo):
                self.pool.hold(info.coefs)
            return png, info
        try:
            raw = text.encode("ascii")                  # b64decode refuses a str with other characters the same way
        except UnicodeEncodeError as exc:
            raise ValueError(NOT_BASE64) from exc
        n = len(raw)
        got = self._buffers(n) if n <= nat.B64_MAX_TEXT else None
        if got is None:
            self.stats["host"] += 1
            return png_of_payload(image)
        buf, pinned, tab_dev, tab = got
        pinned.numpy()[:n] = np.frombuffer(raw, np.uint8)
        del raw, got
        with torch.cuda.device(self.device), torch.cuda.stream(self.stream):
            nat.b64_png_check(pinned.data_ptr(), n, buf.data_ptr(), tab_dev.data_ptr(), self.stream.cuda_stream)
            tab.copy_(tab_dev, non_blocking=True)
            ready = torch.cuda.Event()
            ready.record(self.stream)
        await device_wait(ready)
        del pinned, tab_dev
        t = tab.numpy()
        m = int(t[3])
        if m < 0:
            raise ValueError(NOT_BASE64)
        if m == 0:
            raise ValueError(EMPTY_PNG)
        try:
            info = check_png_tables(t, m)
        except HostParse:
            del buf
            self.stats["host"] += 1
            return png_of_payload(image)
        except UnsupportedPng:
            # palette, 1/2/4/16-bit or interlaced: parse_png_general inflates the decoded bytes, off the event loop
            png = bytes(DevicePng(buf, m, ready))
            del buf
            self.stats["general"] += 1
            try:
                info = await asyncio.get_running_loop().run_in_executor(None, parse_png_general, png)
            except Exception as exc:
                raise ValueError(f"{PNG_FAILED}{exc}") from exc
            return png, info
        except Exception as exc:
            raise ValueError(f"{PNG_FAILED}{exc}") from exc
        self.stats["device"] += 1
        return DevicePng(buf, m, ready), info


_checks: Dict = {}
_cuda_ok: Optional[bool] = None


def device_checks(device=None) -> Optional[DeviceChecks]:
    """The DeviceChecks of `device` (a CUDA device; None: the current one) when this process has a CUDA device and the
    library loads, else None (the host path).  job_complete asks for the device its job's master runs on."""
    global _cuda_ok
    if _cuda_ok is None:
        try:
            import torch
            _cuda_ok = torch.cuda.is_available()
            if _cuda_ok:
                nat.lib()
        except Exception:
            _cuda_ok = False
    if not _cuda_ok:
        return None
    import torch
    dev = torch.device(device) if device is not None else torch.device("cuda")
    if dev.type != "cuda":
        dev = torch.device("cuda")
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    if dev not in _checks:
        _checks[dev] = DeviceChecks(dev)
    return _checks[dev]


def audio_of_payload(payload) -> Optional[dict]:
    """The audio envelope -> AUDIO dict (CPU float32 waveform [batch, channels, samples]), with the reference's rules
    and messages."""
    import torch
    if payload is None:
        return None
    if not isinstance(payload, dict):
        raise ValueError("Field 'audio' must be an object when provided.")
    text, shape = payload.get("data"), payload.get("shape")
    rate, dtype = payload.get("sample_rate", 44100), payload.get("dtype", "float32")
    if not isinstance(text, str) or not text.strip():
        raise ValueError("Field 'audio.data' must be a non-empty base64 string.")
    if not isinstance(shape, list) or len(shape) != 3:
        raise ValueError("Field 'audio.shape' must be a 3-item list [batch, channels, samples].")
    if dtype != "float32":
        raise ValueError("Field 'audio.dtype' must be 'float32'.")
    try:
        dims = tuple(int(d) for d in shape)
    except (TypeError, ValueError) as exc:
        raise ValueError("Field 'audio.shape' must contain integers.") from exc
    if dims[0] <= 0 or dims[1] <= 0 or dims[2] < 0:
        raise ValueError("Field 'audio.shape' must be [batch>0, channels>0, samples>=0].")
    try:
        rate = int(rate)
    except (TypeError, ValueError) as exc:
        raise ValueError("Field 'audio.sample_rate' must be an integer.") from exc
    if rate <= 0:
        raise ValueError("Field 'audio.sample_rate' must be positive.")
    try:
        raw = base64.b64decode(text, validate=True)
    except (binascii.Error, ValueError) as exc:
        raise ValueError("Field 'audio.data' is not valid base64.") from exc
    limit = max_audio_payload_bytes()
    if len(raw) > limit:
        raise ValueError(f"Field 'audio.data' too large: {len(raw)} bytes exceeds {limit}.")
    want = int(np.prod(dims, dtype=np.int64)) * 4
    if len(raw) != want:
        raise ValueError(f"Field 'audio.data' byte size mismatch: expected {want}, got {len(raw)}.")
    wave = torch.from_numpy(np.frombuffer(raw, dtype=np.float32).reshape(dims).copy())
    return {"waveform": wave.contiguous(), "sample_rate": rate}


# --------------------------------------------------------------------------------------
# job state: multi_job_id -> queue of received frames, on the server loop
# --------------------------------------------------------------------------------------
class CollectorStore:
    """The collector jobs of one server, touched only on its event loop.  A queue item is {"png", "info",
    "worker_id", "image_index", "is_last", "audio"}: the PNG as posted (validated, not decoded), as bytes or as a
    DevicePng."""

    def __init__(self):
        self.jobs: Dict[str, asyncio.Queue] = {}
        self.devices: Dict[str, object] = {}
        self._lock: Optional[asyncio.Lock] = None

    @property
    def lock(self) -> asyncio.Lock:
        if self._lock is None:
            self._lock = asyncio.Lock()
        return self._lock

    async def prepare(self, multi_job_id, device=None):
        """The job's queue; `device`: the CUDA device its master decodes on (job_complete checks its images there)."""
        async with self.lock:
            if multi_job_id not in self.jobs:
                self.jobs[multi_job_id] = asyncio.Queue()
            if device is not None:
                self.devices[multi_job_id] = device

    async def put(self, multi_job_id, item: dict) -> bool:
        async with self.lock:
            q = self.jobs.get(multi_job_id)
            if q is None:
                return False
            q.put_nowait(item)
            return True

    async def take(self, multi_job_id, timeout: float) -> List[dict]:
        """Wait up to `timeout` for an item, then take it and every item already queued behind it ([] on a time-out
        or when the job is gone)."""
        async with self.lock:
            q = self.jobs.get(multi_job_id)
        if q is None:
            return []
        try:
            first = await asyncio.wait_for(q.get(), timeout=timeout)
        except asyncio.TimeoutError:
            return []
        return [first] + await self.drain(multi_job_id)

    async def drain(self, multi_job_id) -> List[dict]:
        async with self.lock:
            q = self.jobs.get(multi_job_id)
            out = []
            while q is not None:
                try:
                    out.append(q.get_nowait())
                except asyncio.QueueEmpty:
                    break
            return out

    async def remove(self, multi_job_id):
        async with self.lock:
            self.jobs.pop(multi_job_id, None)
            self.devices.pop(multi_job_id, None)


# --------------------------------------------------------------------------------------
# routes
# --------------------------------------------------------------------------------------
def _error(error, status=500):
    from aiohttp import web
    if isinstance(error, list):
        return web.json_response({"errors": [str(e) for e in error]}, status=status)
    return web.json_response({"error": str(error)}, status=status)


def make_handlers(store: CollectorStore, clock: Callable[[], float] = time.monotonic, checks=None):
    """The two route handlers over `store` -> {(method, path): handler}.  `checks`: the DeviceChecks job_complete uses,
    False for the host path, None for this process's (device_checks())."""
    from aiohttp import web

    async def prepare_job(request):
        try:
            data = await request.json()
            multi_job_id = data.get("multi_job_id")
            if not multi_job_id:
                return _error("Missing multi_job_id", 400)
            await store.prepare(multi_job_id)
            return web.json_response({"status": "success"})
        except Exception as e:
            return _error(e)

    async def job_complete(request):
        try:
            data = await request.json()
        except Exception as exc:
            return _error(f"Invalid JSON payload: {exc}", 400)
        if not isinstance(data, dict):
            return _error("Expected a JSON object body", 400)
        try:
            errors = field_errors(data)
            if errors:
                return _error(errors, 400)
            dev = device_checks(store.devices.get(data["job_id"].strip())) if checks is None else checks
            if dev:
                png, info = await dev.png_of_payload(data["image"])
            else:
                png, info = png_of_payload(data["image"])
            audio = audio_of_payload(data.get("audio")) if data.get("audio") is not None else None
            item = {"png": png, "info": info, "worker_id": data["worker_id"].strip(),
                    "image_index": int(data["batch_idx"]), "is_last": data["is_last"], "audio": audio}
            job_id = data["job_id"].strip()
            deadline = clock() + float(JOB_INIT_GRACE_PERIOD)
            while not await store.put(job_id, item):
                if clock() > deadline:
                    return _error("job not initialized", 404)
                await asyncio.sleep(GRACE_POLL)
            return web.json_response({"status": "success"})
        except Exception as e:
            return _error(e)

    return {("POST", "/distributed/prepare_job"): prepare_job, ("POST", "/distributed/job_complete"): job_complete}


COLLECTOR_ROUTES = (("POST", "/distributed/prepare_job"), ("POST", "/distributed/job_complete"))

STORE = CollectorStore()
_served: set = set()
_loop = None
_warned: set = set()


def register(routes, store: CollectorStore = STORE, loop=None, checks=None) -> set:
    """Add the handlers to an aiohttp RouteTableDef (ComfyUI's PromptServer.instance.routes), skipping, with one warning
    each, every path another package already serves.  -> the (method, path) pairs this module serves."""
    global _loop
    taken = {(getattr(r, "method", None), getattr(r, "path", None)) for r in routes}
    served = set()
    for (method, path), fn in make_handlers(store, checks=checks).items():
        if (method, path) in taken:
            if (method, path) not in _warned:
                _warned.add((method, path))
                warnings.warn(f"comfyui-distributed_b200: {method} {path} is already served by another package; "
                              "this package's collector master role stays off", RuntimeWarning, stacklevel=2)
            continue
        routes.route(method, path)(fn)
        served.add((method, path))
    if store is STORE:
        _served.update(served)
        _loop = loop
    return served


def install(routes, loop=None):
    """Register on ComfyUI's route table once (http_master.install_in_comfyui)."""
    if not _served:
        register(routes, STORE, loop)


def serving() -> bool:
    """This process serves the collector routes (and has the server loop to reach them)."""
    return all(r in _served for r in COLLECTOR_ROUTES) and _server_loop() is not None


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
    STORE.devices.clear()
    STORE._lock = None


# --------------------------------------------------------------------------------------
# frames on the device: decode as they arrive, one gather-unpack into the result
# --------------------------------------------------------------------------------------
class GpuFrames:
    """Each `add`ed batch of queue items is decoded on the side stream into one fresh device buffer, a 16-byte
    aligned u8 [H, W, 3] slot per frame (item["frame"] = (buffer, offset)).  `assemble` writes the result.
    stats["device_frames"] counts the frames decoded from the route's device buffers, with no upload."""

    def __init__(self, device):
        from .http_master import PngDecoder
        self.device = device
        self.decoder = PngDecoder(device)
        self.stats = {"upload_ms": 0.0, "decode_ms": 0.0, "assembly_ms": 0.0, "decode_launches": 0, "device_frames": 0}

    def add(self, items: Sequence[dict]):
        """A PNG kept on this device (DevicePng, stored blocks) is decoded where it lies; any other is uploaded (a
        PngGeneral's filtered stream, to usdu_png_decode_general_u8; a JpegInfo's coefficients, to
        usdu_jpeg_decode_u8)."""
        import torch
        if not items:
            return
        offs, cur = [], 0
        for it in items:
            offs.append(cur)
            cur += (it["info"].H * it["info"].W * 3 + 15) // 16 * 16
        with torch.cuda.device(self.device):
            buf = torch.empty(max(cur, 16), dtype=torch.uint8, device=self.device)
        here = torch.device(self.device)
        on_dev, up = [], []
        for it, o in zip(items, offs):
            png = it["png"]
            if isinstance(png, DevicePng) and png.buf.device == here and isinstance(it["info"], PngInfo) \
                    and it["info"].inflated is None:
                on_dev.append((it["info"], png, o))
            else:
                up.append((it["info"], bytes(png), o))
        self.stats["decode_launches"] += self.decoder.decode(up, buf)
        if on_dev:
            self.decoder.decode_device(on_dev, buf)
            self.stats["decode_launches"] += 1
        self.stats["device_frames"] += len(on_dev)
        for it, o in zip(items, offs):
            it["frame"] = (buf, o)

    def assemble(self, head, items: Sequence[dict], shape: Tuple[int, int, int], dtype):
        """-> CPU tensor [len(head) + len(items), *shape] of `dtype`: `head` (the master's frames, any device, or None)
        converted to dtype, then each item's frame as k / 255 in float32 (then dtype).  Pinned memory; the worker
        frames go through usdu_gather_unpack_f32 straight into it (or into a float32 pinned buffer when dtype is not
        float32)."""
        import torch
        from . import _native as nat
        M = 0 if head is None else int(head.shape[0])
        n = len(items)
        H, W, C = shape
        out = torch.empty((M + n, H, W, C), dtype=dtype, pin_memory=True)
        with torch.cuda.device(self.device):
            main = torch.cuda.current_stream()
            main.wait_stream(self.decoder.side)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            if M:
                out[:M].copy_(head, non_blocking=head.is_cuda)
            if n:
                dst = out[M:] if dtype == torch.float32 else torch.empty((n, H, W, C), dtype=torch.float32,
                                                                          pin_memory=True)
                ptrs = torch.tensor([buf.data_ptr() + o for buf, o in (it["frame"] for it in items)], dtype=torch.int64)
                ptrs = ptrs.to(self.device, non_blocking=False)
                nat.gather_unpack_f32(ptrs.data_ptr(), n, H * W * C, dst.data_ptr(), main.cuda_stream)
            e1.record()
            main.synchronize()
            if n and dtype != torch.float32:
                out[M:].copy_(dst)
        self.stats["assembly_ms"] = e0.elapsed_time(e1)
        self.stats["upload_ms"], self.stats["decode_ms"] = self.decoder.times()
        self.decoder.release()
        return out


# --------------------------------------------------------------------------------------
# the master role (nodes/collector.py:238-469)
# --------------------------------------------------------------------------------------
class HttpCollectorMaster:
    """One collector job with this process as the master of HTTP workers.  `frames` decodes and assembles (GpuFrames
    on the master's device unless given)."""

    def __init__(self, multi_job_id: str, enabled_workers: Sequence, store: CollectorStore = STORE, loop=None,
                 frames=None, device=None):
        self.multi_job_id = multi_job_id
        self.workers: List[str] = []
        for w in enabled_workers:                       # de-duplicated, in order (collector.py:247-255)
            if str(w) not in self.workers:
                self.workers.append(str(w))
        self.store, self.loop = store, loop if loop is not None else _server_loop()
        if self.loop is None:
            raise RuntimeError("HttpCollectorMaster: no server event loop")
        self.frames, self.device = frames, device
        self.stats: dict = {"bytes_received": 0}

    def _call(self, coro, timeout: Optional[float] = 10.0):
        return asyncio.run_coroutine_threadsafe(coro, self.loop).result(timeout)

    def run(self, images, audio=None, delegate_only: bool = False):
        """-> (images, audio) as the reference's master returns them."""
        import torch
        from .nodes.collector import combine_audio
        empty = {"waveform": torch.zeros(1, 2, 1), "sample_rate": EMPTY_AUDIO_SAMPLE_RATE}
        job = self.multi_job_id
        if self.frames is None:
            dev = self.device if self.device is not None else \
                images.device if images.is_cuda else torch.device("cuda", torch.cuda.current_device())
        else:
            dev = getattr(self.frames, "device", None)
        # the queue exists before any local work (collector.py:261-268); the route checks images on the master's device
        self._call(self.store.prepare(job, dev))
        try:
            if self.frames is None:
                self.frames = GpuFrames(dev)
            held, worker_audio = self._collect()
        finally:
            self._call(self.store.remove(job))
        head = None if delegate_only or images.shape[0] == 0 else images
        order = self.workers + sorted(w for w in held if w not in self.workers)
        items = [held[w][i] for w in order if w in held for i in sorted(held[w])]
        audios = [None if delegate_only else audio] + [worker_audio.get(w) for w in self.workers] + \
                 [worker_audio[w] for w in sorted(worker_audio) if w not in self.workers]
        self.stats.update(order=[w for w in order if w in held], frames={w: len(held[w]) for w in order if w in held})
        if not items:                                   # the master's frames alone, or the reference's fallback_images
            out = images.contiguous() if head is None else images.cpu().clone(memory_format=torch.contiguous_format)
            return out, combine_audio(audios, empty)
        shapes = {(it["info"].H, it["info"].W, 3) for it in items}
        if head is not None:
            shapes.add(tuple(int(v) for v in images.shape[1:]))
        if len(shapes) != 1:
            # torch.cat would fail: the reference's except returns the master's own images and audio
            self.stats["fallback"] = f"frames of different shapes: {sorted(shapes)}"
            return images, audio if audio is not None else empty
        dtype = torch.float32 if head is None else torch.promote_types(images.dtype, torch.float32)
        out = self.frames.assemble(head, items, shapes.pop(), dtype)
        self.stats.update(self.frames.stats)
        return out, combine_audio(audios, empty)

    def _collect(self):
        """collector.py:289-446: -> ({worker: {image_index: item}}, {worker: last audio})."""
        mm = _comfy_mm()
        job = self.multi_job_id
        expected, done = set(self.workers), set()
        held: Dict[str, Dict[int, dict]] = {}
        worker_audio: Dict[str, dict] = {}
        timeout = heartbeat_timeout()
        slice_s = min(max(0.1, heartbeat_interval() / 20.0), timeout)
        last_activity = time.time()

        def keep(item):
            held.setdefault(item["worker_id"], {})[item["image_index"]] = item
            if item["is_last"] and item["worker_id"] in expected:
                done.add(item["worker_id"])

        while len(done) < len(expected):
            if mm is not None:
                mm.throw_exception_if_processing_interrupted()
            got = self._call(self.store.take(job, slice_s), slice_s + 10.0)
            self.stats["bytes_received"] += sum(len(it["png"]) for it in got)
            if got:
                for item in got:
                    keep(item)
                    if item.get("audio") is not None:
                        worker_audio[item["worker_id"]] = item["audio"]
                self.frames.add(got)
                last_activity = time.time()
                timeout = heartbeat_timeout()
                continue
            if time.time() - last_activity < timeout:
                continue
            if mm is not None:
                mm.throw_exception_if_processing_interrupted()
            # the workers still missing timed out: take what is queued (its audio is not kept, collector.py:419-437)
            rest = self._call(self.store.drain(job))
            self.stats["bytes_received"] += sum(len(it["png"]) for it in rest)
            for item in rest:
                keep(item)
            self.frames.add(rest)
            break
        return held, worker_audio


def _comfy_mm():
    try:
        import comfy.model_management as mm
        return mm
    except ImportError:
        return None
