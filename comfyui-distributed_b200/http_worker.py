"""Worker side of the reference's static-mode HTTP protocol (upscale/modes/static.py:191-314,
upscale/worker_comms.py:16-188), so that a stock reference master can hand tiles to a worker whose tile step runs on
this package's kernels (engine.WorkerJob), and the worker side of its DistributedCollector (nodes/collector.py:84-119,
`send_collector_batch`).

Blocking HTTP on the caller's thread (ComfyUI's prompt executor) with the standard library; no event loop.  What goes on
the wire is what the reference's worker sends: the job-ready poll, one `request_image` per tile, a heartbeat after every
tile, the processed tiles as level-0 PNGs in size-aware multipart chunks every COMFYUI_MAX_BATCH tiles, and `is_last` on
the final chunk (or the empty completion signal).  Retry counts, delays and timeouts are the reference's.

The tile PNGs are the bytes Pillow writes at compress_level=0.  They are encoded on the GPU (csrc/usdu_png.cu,
usdu_png_encode_u8) into a framing read off the installed Pillow for each tile shape (`png_layout`); a shape whose framing
fails its checks is PIL-encoded on the host, as before.
"""
from __future__ import annotations

import base64
import io
import json
import os
import time
import urllib.error
import urllib.parse
import urllib.request
import uuid
import warnings
from typing import Callable, Iterable, List, Optional, Sequence, Tuple, Union

import numpy as np

from .lru import LruCache

JOB_POLL_INTERVAL = 1.0            # utils/constants.py:53-54
JOB_POLL_MAX_ATTEMPTS = 20
STATUS_TIMEOUT = 5.0               # job-status poll and heartbeat (static.py:36-39, :295-298)
REQUEST_RETRIES = 10               # tile request (worker_comms.py:132-169)
REQUEST_TOTAL_TIMEOUT = 30.0
SEND_RETRIES = 5                   # tile upload (worker_comms.py:88-104)
TILE_SEND_TIMEOUT = 60.0           # utils/constants.py TILE_SEND_TIMEOUT
CHUNK_HEADROOM = 1024 * 1024       # worker_comms.py:49
TILE_OVERHEAD = 1024               # worker_comms.py:65
COLLECTOR_TIMEOUT = 60.0           # one job_complete POST (collector.py:110-116)

TileStep = Callable[[int], Union[np.ndarray, List[bytes]]]
"""step(tile id) -> the processed tile of every frame, uint8 [B, ph, pw, 3] on the host, or already as B PNG files."""


class HttpError(RuntimeError):
    def __init__(self, method: str, url: str, status: int, body: bytes):
        super().__init__(f"{method} {url}: HTTP {status}: {body[:200].decode('utf-8', 'replace')}")
        self.status = status


# no proxy from the environment: the master is addressed directly, like the reference's aiohttp session
_OPENER = urllib.request.build_opener(urllib.request.ProxyHandler({}))


def _call(url: str, method: str, body: Optional[bytes] = None, ctype: Optional[str] = None,
          timeout: float = STATUS_TIMEOUT) -> Tuple[int, bytes]:
    """One blocking request -> (status, body); an HTTP error status is returned, a connection error raises."""
    req = urllib.request.Request(url, data=body, method=method, headers={"Content-Type": ctype} if ctype else {})
    try:
        with _OPENER.open(req, timeout=timeout) as r:
            return r.status, r.read()
    except urllib.error.HTTPError as e:
        with e:
            return e.code, e.read()


def encode_png(tile: np.ndarray) -> bytes:
    """PIL PNG at compress_level=0, as worker_comms.py:30-34 (the master reads pixels, not bytes)."""
    from PIL import Image      # ComfyUI ships Pillow; only the HTTP worker needs it
    bio = io.BytesIO()
    Image.fromarray(np.ascontiguousarray(tile)).save(bio, format="PNG", compress_level=0)
    return bio.getvalue()


# --------------------------------------------------------------------------------------
# encode_png's bytes on the GPU: Pillow's framing for the shape + the filtered stream and checksums from the kernels
# --------------------------------------------------------------------------------------
class PngLayout:
    """The framing of Pillow's level-0 PNG of an RGB frame [H, W, 3], in the tables usdu_png_encode_u8 takes (see
    include/usdu_b200.h): `template` (a file of this shape), `runs` int64 [n, 3] (file offset, stream offset, length)
    of the filtered stream R inside it, `chunks` int64 [n, 2] (file offset, data length) of every IDAT chunk, and
    `adler_at`, the file offsets of the four Adler-32 bytes."""

    def __init__(self, H: int, W: int, template: bytes, runs: np.ndarray, chunks: np.ndarray, adler_at: Sequence[int]):
        self.H, self.W, self.template = int(H), int(W), bytes(template)
        self.runs = np.ascontiguousarray(runs, np.int64).reshape(-1, 3)
        self.chunks = np.ascontiguousarray(chunks, np.int64).reshape(-1, 2)
        self.adler_at = [int(p) for p in adler_at]
        self._device = {}
        self._check()

    @property
    def png_len(self) -> int:
        return len(self.template)

    @property
    def raw_len(self) -> int:
        return self.H * (1 + 3 * self.W)

    def _check(self):
        """ValueError unless the tables are what the kernels assume: runs cover R once, in order, inside IDAT data;
        the Adler bytes lie in IDAT data outside every run; chunks are sorted, disjoint and inside the file."""
        n = self.png_len
        if len(self.runs) == 0 or len(self.chunks) == 0 or len(self.adler_at) != 4:
            raise ValueError("empty layout")
        ends = self.runs[:, 1] + self.runs[:, 2]
        if (self.runs[0, 1] != 0 or ends[-1] != self.raw_len or (self.runs[1:, 1] != ends[:-1]).any()
                or (self.runs[:, 2] <= 0).any() or (np.diff(self.runs[:, 0]) <= 0).any()):
            raise ValueError("the runs do not cover the filtered stream in order")
        c_end = self.chunks[:, 0] + 12 + self.chunks[:, 1]
        if (self.chunks[:, 0] < 0).any() or (self.chunks[:, 1] < 0).any() or c_end[-1] > n or \
                (self.chunks[1:, 0] < c_end[:-1]).any():
            raise ValueError("IDAT chunks overlap or leave the file")
        data = np.zeros(n + 1, np.int64)              # +1 inside IDAT data, -1 (twice) for a run or Adler byte
        for off, ln in self.chunks.tolist():
            data[off + 8] += 1
            data[off + 8 + ln] -= 1
        in_data = np.cumsum(data)[:n] > 0
        used = np.zeros(n + 1, np.int64)
        for f, _, ln in self.runs.tolist():
            used[f] += 1
            used[f + ln] -= 1
        used = np.cumsum(used)[:n]
        used[self.adler_at] += 1
        if (used > 1).any() or not in_data[used > 0].all():
            raise ValueError("a run or an Adler byte lies outside IDAT data or on another one")

    def framing(self) -> tuple:
        """Everything that does not depend on pixel values: the tables and the template with R, the Adler bytes and
        the IDAT CRCs blanked."""
        t = np.frombuffer(self.template, np.uint8).copy()
        for f, _, ln in self.runs.tolist():
            t[f: f + ln] = 0
        t[self.adler_at] = 0
        for off, ln in self.chunks.tolist():
            t[off + 8 + ln: off + 12 + ln] = 0
        return (self.H, self.W, t.tobytes(), self.runs.tobytes(), self.chunks.tobytes(), tuple(self.adler_at))

    def device_tables(self, device):
        """(template, runs, chunks) on `device`, uploaded once per device."""
        import torch
        key = str(device)
        if key not in self._device:
            self._device[key] = tuple(torch.from_numpy(np.frombuffer(a, np.uint8).copy() if isinstance(a, bytes) else a)
                                      .to(device) for a in (self.template, self.runs, self.chunks))
        return self._device[key]


def layout_from_png(data: bytes) -> PngLayout:
    """The layout of one of Pillow's level-0 RGB PNGs, from http_master.parse_png's segment and chunk tables."""
    from .http_master import parse_png
    info = parse_png(data)
    if info.C != 3 or info.inflated is not None:
        raise ValueError("not a stored-block RGB PNG")
    starts = [r for _, r in info.segs] + [info.raw_len]
    runs = [(off, r, starts[i + 1] - r) for i, (off, r) in enumerate(info.segs)]
    return PngLayout(info.H, info.W, data, np.asarray(runs, np.int64), np.asarray(info.idat, np.int64), info.trailer)


def png_probe(H: int, W: int, variant: int = 0) -> np.ndarray:
    """A u8 RGB frame [H, W, 3] on which, given seven rows and four columns or more, each of Pillow's filters None, Up,
    Sub and Paeth wins on some row.  Rows cycle through noise, a duplicate of the row above (Up), a horizontal ramp
    (Sub), a zero row, a row constant on its left half and noisy on its right, a row constant on its left half with
    another value and a copy of the row above on its right (Paeth: Sub wins on the left, Up on the right), and values
    126..130 (the cost's wrap).  Row 0, with zeros above it, ties None with Up and Sub with Paeth.  `variant` changes
    the values, not the shape."""
    v = int(variant) % 64
    rng = np.random.default_rng(1000 + v)
    x = np.arange(W, dtype=np.int64)[:, None]
    half = W // 2
    img = np.zeros((H, W, 3), np.uint8)
    for r in range(H):
        k = r % 7
        if k == 0:
            img[r] = rng.integers(0, 256, (W, 3))
        elif k == 1:
            img[r] = img[r - 1]
        elif k == 2:
            img[r] = (2 * x + 40 * v + np.array([0, 85, 170])) % 256
        elif k == 4:
            img[r, :half] = 50 + v
            img[r, half:] = rng.integers(0, 256, (W - half, 3))
        elif k == 5:
            img[r, :half] = 180 + v
            img[r, half:] = img[r - 1, half:]
        elif k == 6:
            img[r] = rng.integers(126, 131, (W, 3))
    return img


def encode_png_gpu(frames, layout: PngLayout, out, scratch=None):
    """Enqueue usdu_png_encode_u8 on the current stream: frames = contiguous CUDA u8 [B, H, W, 3], out = CUDA u8 of at
    least B * layout.png_len bytes, frame b's file at out[b * png_len:]."""
    import torch
    from . import _native as nat
    B, H, W, C = frames.shape
    if (H, W, C) != (layout.H, layout.W, 3) or frames.dtype != torch.uint8 or not frames.is_contiguous():
        raise ValueError(f"frames {frames.dtype} {tuple(frames.shape)} do not fit a layout of {layout.H}x{layout.W}")
    if out.numel() < B * layout.png_len:
        raise ValueError(f"output of {out.numel()} bytes for {B} files of {layout.png_len}")
    if scratch is None:
        scratch = torch.empty(nat.png_encode_scratch_bytes(B, H, W), dtype=torch.uint8, device=frames.device)
    tmpl, runs, chunks = layout.device_tables(frames.device)
    nat.png_encode_u8(frames.data_ptr(), B, H, W, 3, tmpl.data_ptr(), layout.png_len, runs.data_ptr(), len(layout.runs),
                      chunks.data_ptr(), len(layout.chunks), layout.adler_at, scratch.data_ptr(), out.data_ptr(),
                      torch.cuda.current_stream(frames.device).cuda_stream)
    return out


def _checked_layout(H: int, W: int, device) -> PngLayout:
    """Pillow's framing for [H, W, 3], checked: two probes of different content must frame alike, and the kernels must
    reproduce Pillow's bytes of both.  ValueError otherwise."""
    import torch
    probes = [png_probe(H, W, v) for v in (0, 1)]
    files = [encode_png(p) for p in probes]
    layout = layout_from_png(files[0])
    if layout_from_png(files[1]).framing() != layout.framing():
        raise ValueError("Pillow's framing depends on the pixel values")
    with torch.cuda.device(device):
        frames = torch.from_numpy(np.stack(probes)).to(device)
        out = torch.empty(2 * layout.png_len, dtype=torch.uint8, device=device)
        encode_png_gpu(frames, layout, out)
        got = out.cpu().numpy().tobytes()
    if got != b"".join(files):
        raise ValueError("the GPU encoder's bytes differ from Pillow's")
    return layout


_LAYOUTS: LruCache = LruCache(32)


def png_layout(H: int, W: int, device=None) -> Optional[PngLayout]:
    """The checked layout of [H, W, 3] tiles, or None (after one warning per shape) when the installed Pillow's bytes
    cannot be reproduced: that shape's tiles are then PIL-encoded on the host."""
    import torch
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    key = (int(H), int(W), str(device))
    if key in _LAYOUTS:
        return _LAYOUTS.get(key)
    try:
        layout = _checked_layout(int(H), int(W), device)
    except (ValueError, TypeError) as e:
        warnings.warn(f"PNG tiles of {W}x{H} are encoded with PIL on the host: {e}", RuntimeWarning, stacklevel=2)
        layout = None
    return _LAYOUTS.put(key, layout)


def multipart(parts: Sequence[Tuple[str, bytes, Optional[str], Optional[str]]]) -> Tuple[bytes, str]:
    """(name, value, filename, content type) parts -> (multipart/form-data body, its Content-Type header)."""
    boundary = uuid.uuid4().hex
    out = io.BytesIO()
    for name, value, filename, ctype in parts:
        disp = f'form-data; name="{name}"' + (f'; filename="{filename}"' if filename else "")
        out.write(f"--{boundary}\r\nContent-Disposition: {disp}\r\n".encode())
        if ctype:
            out.write(f"Content-Type: {ctype}\r\n".encode())
        out.write(b"\r\n")
        out.write(value)
        out.write(b"\r\n")
    out.write(f"--{boundary}--\r\n".encode())
    return out.getvalue(), f"multipart/form-data; boundary={boundary}"


def _interrupt_poll():
    try:        # ComfyUI's user cancel, polled once per tile
        import comfy.model_management as mm
        return mm.throw_exception_if_processing_interrupted
    except ImportError:
        return None


class HttpStaticWorker:
    """One static-mode worker of the reference's master for one job.  `geometry[t]` = (x, y, extracted_width,
    extracted_height) of tile t's crop window, which the master needs to place the tile; `batch_size` frames per tile."""

    def __init__(self, master_url: str, multi_job_id: str, worker_id: str, padding: int,
                 geometry: Sequence[Tuple[int, int, int, int]], batch_size: int):
        self.master_url = master_url
        self.multi_job_id = multi_job_id
        self.worker_id = str(worker_id)
        self.padding = int(padding)
        self.geometry = [tuple(int(v) for v in g) for g in geometry]
        self.batch_size = int(batch_size)
        self.max_batch = int(os.environ.get("COMFYUI_MAX_BATCH", "20"))
        self.max_payload = int(os.environ.get("COMFYUI_MAX_PAYLOAD_SIZE", str(50 * 1024 * 1024)))
        self.pulled: List[int] = []        # tile ids in processing order
        self.chunks = 0                    # tile uploads (multipart POSTs with tiles)
        self.times = {"request_s": 0.0, "step_s": 0.0, "encode_s": 0.0, "post_s": 0.0, "heartbeat_s": 0.0}

    # -- HTTP ---------------------------------------------------------------------------
    def _call(self, method: str, path: str, body: Optional[bytes] = None, ctype: Optional[str] = None,
              timeout: float = STATUS_TIMEOUT) -> Tuple[int, bytes]:
        return _call(self.master_url + path, method, body, ctype, timeout)

    def _post_json(self, path: str, obj: dict, timeout: float) -> Tuple[int, bytes]:
        return self._call("POST", path, json.dumps(obj).encode(), "application/json", timeout)

    def _post_form(self, parts, retries: int):
        body, ctype = multipart(parts)
        path = "/distributed/submit_tiles"
        delay = 0.5
        for attempt in range(retries):
            try:
                status, text = self._call("POST", path, body, ctype, TILE_SEND_TIMEOUT)
                if status >= 400:
                    raise HttpError("POST", self.master_url + path, status, text)
                return
            except Exception:
                if attempt == retries - 1:
                    raise
                time.sleep(delay)
                delay = min(delay * 2, 5.0)

    # -- protocol steps -----------------------------------------------------------------
    def wait_ready(self) -> bool:
        """Poll the master until it has created the job (static.py:33-47): False after 20 tries 1 s apart."""
        path = "/distributed/job_status?multi_job_id=" + urllib.parse.quote(self.multi_job_id, safe="")
        for _ in range(JOB_POLL_MAX_ATTEMPTS):
            try:
                status, body = self._call("GET", path)
                if status == 200 and json.loads(body).get("ready", False):
                    return True
            except Exception:      # unreachable master: not ready yet (worker_comms.py:246-258)
                pass
            time.sleep(JOB_POLL_INTERVAL)
        return False

    def request_tile(self) -> Optional[int]:
        """The next tile id, or None when the queue is empty or the master stops answering (worker_comms.py:124-188):
        404 = job not there yet, wait 1 s; any other status, try again at once; a connection error, back off and raise
        on the last of 10 attempts; give up after 30 s."""
        delay = 0.5
        start = time.monotonic()
        for attempt in range(REQUEST_RETRIES):
            if time.monotonic() - start > REQUEST_TOTAL_TIMEOUT:
                return None
            try:
                status, body = self._post_json("/distributed/request_image",
                                               {"worker_id": self.worker_id, "multi_job_id": self.multi_job_id},
                                               REQUEST_TOTAL_TIMEOUT)
                if status == 200:
                    tile = json.loads(body).get("tile_idx")
                    return None if tile is None else int(tile)
                if status == 404:
                    time.sleep(1.0)
            except Exception:
                if attempt == REQUEST_RETRIES - 1:
                    raise
                time.sleep(delay)
                delay = min(delay * 2, 5.0)
        return None

    def heartbeat(self):
        """POST /distributed/heartbeat; failures are ignored (utils/usdu_managment.py:28-37)."""
        try:
            self._post_json("/distributed/heartbeat", {"multi_job_id": self.multi_job_id, "worker_id": self.worker_id},
                            STATUS_TIMEOUT)
        except Exception:
            pass

    def send(self, tiles: List[Tuple[bytes, dict]], final: bool):
        """Upload (png, metadata) entries in chunks under COMFYUI_MAX_PAYLOAD_SIZE - 1 MB (worker_comms.py:16-108);
        `final` marks the last chunk `is_last`.  No tiles and `final`: the completion signal alone (:110-122)."""
        head = [("multi_job_id", self.multi_job_id.encode(), None, None), ("worker_id", self.worker_id.encode(), None, None)]
        if not tiles:
            if final:
                self._post_form(head + [("is_last", b"true", None, None), ("batch_size", b"0", None, None)], retries=1)
            return
        max_bytes = self.max_payload - CHUNK_HEADROOM
        i = 0
        while i < len(tiles):
            used, j = 0, i
            while j < len(tiles):          # the first tile of a chunk always goes in, however large
                if used + len(tiles[j][0]) + TILE_OVERHEAD > max_bytes and j > i:
                    break
                used += len(tiles[j][0]) + TILE_OVERHEAD
                j += 1
            parts = head + [("padding", str(self.padding).encode(), None, None)]
            parts += [(f"tile_{k - i}", tiles[k][0], f"tile_{k}.png", "image/png") for k in range(i, j)]
            parts += [("is_last", str(bool(final and j >= len(tiles))).encode(), None, None),
                      ("batch_size", str(j - i).encode(), None, None),
                      ("tiles_metadata", json.dumps([tiles[k][1] for k in range(i, j)]).encode(), None, "application/json")]
            self._post_form(parts, SEND_RETRIES)
            self.chunks += 1
            i = j

    def run(self, step: TileStep) -> bool:
        """Pull tile ids until the master's queue is empty, processing each with `step` and uploading the results.  A
        step returns either the u8 tiles (PIL-encoded here) or their B PNG files (WorkerJob.step_png).  False (nothing processed or sent) when the job never became ready, as static.py:222-224."""
        poll = _interrupt_poll()
        if not self.wait_ready():
            return False
        n_tiles = len(self.geometry)
        pending: List[Tuple[bytes, dict]] = []
        clock = time.perf_counter
        while True:
            if poll is not None:
                poll()
            t0 = clock()
            tile_id = self.request_tile()
            t1 = clock()
            self.times["request_s"] += t1 - t0
            if tile_id is None:
                break
            if not 0 <= tile_id < n_tiles:
                raise ValueError(f"master handed out tile {tile_id}; this job has {n_tiles} tiles")
            self.pulled.append(tile_id)
            out = step(tile_id)
            t2 = clock()
            if isinstance(out, (list, tuple)):
                if len(out) != self.batch_size or not all(isinstance(f, (bytes, bytearray)) for f in out):
                    raise ValueError(f"tile step returned {len(out)} items, expected {self.batch_size} PNG files")
                pngs = [bytes(f) for f in out]
            else:
                if out.dtype != np.uint8 or out.ndim != 4 or out.shape[0] != self.batch_size or out.shape[3] != 3:
                    raise ValueError(f"tile step returned {out.dtype} {tuple(out.shape)}, expected uint8 [{self.batch_size}, h, w, 3]")
                pngs = [encode_png(out[b]) for b in range(self.batch_size)]
            x, y, ew, eh = self.geometry[tile_id]
            for b in range(self.batch_size):
                pending.append((pngs[b], {"tile_idx": tile_id, "x": x, "y": y, "extracted_width": ew,
                                          "extracted_height": eh, "batch_idx": b, "global_idx": b * n_tiles + tile_id}))
            t3 = clock()
            self.heartbeat()
            t4 = clock()
            if len(pending) >= self.max_batch:
                self.send(pending, final=False)
                pending = []
            t5 = clock()
            self.times["step_s"] += t2 - t1
            self.times["encode_s"] += t3 - t2
            self.times["heartbeat_s"] += t4 - t3
            self.times["post_s"] += t5 - t4
        t0 = clock()
        self.send(pending, final=True)
        self.times["post_s"] += clock() - t0
        return True


# --------------------------------------------------------------------------------------
# DistributedCollector worker (nodes/collector.py:84-119 -> api/job_routes.py:273-343)
# --------------------------------------------------------------------------------------
def max_audio_payload_bytes() -> int:
    return int(os.environ.get("COMFYUI_MAX_AUDIO_PAYLOAD_BYTES", str(256 * 1024 * 1024)))


def encode_audio_payload(audio) -> Optional[dict]:
    """The reference's audio envelope (utils/audio_payload.py:16-43): a float32 contiguous waveform's bytes in base64,
    its shape, dtype "float32" and int(sample_rate) (44100 when that fails).  None for no audio or an empty waveform;
    ValueError over COMFYUI_MAX_AUDIO_PAYLOAD_BYTES."""
    import torch
    if not isinstance(audio, dict):
        return None
    wave = audio.get("waveform")
    if wave is None or not isinstance(wave, torch.Tensor) or wave.numel() == 0:
        return None
    try:
        rate = int(audio.get("sample_rate", 44100))
    except (TypeError, ValueError):
        rate = 44100
    w = wave.detach().to(device="cpu", dtype=torch.float32).contiguous()
    data = w.numpy().tobytes()
    limit = max_audio_payload_bytes()
    if len(data) > limit:
        raise ValueError(f"Audio payload too large: {len(data)} bytes exceeds {limit}.")
    return {"sample_rate": rate, "shape": [int(d) for d in w.shape], "dtype": "float32",
            "data": base64.b64encode(data).decode("ascii")}


def collector_body(job_id: str, worker_id: str, batch_idx: int, text, is_last: bool,
                   audio_json: Optional[bytes] = None) -> bytes:
    """The JSON envelope of one image, built as bytes around the base64 text (which needs no escaping):
    {"job_id", "worker_id", "batch_idx", "image": "data:image/png;base64,...", "is_last"[, "audio"]}."""
    head = (b'{"job_id": ' + json.dumps(str(job_id)).encode() + b', "worker_id": ' + json.dumps(str(worker_id)).encode()
            + b', "batch_idx": ' + str(int(batch_idx)).encode() + b', "image": "data:image/png;base64,')
    tail = b'", "is_last": ' + (b"true" if is_last else b"false")
    if audio_json is not None:
        tail += b', "audio": ' + audio_json
    return b"".join((head, text, tail, b"}"))


def send_collector_batch(master_url: str, job_id: str, worker_id: str, count: int, texts: Iterable, audio=None,
                         post_times: Optional[List[float]] = None) -> int:
    """POST `count` images to {master_url}/distributed/job_complete, one per image in batch order, `is_last` on the
    last, the audio envelope beside it.  `texts` yields each image's base64 PNG text (bytes-like) and is only advanced
    after the previous image was posted.  Any status >= 400 or connection error raises, with no retry, as the
    reference re-raises.  count = 0 sends nothing.  -> images sent."""
    if count == 0:
        return 0
    audio_payload = encode_audio_payload(audio)
    audio_json = None if audio_payload is None else json.dumps(audio_payload).encode()
    url = master_url + "/distributed/job_complete"
    sent = 0
    for text in texts:
        if sent >= count:
            raise ValueError(f"more than {count} images to send")
        last = sent == count - 1
        body = collector_body(job_id, worker_id, sent, text, last, audio_json if last else None)
        t0 = time.perf_counter()
        status, reply = _call(url, "POST", body, "application/json", COLLECTOR_TIMEOUT)
        if post_times is not None:
            post_times.append(time.perf_counter() - t0)
        if status >= 400:
            raise HttpError("POST", url, status, reply)
        sent += 1
    if sent != count:
        raise ValueError(f"{sent} of {count} images encoded")
    return sent
