"""Worker side of the reference's static-mode HTTP protocol (upscale/modes/static.py:191-314,
upscale/worker_comms.py:16-188), so that a stock reference master can hand tiles to a worker whose tile step runs on
this package's kernels (engine.WorkerJob), and the worker side of its DistributedCollector (nodes/collector.py:84-119,
`send_collector_batch`).

Blocking HTTP on the caller's thread (ComfyUI's prompt executor) with the standard library; no event loop.  What goes on
the wire is what the reference's worker sends: the job-ready poll, one `request_image` per tile, a heartbeat after every
tile, the processed tiles as level-0 PNGs in size-aware multipart chunks every COMFYUI_MAX_BATCH tiles, and `is_last` on
the final chunk (or the empty completion signal).  Retry counts, delays and timeouts are the reference's.
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
from typing import Callable, Iterable, List, Optional, Sequence, Tuple

import numpy as np

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

TileStep = Callable[[int], np.ndarray]
"""step(tile id) -> the processed tile of every frame, uint8 [B, ph, pw, 3] on the host."""


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
        """Pull tile ids until the master's queue is empty, processing each with `step` and uploading the results.
        False (nothing processed or sent) when the job never became ready, as static.py:222-224."""
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
            if out.dtype != np.uint8 or out.ndim != 4 or out.shape[0] != self.batch_size or out.shape[3] != 3:
                raise ValueError(f"tile step returned {out.dtype} {tuple(out.shape)}, expected uint8 [{self.batch_size}, h, w, 3]")
            x, y, ew, eh = self.geometry[tile_id]
            for b in range(self.batch_size):
                pending.append((encode_png(out[b]), {"tile_idx": tile_id, "x": x, "y": y, "extracted_width": ew,
                                                     "extracted_height": eh, "batch_idx": b,
                                                     "global_idx": b * n_tiles + tile_id}))
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
