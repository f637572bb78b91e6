"""The static-mode master's host side (http_master.py): its routes against the reference's own (api/usdu_routes.py,
loaded by oracle/ref_static_run._Env), the PNG validation and segment table against PIL, and the job store's queue,
time-out and completion rules with a fake clock."""
import asyncio
import io
import json
import struct
import zlib

import numpy as np
import pytest
from PIL import Image

import ref_static_run
from __graft_entry__ import load_package

load_package()
from comfyui_distributed_b200 import http_master as hm  # noqa: E402
from comfyui_distributed_b200.http_worker import _call, encode_png, multipart  # noqa: E402

JOB = "jobM"


# --------------------------------------------------------------------------------------
# PNG corpus
# --------------------------------------------------------------------------------------
def png_of(arr: np.ndarray, level: int) -> bytes:
    bio = io.BytesIO()
    Image.fromarray(arr).save(bio, format="PNG", compress_level=level)
    return bio.getvalue()


def image(mode: str, h: int, w: int, seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    c = {"L": 1, "LA": 2, "RGB": 3, "RGBA": 4}[mode]
    # smooth ramps plus noise: PIL picks different filters row by row
    yy, xx = np.mgrid[0:h, 0:w]
    base = ((xx * 3 + yy * 5)[..., None] + np.arange(c) * 40) % 256
    a = np.where(rng.random((h, w, 1)) < 0.3, rng.integers(0, 256, (h, w, c)), base).astype(np.uint8)
    return a[..., 0] if c == 1 else a


CORPUS = ([(m, h, w) for m in ("L", "LA", "RGB", "RGBA") for h, w in ((1, 1), (1, 77), (53, 1), (37, 70))]
          + [("RGB", 544, 544), ("RGBA", 130, 260), ("L", 300, 300)])


def pil_rgb(data: bytes) -> np.ndarray:
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


# every corpus image at every compress level, except 544x544 at levels 0, 1, 6 and 9 only (the numpy model is slow)
@pytest.mark.parametrize("mode,h,w,level", [(m, h, w, lv) for m, h, w in CORPUS for lv in range(10)
                                            if (h, w) != (544, 544) or lv in (0, 1, 6, 9)])
def test_model_unfilter_equals_pil(mode, h, w, level):
    data = png_of(image(mode, h, w, h * 7 + w), level)
    info = hm.parse_png(data)
    assert (info.W, info.H) == (w, h)
    assert (info.inflated is None) == (level == 0)        # PIL's level 0 writes stored blocks
    assert hm.filtered_stream(info, data) == zlib.decompress(b"".join(_idat(data)))
    assert np.array_equal(hm.unfilter_model(info, data), pil_rgb(data))


def test_rows_straddle_stored_blocks():
    data = png_of(image("RGB", 544, 544, 1), 0)
    info = hm.parse_png(data)
    rowlen = 1 + 544 * 3
    starts = [s for _, s in info.segs]
    assert len(starts) > 10
    assert any(s % rowlen not in (0,) for s in starts[1:])        # some block boundary falls inside a row
    filters = set(np.frombuffer(hm.filtered_stream(info, data), np.uint8)[::rowlen].tolist())
    assert len(filters) >= 2, filters


def _chunks(data):
    pos, out = 8, []
    while pos < len(data):
        ln, = struct.unpack_from(">I", data, pos)
        out.append((data[pos + 4: pos + 8], pos, ln))
        pos += 12 + ln
    return out


def _idat(data):
    return [data[p + 8: p + 8 + ln] for t, p, ln in _chunks(data) if t == b"IDAT"]


def _flip(data, i, mask=0x40):
    d = bytearray(data)
    d[i] ^= mask
    return bytes(d)


def _corruptions(data):
    """(name, bytes) with one byte changed: a chunk CRC (IHDR, IDAT, IEND), IDAT data, the Adler-32, a filter byte,
    NLEN, LEN, the zlib header; and truncations."""
    ch = _chunks(data)
    ihdr, idat, iend = ch[0], [c for c in ch if c[0] == b"IDAT"], ch[-1]
    z = idat[0][1] + 8
    info = hm.parse_png(data)
    rowlen = 1 + info.W * info.C
    out = [("ihdr_crc", _flip(data, ihdr[1] + 8 + ihdr[2])), ("idat_crc", _flip(data, idat[0][1] + 8 + idat[0][2])),
           ("iend_crc", _flip(data, iend[1] + 8 + iend[2])), ("zlib_header", _flip(data, z)),
           ("adler", _flip(data, idat[-1][1] + 8 + idat[-1][2] - 1)), ("truncated", data[: z + 40]),
           ("no_signature", _flip(data, 1)), ("ihdr_depth", _flip(data, ihdr[1] + 8 + 8, 0x18))]
    if info.inflated is None:
        last = len(info.segs) - 1
        row = min(info.H - 1, 2)
        # the file offset of row `row`'s filter byte
        q = row * rowlen
        k = max(i for i, (_, s) in enumerate(info.segs) if s <= q)
        fb = info.segs[k][0] + q - info.segs[k][1]
        out += [("data", _flip(data, info.segs[last][0] + 3 if info.raw_len - info.segs[last][1] > 3 else fb)),
                ("nlen", _flip(data, info.segs[0][0] - 1)), ("len", _flip(data, info.segs[0][0] - 3, 0x01)),
                ("filter_7", bytes(data[:fb]) + b"\x07" + bytes(data[fb + 1:])),
                ("filter_swap", bytes(data[:fb]) + bytes([(data[fb] + 1) % 5]) + bytes(data[fb + 1:]))]
    else:
        out += [("data", _flip(data, z + 2 + len(_idat(data)[0]) // 2))]
    return out


@pytest.mark.parametrize("mode,h,w,level", [("RGB", 544, 544, 0), ("RGBA", 37, 70, 0), ("L", 53, 1, 0),
                                            ("LA", 37, 70, 0), ("RGB", 37, 70, 6), ("RGB", 1, 1, 0)])
def test_refused_exactly_when_pil_refuses(mode, h, w, level):
    data = png_of(image(mode, h, w, 3), level)
    for name, bad in _corruptions(data):
        try:
            want = pil_rgb(bad)
        except Exception:
            want = None
        try:
            info = hm.parse_png(bad)
        except ValueError:
            info = None
        assert (info is None) == (want is None), (name, want is None)
        if info is not None:
            assert np.array_equal(hm.unfilter_model(info, bad), want), name


def test_unsupported_pngs_are_refused():
    rgb = image("RGB", 20, 30, 5)
    for im in (Image.fromarray(rgb).convert("P"), Image.fromarray(image("L", 20, 30, 5).astype(np.uint16) * 200)):
        bio = io.BytesIO()
        im.save(bio, format="PNG")
        with pytest.raises(ValueError, match="unsupported"):
            hm.parse_png(bio.getvalue())
    data = bytearray(png_of(rgb, 0))         # set the interlace flag and fix the IHDR CRC
    data[8 + 8 + 12] = 1
    data[8 + 8 + 13: 8 + 8 + 17] = struct.pack(">I", zlib.crc32(bytes(data[8 + 4: 8 + 8 + 13])))
    with pytest.raises(ValueError, match="interlaced"):
        hm.parse_png(bytes(data))


# --------------------------------------------------------------------------------------
# the job store, fake clock
# --------------------------------------------------------------------------------------
def _geom(T):
    return [(0, 0, 8, 8, 8, 8)] * T


def test_store_requeue_is_last_duplicates_and_master_overwrite(monkeypatch):
    monkeypatch.setenv("COMFYUI_HEARTBEAT_TIMEOUT", "60")
    now = [1000.0]
    store = hm.JobStore(clock=lambda: now[0])

    async def go():
        await store.init_job(JOB, 2, _geom(4), ["w1", "w2"])
        job = store.jobs[JOB]
        assert job.worker_status == {"w1": 1000.0, "w2": 1000.0}
        for w, tid in (("w1", await job.pending.get()), ("w1", await job.pending.get()), ("w2", await job.pending.get())):
            job.assigned_to_workers[w].append(tid)
        assert job.assigned_to_workers == {"w1": [0, 1], "w2": [2]}
        # w1 completes tile 0 (both frames) and frame 0 of tile 1; w2 posts tile 0 frame 0 again
        t = lambda tid, b, tag: {"tile_idx": tid, "batch_idx": b, "global_idx": b * 4 + tid, "tag": tag}
        job.queue.put_nowait({"worker_id": "w1", "tiles": [t(0, 0, "a"), t(0, 1, "a"), t(1, 0, "a")], "is_last": False})
        job.queue.put_nowait({"worker_id": "w2", "tiles": [t(0, 0, "dup"), t(2, 0, "b"), t(2, 1, "b")], "is_last": True})
        kept = await store.drain(JOB)
        assert [(g, e["tag"]) for g, e in kept] == [(0, "a"), (4, "a"), (1, "a"), (2, "b"), (6, "b")]
        assert job.completed_tasks[0]["tag"] == "a"                 # the duplicate global_idx was ignored
        assert "w2" not in job.worker_status                        # is_last dropped w2
        # the master's own mark overwrites a worker's entry
        await store.mark_completed(JOB, 1, {"batch_idx": 0, "tile_idx": 1})
        assert job.completed_tasks[1] == {"batch_idx": 0, "tile_idx": 1}
        # not timed out yet: nothing moves
        now[0] += 60
        assert await store.requeue_timed_out(JOB) == 0
        # timed out: tile 1 (frame 1 missing) goes back, tile 0 (complete) does not
        now[0] += 1
        assert await store.requeue_timed_out(JOB) == 1
        assert "w1" not in job.worker_status and job.assigned_to_workers["w1"] == []
        left = [job.pending.get_nowait() for _ in range(job.pending.qsize())]
        assert sorted(left) == [1, 3]
        await store.cleanup(JOB)
        assert JOB not in store.jobs

    asyncio.run(go())


def test_store_heartbeat_keeps_a_worker(monkeypatch):
    monkeypatch.setenv("COMFYUI_HEARTBEAT_TIMEOUT", "5")
    now = [0.0]
    store = hm.JobStore(clock=lambda: now[0])

    async def go():
        await store.init_job(JOB, 1, _geom(2), ["w1"])
        job = store.jobs[JOB]
        job.assigned_to_workers["w1"].append(await job.pending.get())
        now[0] = 4.0
        job.worker_status["w1"] = store.clock()                   # a heartbeat
        now[0] = 8.0
        assert await store.requeue_timed_out(JOB) == 0
        now[0] = 9.5
        assert await store.requeue_timed_out(JOB) == 1

    asyncio.run(go())


# --------------------------------------------------------------------------------------
# routes against the reference's
# --------------------------------------------------------------------------------------
pytestmark_ref = pytest.mark.skipif(not ref_static_run.available(), reason="reference bundle (oracle/_ref) not present")


class _Servers:
    """The reference's routes (its own module-level job store) and ours (a JobStore), on one loop, two ports."""

    def __init__(self):
        from aiohttp import web
        self.env = ref_static_run._Env()
        self.store = hm.JobStore()
        routes = web.RouteTableDef()
        hm.register(routes, self.store, self.env.loop)
        app = web.Application(client_max_size=1 << 30)
        app.add_routes(routes)
        self.runner = web.AppRunner(app)
        self.port = ref_static_run._free_port()
        self.env._call(self.runner.setup())
        self.env._call(web.TCPSite(self.runner, "127.0.0.1", self.port).start())
        self.urls = {"ref": f"http://127.0.0.1:{self.env.port}", "ours": f"http://127.0.0.1:{self.port}"}

    def create(self, B, T, workers, geometry):
        js = self.env.mods["upscale.job_store"]
        self.env._call(js.init_static_job_batched(JOB, B, T, workers))
        self.env._call(self.store.init_job(JOB, B, geometry, workers))

    def both(self, method, path, body=None, ctype=None):
        out = {}
        for k, u in self.urls.items():
            status, text = _call(u + path, method, body, ctype)
            out[k] = (status, json.loads(text) if text else None)
        return out

    def close(self):
        try:
            self.env._call(self.runner.cleanup())
        finally:
            self.env.close()


def _json(obj):
    return json.dumps(obj).encode(), "application/json"


def _form(fields):
    return multipart([(k, v if isinstance(v, bytes) else str(v).encode(), fn, ct) for k, v, fn, ct in fields])


@pytestmark_ref
def test_routes_answer_as_the_reference(monkeypatch):
    monkeypatch.setenv("COMFYUI_MAX_PAYLOAD_SIZE", "300000")       # read when _Env loads the reference's job store
    tile = image("RGB", 24, 40, 9)
    png = encode_png(tile)
    geometry = [(8, 16, 40, 24, 40, 24), (40, 16, 40, 24, 40, 24)]
    meta = [{"tile_idx": 1, "x": 40, "y": 16, "extracted_width": 40, "extracted_height": 24, "batch_idx": 0,
             "global_idx": 1}]
    s = _Servers()
    try:
        def same(method, path, body=None, ctype=None, prefix=None):
            r = s.both(method, path, body, ctype)
            if prefix is None:
                assert r["ref"] == r["ours"], (path, r)
            else:          # the reference's message ends with PIL's exception text: compare the status and the prefix
                assert r["ref"][0] == r["ours"][0], (path, r)
                assert r["ref"][1]["error"].startswith(prefix) and r["ours"][1]["error"].startswith(prefix), r
            return r["ours"]

        head = [("multi_job_id", JOB, None, None), ("worker_id", "w1", None, None)]
        # unknown job
        assert same("GET", "/distributed/job_status?multi_job_id=" + JOB) == (200, {"ready": False})
        same("GET", "/distributed/job_status")
        assert same("POST", "/distributed/request_image", *_json({"worker_id": "w1", "multi_job_id": JOB}))[0] == 404
        assert same("POST", "/distributed/heartbeat", *_json({"worker_id": "w1", "multi_job_id": JOB}))[0] == 404
        assert same("POST", "/distributed/heartbeat", *_json({"worker_id": "w1"}))[0] == 400
        same("POST", "/distributed/heartbeat", b"not json", "application/json")
        assert same("POST", "/distributed/submit_tiles", *_form(head + [("is_last", "true", None, None),
                                                                         ("batch_size", "0", None, None)]))[0] == 400
        assert same("POST", "/distributed/submit_tiles", *_form(head + [
            ("padding", "8", None, None), ("tile_0", png, "t.png", "image/png"), ("is_last", "false", None, None),
            ("batch_size", "1", None, None), ("tiles_metadata", json.dumps(meta), None, "application/json")]))[0] == 404
        # job ready; tiles handed out, then the queue is empty
        s.create(1, 2, ["w1", "w2"], geometry)
        assert same("GET", "/distributed/job_status?multi_job_id=" + JOB) == (200, {"ready": True})
        assert same("POST", "/distributed/request_image", *_json({"worker_id": "w1", "multi_job_id": JOB})) == \
            (200, {"tile_idx": 0, "estimated_remaining": 1, "batched_static": True})
        assert same("POST", "/distributed/request_image", *_json({"worker_id": "w2", "multi_job_id": JOB}))[1]["tile_idx"] == 1
        assert same("POST", "/distributed/request_image", *_json({"worker_id": "w1", "multi_job_id": JOB})) == \
            (200, {"tile_idx": None})
        assert same("POST", "/distributed/request_image", *_json({"multi_job_id": JOB}))[0] == 400
        assert same("POST", "/distributed/heartbeat", *_json({"worker_id": "w1", "multi_job_id": JOB})) == \
            (200, {"status": "success"})
        # submit_tiles: size limit, form errors, corrupt PNG, a good tile, the completion signal
        assert same("POST", "/distributed/submit_tiles", *_form(head + [("blob", b"x" * 310000, None, None)]))[0] == 413
        assert same("POST", "/distributed/submit_tiles", *_form([("worker_id", "w1", None, None)]))[0] == 400
        assert same("POST", "/distributed/submit_tiles", *_form(head + [("batch_size", "1", None, None)]))[1] == \
            {"error": "Missing tiles_metadata"}
        same("POST", "/distributed/submit_tiles", *_form(head + [("tiles_metadata", "{bad", None, None)]))
        same("POST", "/distributed/submit_tiles", *_form(head + [("tiles_metadata", '{"a": 1}', None, None)]))
        same("POST", "/distributed/submit_tiles", *_form(head + [("batch_size", "x", None, None)]))
        assert same("POST", "/distributed/submit_tiles", *_form(head + [
            ("tiles_metadata", json.dumps(meta), None, None)]))[1] == {"error": "Missing tile data for index 0"}
        bad = _flip(png, len(png) - 18)           # inside the Adler-32 (IEND: 12 bytes, IDAT CRC: 4)
        assert same("POST", "/distributed/submit_tiles", *_form(head + [
            ("tile_0", bad, "t.png", "image/png"), ("tiles_metadata", json.dumps(meta), None, None)]),
            prefix="Invalid image data for tile 0: ")[0] == 400
        assert same("POST", "/distributed/submit_tiles", *_form(head + [
            ("padding", "8", None, None), ("tile_0", png, "t.png", "image/png"), ("is_last", "false", None, None),
            ("batch_size", "1", None, None), ("tiles_metadata", json.dumps(meta), None, None)])) == \
            (200, {"status": "success"})
        assert same("POST", "/distributed/submit_tiles", *_form(head + [("is_last", "true", None, None),
                                                                         ("batch_size", "0", None, None)])) == \
            (200, {"status": "success"})
        # submit_image: dynamic mode has no job here
        assert same("POST", "/distributed/submit_image", *_form(head + [("is_last", "true", None, None)])) == \
            (400, {"error": "Job not configured for image submissions"})
        assert same("POST", "/distributed/submit_image", *_form(head))[0] == 400
        # our extra checks: the window and the size must be the plan's
        wrong = [dict(meta[0], x=41)]
        r = s.both("POST", "/distributed/submit_tiles", *_form(head + [
            ("tile_0", png, "t.png", "image/png"), ("batch_size", "1", None, None),
            ("tiles_metadata", json.dumps(wrong), None, None)]))
        assert r["ref"][0] == 200 and r["ours"][0] == 400 and "differs from the plan" in r["ours"][1]["error"]
        small = encode_png(tile[:, :-1])
        r = s.both("POST", "/distributed/submit_tiles", *_form(head + [
            ("tile_0", small, "t.png", "image/png"), ("batch_size", "1", None, None),
            ("tiles_metadata", json.dumps(meta), None, None)]))
        assert r["ours"][0] == 400 and "processing size" in r["ours"][1]["error"]
        # what reached our queue: the good tile (bytes kept, not decoded), then the completion signal
        kept = s.env._call(s.store.drain(JOB))
        assert [(g, e["tile_idx"], e["png"] == png, e["padding"]) for g, e in kept] == [(1, 1, True, 8)]
        assert "w1" not in s.store.jobs[JOB].worker_status
    finally:
        s.close()


def test_register_skips_paths_served_elsewhere():
    from aiohttp import web
    routes = web.RouteTableDef()

    @routes.get("/distributed/job_status")
    async def other(request):      # another package got there first
        return web.json_response({})

    with pytest.warns(RuntimeWarning, match="already served"):
        served = hm.register(routes, hm.JobStore())
    assert ("GET", "/distributed/job_status") not in served and len(served) == 4
