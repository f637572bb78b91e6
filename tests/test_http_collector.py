"""The collector master's host side (http_collector.py): its job_complete and prepare_job routes against the
reference's own (api/job_routes.py, loaded through tests/collector_master.load), the master role's collect rules with a
numpy stand-in for the GPU decode and assembly, and the numpy un-filter model on rows wider than the tile limit."""
import base64
import io
import json
import sys
import threading
import types
import zlib

import numpy as np
import pytest
import torch
from PIL import Image

import collector_master
from __graft_entry__ import load_package
from test_http_master import _corruptions, image, png_of

load_package()
from comfyui_distributed_b200 import _native as nat  # noqa: E402
from comfyui_distributed_b200 import http_collector as hc  # noqa: E402
from comfyui_distributed_b200 import http_master as hm  # noqa: E402
from comfyui_distributed_b200.http_worker import _call  # noqa: E402
from comfyui_distributed_b200.nodes import collector  # noqa: E402

JOB = "jobC"
needs_ref = pytest.mark.skipif(not collector_master.available(), reason="reference bundle (oracle/_ref) not present")


def data_url(png: bytes) -> str:
    return "data:image/png;base64," + base64.b64encode(png).decode()


def audio_env(wave: torch.Tensor, rate=48000) -> dict:
    w = wave.to(torch.float32).contiguous()
    return {"sample_rate": rate, "shape": list(w.shape), "dtype": "float32",
            "data": base64.b64encode(w.numpy().tobytes()).decode()}


def body(worker, idx, png, is_last, audio=None, job=JOB) -> bytes:
    d = {"job_id": job, "worker_id": worker, "batch_idx": idx, "image": data_url(png), "is_last": is_last}
    if audio is not None:
        d["audio"] = audio
    return json.dumps(d).encode()


def u8_png(seed, h, w, level=0) -> bytes:
    return png_of(image("RGB", h, w, seed), level)


# --------------------------------------------------------------------------------------
# this package's routes on an in-process server
# --------------------------------------------------------------------------------------
class Ours:
    """http_collector's routes (module store) on 127.0.0.1, served from its own loop thread; `bodies` holds every POST
    body that reached job_complete, in arrival order."""

    def __init__(self, loop=None):
        import asyncio
        from aiohttp import web
        hc.reset_for_tests()
        self.own_loop = loop is None
        self.loop = loop or asyncio.new_event_loop()
        if self.own_loop:
            self.thread = threading.Thread(target=self.loop.run_forever, daemon=True)
            self.thread.start()
        self.bodies = []

        @web.middleware
        async def record(request, handler):
            if request.path == "/distributed/job_complete":
                self.bodies.append(await request.read())
            return await handler(request)

        routes = web.RouteTableDef()
        assert hc.register(routes, hc.STORE, self.loop) == set(hc.COLLECTOR_ROUTES)
        app = web.Application(client_max_size=1 << 30, middlewares=[record])
        app.add_routes(routes)
        self.runner = web.AppRunner(app)
        self.call(self.runner.setup())
        self.port = _free_port()
        self.call(web.TCPSite(self.runner, "127.0.0.1", self.port).start())
        self.url = f"http://127.0.0.1:{self.port}"
        assert hc.serving()

    def call(self, coro, timeout=60):
        import asyncio
        return asyncio.run_coroutine_threadsafe(coro, self.loop).result(timeout)

    def close(self):
        try:
            self.call(self.runner.cleanup())
        finally:
            hc.reset_for_tests()
            if self.own_loop:
                self.loop.call_soon_threadsafe(self.loop.stop)
                self.thread.join(10)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def _free_port() -> int:
    import socket
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def post(url, raw: bytes, path="/distributed/job_complete"):
    status, text = _call(url + path, "POST", raw, "application/json", timeout=120)
    return status, json.loads(text) if text else None


class NumpyFrames:
    """http_collector.GpuFrames in numpy: the decode is http_master.unfilter_model, the assembly torch.cat of the
    master's frames with np.float32(k) / 255 of each worker frame."""

    def __init__(self):
        self.stats = {"upload_ms": 0.0, "decode_ms": 0.0, "assembly_ms": 0.0, "decode_launches": 0}
        self.added = []

    def add(self, items):
        for it in items:
            it["frame"] = hm.unfilter_model(it["info"], it["png"])
        self.added.append(len(items))

    def assemble(self, head, items, shape, dtype):
        parts = [] if head is None else [head.cpu().to(dtype)]
        parts += [torch.from_numpy(it["frame"].astype(np.float32) / 255)[None].to(dtype) for it in items]
        return torch.cat(parts, 0)


# --------------------------------------------------------------------------------------
# routes against the reference's
# --------------------------------------------------------------------------------------
class RefRoutes:
    """The reference's job_complete and prepare_job handlers on the loop of `ours`, on a second port."""

    def __init__(self, loop):
        import asyncio
        from aiohttp import web
        _, routes, _ = collector_master.load()
        self.mod = routes
        inst = routes.prompt_server
        inst.distributed_pending_jobs = {}
        self.loop = loop

        async def make_lock():
            inst.distributed_jobs_lock = asyncio.Lock()
        asyncio.run_coroutine_threadsafe(make_lock(), loop).result(10)
        self.inst = inst
        app = web.Application(client_max_size=1 << 30)
        app.router.add_post("/distributed/job_complete", routes.job_complete_endpoint)
        app.router.add_post("/distributed/prepare_job", routes.prepare_job_endpoint)
        self.runner = web.AppRunner(app)
        asyncio.run_coroutine_threadsafe(self.runner.setup(), loop).result(10)
        self.port = _free_port()
        asyncio.run_coroutine_threadsafe(web.TCPSite(self.runner, "127.0.0.1", self.port).start(), loop).result(10)
        self.url = f"http://127.0.0.1:{self.port}"

    def close(self):
        import asyncio
        asyncio.run_coroutine_threadsafe(self.runner.cleanup(), self.loop).result(10)


def _route_table():
    """(name, raw body, prefix) -- prefix: compare only the start of the error message (PIL's text follows it)."""
    png = u8_png(1, 9, 13)
    good = {"job_id": JOB, "worker_id": "w1", "batch_idx": 0, "image": data_url(png), "is_last": False}
    j = lambda **kw: json.dumps({**good, **kw}).encode()
    wave = torch.rand(1, 2, 30, generator=torch.Generator().manual_seed(2))
    env = audio_env(wave)
    rows = [("invalid_json", b"{not json", None), ("array", b"[1, 2]", None), ("string", b'"x"', None),
            ("job_id_empty", j(job_id=" "), None), ("job_id_int", j(job_id=5), None),
            ("worker_id_missing", json.dumps({k: v for k, v in good.items() if k != "worker_id"}).encode(), None),
            ("batch_idx_negative", j(batch_idx=-1), None), ("batch_idx_str", j(batch_idx="0"), None),
            ("batch_idx_float", j(batch_idx=1.0), None), ("image_empty", j(image="  "), None),
            ("image_int", j(image=3), None), ("audio_list", j(audio=[1]), None), ("is_last_str", j(is_last="true"), None),
            ("is_last_missing", json.dumps({k: v for k, v in good.items() if k != "is_last"}).encode(), None),
            ("all_fields", json.dumps({"job_id": "", "worker_id": 1, "batch_idx": -2, "image": "", "audio": 7,
                                       "is_last": 0}).encode(), None),
            ("data_url_no_comma", j(image="data:image/png;base64" + base64.b64encode(png).decode()), None),
            ("data_url_jpeg", j(image="data:image/jpeg;base64," + base64.b64encode(png).decode()), None),
            ("data_url_upper", j(image="DATA:image/png;base64," + base64.b64encode(png).decode()), None),
            ("b64_alphabet", j(image="iVBOR$$w0KGgo="), None), ("b64_padding", j(image="iVBORw0KGgo"), None),
            ("b64_non_ascii", j(image="iVBORw0KGgoé"), None), ("b64_empty", j(image="data:image/png;base64,"), None),
            ("not_png", j(image=base64.b64encode(b"GIF89a not an image").decode()), "Failed to decode PNG image payload: "),
            ("bare_base64", j(image=base64.b64encode(png).decode()), None),
            ("whitespace", j(image="  " + data_url(png) + "\n"), None)]
    for mode, h, w, level in (("RGBA", 37, 70, 0), ("L", 53, 1, 0), ("LA", 37, 70, 0), ("RGB", 37, 70, 6), ("RGB", 1, 1, 0)):
        for name, bad in _corruptions(png_of(image(mode, h, w, 4), level)):
            rows.append((f"png_{mode}_{level}_{name}", j(image=data_url(bad)), "Failed to decode PNG image payload: "))
    aud = lambda **kw: j(audio={**env, **kw}, is_last=True)
    rows += [("audio_no_data", j(audio={k: v for k, v in env.items() if k != "data"}), None),
             ("audio_data_empty", aud(data=" "), None), ("audio_shape_2", aud(shape=[2, 30]), None),
             ("audio_shape_str", aud(shape="1,2,30"), None), ("audio_dtype", aud(dtype="float16"), None),
             ("audio_shape_items", aud(shape=[1, "two", 30]), None), ("audio_shape_zero", aud(shape=[0, 2, 30]), None),
             ("audio_samples_negative", aud(shape=[1, 2, -1]), None), ("audio_rate_str", aud(sample_rate="fast"), None),
             ("audio_rate_zero", aud(sample_rate=0), None), ("audio_b64", aud(data="AAA$"), None),
             ("audio_size", aud(shape=[1, 2, 31]), None), ("audio_too_large", aud(data=base64.b64encode(
                 np.zeros(2 * 2 * 40, np.float32).tobytes()).decode(), shape=[2, 2, 40]), None),
             ("audio_good", aud(), None), ("good", j(), None), ("good_last", j(is_last=True, batch_idx=1), None)]
    return rows


@needs_ref
def test_routes_answer_as_the_reference(monkeypatch):
    ours = Ours()
    ref = RefRoutes(ours.loop)
    monkeypatch.setattr(ref.mod, "JOB_INIT_GRACE_PERIOD", 0.3)
    monkeypatch.setattr(hc, "JOB_INIT_GRACE_PERIOD", 0.3)
    ap = sys.modules[f"{collector_master.PKG}.utils.audio_payload"]
    monkeypatch.setattr(ap, "MAX_AUDIO_PAYLOAD_BYTES", 2 * 2 * 30 * 4 + 8)
    monkeypatch.setenv("COMFYUI_MAX_AUDIO_PAYLOAD_BYTES", str(2 * 2 * 30 * 4 + 8))
    try:
        def same(raw, prefix=None, path="/distributed/job_complete", name=""):
            r, o = post(ref.url, raw, path), post(ours.url, raw, path)
            if prefix is None or r[0] < 400:           # some corruptions PIL accepts (the IDAT and IEND CRCs)
                assert r == o, (name, r, o)
            else:
                assert r[0] == o[0] and r[1]["error"].startswith(prefix) and o[1]["error"].startswith(prefix), \
                    (name, r, o)
            return o

        table = _route_table()
        # no job yet: every request that passes the checks waits out the grace period, then 404
        assert same(table[-1][1], name="unknown job") == (404, {"error": "job not initialized"})
        # prepare_job
        same(b"{bad", path="/distributed/prepare_job")
        same(b"[]", path="/distributed/prepare_job")
        assert same(b"{}", path="/distributed/prepare_job")[0] == 400
        assert same(json.dumps({"multi_job_id": JOB}).encode(), path="/distributed/prepare_job") == \
            (200, {"status": "success"})
        accepted = []
        for name, raw, prefix in table:
            status, _ = same(raw, prefix, name=name)
            if status == 200:
                accepted.append(json.loads(raw))
        assert {n for n, *_ in table} >= {"good", "audio_good"} and len(accepted) >= 4
        # what reached our queue: the accepted POSTs in order, PNG bytes kept (not decoded), audio decoded
        items = ours.call(hc.STORE.drain(JOB))
        assert len(items) == len(accepted) == ref.inst.distributed_pending_jobs[JOB].qsize()
        for it, d in zip(items, accepted):
            assert it["png"] == base64.b64decode(d["image"].strip().partition(",")[2] or d["image"].strip())
            assert set(it) == {"png", "info", "worker_id", "image_index", "is_last", "audio"}
            assert (it["worker_id"], it["image_index"], it["is_last"]) == (d["worker_id"], d["batch_idx"], d["is_last"])
            assert (it["audio"] is None) == ("audio" not in d)
    finally:
        ref.close()
        ours.close()


def test_register_skips_paths_served_elsewhere():
    from aiohttp import web
    routes = web.RouteTableDef()

    @routes.post("/distributed/job_complete")
    async def other(request):
        return web.json_response({})

    with pytest.warns(RuntimeWarning, match="already served"):
        served = hc.register(routes, hc.CollectorStore())
    assert served == {("POST", "/distributed/prepare_job")}


def test_install_in_comfyui_serves_both_route_sets(monkeypatch):
    from aiohttp import web
    inst = types.SimpleNamespace(routes=web.RouteTableDef(), loop=object())
    monkeypatch.setitem(sys.modules, "server", types.SimpleNamespace(PromptServer=types.SimpleNamespace(instance=inst)))
    hm.reset_for_tests()
    hc.reset_for_tests()
    try:
        hm.install_in_comfyui()
        paths = {(r.method, r.path) for r in inst.routes}
        assert set(hm.MASTER_ROUTES) <= paths and set(hc.COLLECTOR_ROUTES) <= paths
        assert hm.serving() and hc.serving()
    finally:
        hm.reset_for_tests()
        hc.reset_for_tests()


# --------------------------------------------------------------------------------------
# the master role, numpy frames
# --------------------------------------------------------------------------------------
def run_master(ours, images, enabled, posts, audio=None, delegate_only=False, frames=None):
    """Our node as the master in a thread; `posts` (raw bodies) go to our route from this thread once the job's queue
    exists.  -> ((images, audio), node, statuses)."""
    node = collector.DistributedCollectorNode()
    node.frames = frames or NumpyFrames()
    out = {}

    def go():
        try:
            out["r"] = node.run(images, audio=audio, multi_job_id=JOB, enabled_worker_ids=json.dumps(enabled),
                                delegate_only=delegate_only)
        except BaseException as e:          # noqa: BLE001 - re-raised in the test thread
            out["e"] = e
    t = threading.Thread(target=go)
    t.start()
    statuses = [post(ours.url, raw)[0] for raw in posts]
    t.join(120)
    assert not t.is_alive()
    if "e" in out:
        raise out["e"]
    return out["r"], node, statuses


def ref_master(images, enabled, posts, audio=None, delegate_only=False, timeout=60.0):
    """The reference's master given the same POST bodies, in the same order."""
    with collector_master.Master(worker_timeout=timeout, keep_bodies=False) as m:
        fut = m.collect(images, JOB, enabled, audio=audio, delegate_only=delegate_only)
        for raw in posts:
            post(m.url, raw)
        return fut.result(300)


def same_result(a, b):
    assert a[0].dtype == b[0].dtype and a[0].shape == b[0].shape, (a[0].dtype, a[0].shape, b[0].dtype, b[0].shape)
    assert torch.equal(a[0].cpu(), b[0].cpu())
    assert torch.equal(a[1]["waveform"], b[1]["waveform"]) and a[1]["sample_rate"] == b[1]["sample_rate"]


def _frame(seed, h=6, w=5):
    return image("RGB", h, w, seed)


@needs_ref
def test_order_duplicates_and_audio_as_the_reference(monkeypatch):
    monkeypatch.setenv("COMFYUI_HEARTBEAT_TIMEOUT", "60")
    master = torch.rand(2, 6, 5, 3, generator=torch.Generator().manual_seed(1))
    waves = [torch.rand(1, 2, 10 + i, generator=torch.Generator().manual_seed(10 + i)) for i in range(4)]
    png = lambda s: png_of(_frame(s), s % 2)                       # level 0 and level 1 PNGs
    posts = [body("w1", 1, png(1), False), body("w1", 0, png(2), False),
             body("zz", 0, png(3), True, audio_env(waves[0], 22050)),      # unexpected: no completion
             body("aa", 3, png(4), False),
             body("w2", 0, png(5), False, audio_env(waves[1])),
             body("w2", 0, png(6), False, audio_env(waves[2], 16000)),     # replaces image 0 and the audio
             body("w2", 2, png(7), True),
             body("w2", 1, png(8), True),                                   # a duplicate is_last
             body("w1", 2, png(9), True, audio_env(waves[3]))]
    enabled = ["w2", "w1", "w2"]                                            # de-duplicated, order kept
    with Ours() as ours:
        got, node, statuses = run_master(ours, master, enabled, posts, audio={"waveform": waves[0], "sample_rate": 8000})
    assert statuses == [200] * len(posts)
    assert node.last_stats["order"] == ["w2", "w1", "aa", "zz"]
    assert node.last_stats["frames"] == {"w2": 3, "w1": 3, "aa": 1, "zz": 1}
    want = ref_master(master, enabled, posts, audio={"waveform": waves[0], "sample_rate": 8000})
    same_result(got, want)
    assert got[0].shape[0] == 2 + 8


@needs_ref
@pytest.mark.parametrize("variant", ["delegate", "fp16", "fp64", "empty_master"])
def test_master_variants_as_the_reference(monkeypatch, variant):
    monkeypatch.setenv("COMFYUI_HEARTBEAT_TIMEOUT", "60")
    master = torch.rand(2, 6, 5, 3, generator=torch.Generator().manual_seed(3))
    if variant == "fp16":
        master = master.half()
    elif variant == "fp64":
        master = master.double()
    elif variant == "empty_master":
        master = master[:0]
    posts = [body("w1", 0, png_of(_frame(20), 0), False), body("w1", 1, png_of(_frame(21), 1), True)]
    kw = dict(delegate_only=variant == "delegate")
    with Ours() as ours:
        got, _, _ = run_master(ours, master, ["w1"], posts, **kw)
    same_result(got, ref_master(master, ["w1"], posts, **kw))


@needs_ref
def test_mismatched_sizes_fall_back_to_the_master_images(monkeypatch):
    monkeypatch.setenv("COMFYUI_HEARTBEAT_TIMEOUT", "60")
    master = torch.rand(1, 6, 5, 3, generator=torch.Generator().manual_seed(4))
    audio = {"waveform": torch.rand(1, 1, 7), "sample_rate": 1000}
    posts = [body("w1", 0, png_of(_frame(30, 7, 5), 0), True)]
    with Ours() as ours:
        got, node, _ = run_master(ours, master, ["w1"], posts, audio=audio)
    assert got[0] is master and got[1] is audio and "fallback" in node.last_stats
    same_result(got, ref_master(master, ["w1"], posts, audio=audio))


@needs_ref
def test_timeout_drains_and_stops(monkeypatch):
    """A worker that never sends is_last: after COMFYUI_HEARTBEAT_TIMEOUT without a POST the master takes what is
    queued and returns; the audio of that last drain is not kept, as in the reference."""
    monkeypatch.setenv("COMFYUI_HEARTBEAT_TIMEOUT", "1")
    monkeypatch.setenv("COMFYUI_HEARTBEAT_INTERVAL", "2")
    master = torch.rand(1, 6, 5, 3, generator=torch.Generator().manual_seed(5))
    posts = [body("w1", 0, png_of(_frame(40), 0), False), body("w2", 0, png_of(_frame(41), 0), True)]
    with Ours() as ours:
        got, node, _ = run_master(ours, master, ["w1", "w2"], posts)
        assert JOB not in hc.STORE.jobs
    assert got[0].shape[0] == 3
    same_result(got, ref_master(master, ["w1", "w2"], posts, timeout=1))


def test_interrupt_raises_and_removes_the_job(monkeypatch):
    class Interrupted(Exception):
        pass
    flag = threading.Event()

    def throw():
        if flag.is_set():
            raise Interrupted()
    mm = types.SimpleNamespace(throw_exception_if_processing_interrupted=throw, InterruptProcessingException=Interrupted)
    monkeypatch.setitem(sys.modules, "comfy", types.SimpleNamespace(model_management=mm))
    monkeypatch.setitem(sys.modules, "comfy.model_management", mm)
    monkeypatch.setenv("COMFYUI_HEARTBEAT_TIMEOUT", "60")
    with Ours() as ours:
        node = collector.DistributedCollectorNode()
        node.frames = NumpyFrames()
        err = {}

        def go():
            try:
                node.run(torch.zeros(1, 6, 5, 3), multi_job_id=JOB, enabled_worker_ids='["w1"]')
            except Interrupted as e:
                err["e"] = e
        t = threading.Thread(target=go)
        t.start()
        assert post(ours.url, body("w1", 0, png_of(_frame(50), 0), False))[0] == 200
        flag.set()
        t.join(30)
        assert "e" in err and JOB not in hc.STORE.jobs


def test_store_take_batches_what_is_queued():
    import asyncio
    store = hc.CollectorStore()

    async def go():
        assert await store.take(JOB, 0.01) == []
        await store.prepare(JOB)
        assert await store.take(JOB, 0.01) == []
        for i in range(3):
            assert await store.put(JOB, {"i": i})
        assert [d["i"] for d in await store.take(JOB, 0.01)] == [0, 1, 2]
        await store.remove(JOB)
        assert not await store.put(JOB, {"i": 9})

    asyncio.run(go())


def test_other_cases_keep_their_behaviour(monkeypatch):
    """Without the routes, or with no enabled worker, the master returns its own images (collector.py:255-259)."""
    hc.reset_for_tests()
    x = torch.rand(1, 4, 4, 3)
    out = collector.DistributedCollectorNode().run(x, multi_job_id=JOB, enabled_worker_ids='["w1"]')
    assert out[0] is x
    with Ours():
        out = collector.DistributedCollectorNode().run(x, multi_job_id=JOB, enabled_worker_ids="[]")
        assert out[0] is x


# --------------------------------------------------------------------------------------
# the numpy model on rows wider than the old 14,336-byte limit
# --------------------------------------------------------------------------------------
def png_with_filters(rows: np.ndarray, filters, C: int) -> bytes:
    """A PNG whose filtered stream has `filters[r]` and random bytes in row r (any bytes are a valid filtered row)."""
    H, n = rows.shape
    W = n // C
    R = np.concatenate([np.asarray(filters, np.uint8)[:, None], rows], 1).tobytes()
    color = {1: 0, 2: 4, 3: 2, 4: 6}[C]
    chunk = lambda t, d: len(d).to_bytes(4, "big") + t + d + zlib.crc32(t + d).to_bytes(4, "big")
    ihdr = W.to_bytes(4, "big") + H.to_bytes(4, "big") + bytes([8, color, 0, 0, 0])
    return hm.PNG_SIGNATURE + chunk(b"IHDR", ihdr) + chunk(b"IDAT", zlib.compress(R, 1)) + chunk(b"IEND", b"")


@pytest.mark.parametrize("C,W", [(3, 4800), (4, 16384), (1, 14337), (2, 9000)])
def test_model_unfilter_wide_rows_every_filter(C, W):
    rng = np.random.default_rng(W)
    filters = [0, 1, 2, 3, 4, 4, 3, 2, 1]
    data = png_with_filters(rng.integers(0, 256, (len(filters), W * C), dtype=np.uint8), filters, C)
    info = hm.parse_png(data)
    assert W * C > 14336 or C == 2
    assert np.array_equal(hm.unfilter_model(info, data), np.asarray(Image.open(io.BytesIO(data)).convert("RGB")))


def test_row_limit():
    assert hm.PNG_MAX_ROW_BYTES == nat.PNG_MAX_ROW_BYTES == 65536
    ok = png_with_filters(np.zeros((1, 65536), np.uint8), [0], 4)
    hm.parse_png(ok)
    wide = png_with_filters(np.zeros((1, 65540), np.uint8), [0], 4)
    assert np.asarray(Image.open(io.BytesIO(wide)).convert("RGB")).shape == (1, 16385, 3)     # PIL accepts it
    with pytest.raises(ValueError, match="rows of 65540 bytes"):
        hm.parse_png(wide)
    with pytest.raises(ValueError, match="^Failed to decode PNG image payload: unsupported PNG: rows"):
        hc.png_of_payload(data_url(wide))
