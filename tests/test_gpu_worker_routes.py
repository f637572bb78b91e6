"""The worker routes on the GPU: POST /distributed/clear_memory releases this package's device caches after a 4K USDU
job and a collector job (and says how many bytes that gives back), defers the release while a job runs, and the
reference's worker_ws dispatch message (its shape as tests/golden/worker_routes.json records it) runs the USDU and
collector prompts of test_gpu_orchestrator.py on workers served by these routes.  Results are checked against
oracle/usdu_oracle.py alone."""
import json
import os
import threading
import uuid

import numpy as np
import pytest
import torch

import ref_orchestration as ro
import ref_worker_routes as rw
import test_gpu_orchestrator as tgo
import usdu_oracle as orc
from __graft_entry__ import load_package
from inputs import make_input
from test_orchestrator import Loop

load_package()
from comfyui_distributed_b200 import dist, engine, worker_routes as wr  # noqa: E402
from comfyui_distributed_b200 import orchestrator  # noqa: E402
from comfyui_distributed_b200.denoise import T0Denoiser  # noqa: E402
from comfyui_distributed_b200.http_worker import _call  # noqa: E402
from comfyui_distributed_b200.nodes import DistributedCollectorNode, UltimateSDUpscaleDistributed  # noqa: E402
from comfyui_distributed_b200.nodes import collector  # noqa: E402
from comfyui_distributed_b200.testing import T0Model  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "worker_routes.json")))


def _caches():
    """Entries left in every cache release_device_caches drops."""
    return {"DevicePlan": len(engine.DevicePlan._cache), "GraphedWaves": len(engine.GraphedWaves._cache),
            "HostPipeline": len(engine.HostPipeline._cache), "PINNED_RESULTS": len(engine.PINNED_RESULTS.bufs),
            "PINNED_STAGING": len(engine.PINNED_STAGING.bufs), "text_pool": int(collector._text_pool is not None),
            "StaticJob": len(dist.StaticJob._cache), "ExactJob": len(dist.ExactJob._cache),
            "PeerPayload": len(dist.PeerPayload._cache), "payloads": len(dist._PAYLOADS)}


EMPTY = dict.fromkeys(_caches(), 0)


class Routes:
    """These routes, a job_complete stand-in that accepts every image, on 127.0.0.1; ComfyUI's
    comfy.model_management, folder_paths and app.logger as stand-ins."""

    def __init__(self, tmp_path):
        from aiohttp import web
        self.lp, self.posts = Loop(), []
        routes = web.RouteTableDef()
        wr.register(routes, rw.reset_server(ro.PromptServer()), ro.validator(False), module_state=False)

        @routes.post("/distributed/job_complete")
        async def job_complete(request):
            self.posts.append((await request.json())["batch_idx"])
            return web.json_response({"status": "success"})
        self.url = f"http://127.0.0.1:{self.lp.serve(routes)}"
        self.calls = []
        self._mods = rw.modules_patched({}, rw.make_files(str(tmp_path)), self.calls)
        self._mods.__enter__()

    def clear_memory(self):
        status, body = _call(self.url + "/distributed/clear_memory", "POST", b"{}", "application/json", timeout=120)
        return status, json.loads(body)

    def close(self):
        try:
            self.lp.close()
        finally:
            self._mods.__exit__(None, None, None)


@pytest.fixture
def routes(tmp_path):
    r = Routes(tmp_path)
    engine.release_device_caches()
    yield r
    r.close()


def _usdu(img, model, seed, tile, pad, blur):
    (out,) = UltimateSDUpscaleDistributed().run(torch.from_numpy(img), model, None, None, None, seed, 20, 8.0, "euler",
                                                "normal", 0.5, tile, tile, pad, blur, True, False)
    assert not out.is_cuda
    return out.numpy().copy()


@pytest.mark.timeout(900)
def test_idle_release_frees_the_caches(routes):
    seed, tile, pad, blur = 11, 512, 32, 8
    img = make_input("noise", 5, 1, 2160, 3840)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    first = _usdu(img, T0Model(), seed, tile, pad, blur)           # host tensor, graphed host pipeline
    frames = torch.rand(3, 720, 1280, 3, generator=torch.Generator().manual_seed(4))
    DistributedCollectorNode().run(frames, multi_job_id="j", is_worker=True, master_url=routes.url, worker_id="w1",
                                   enabled_worker_ids='["w1"]')
    assert routes.posts == [0, 1, 2]
    torch.cuda.synchronize()
    held, reserved = torch.cuda.memory_allocated(), torch.cuda.memory_reserved()
    filled = _caches()
    assert filled["HostPipeline"] and filled["DevicePlan"] and filled["PINNED_RESULTS"] and filled["text_pool"]

    assert routes.clear_memory() == (200, {"status": "success", "message": "GPU memory cleared."})
    assert routes.calls == ["unload_all_models", "soft_empty_cache"]
    assert _caches() == EMPTY
    assert torch.cuda.memory_allocated() == base
    assert torch.cuda.memory_reserved() < reserved
    print(f"\nclear_memory after a 4K USDU job and a 3-frame 720p collector job on {torch.cuda.get_device_name()}: "
          f"{held - base} bytes allocated and {reserved - torch.cuda.memory_reserved()} bytes reserved released")

    again = _usdu(img, T0Model(), seed, tile, pad, blur)
    assert np.array_equal(again, first)
    assert np.array_equal(first, orc.process_single(img, orc.make_t0_denoiser(seed, 0.5), tile, tile, pad, blur, True))


class BlockingT0Model:
    """T0's sampler, held inside its first tile until `go` is set."""

    def __init__(self):
        self.entered, self.go = threading.Event(), threading.Event()

    def as_usdu_denoiser(self, seed, denoise, **_):
        inner, model = T0Denoiser(seed, denoise), self

        def denoise_tiles(tiles, rows):
            if not model.entered.is_set():
                model.entered.set()
                assert model.go.wait(300), "the test never let the sampler go on"
            return inner(tiles, rows)
        return denoise_tiles


@pytest.mark.timeout(600)
def test_release_during_a_job_waits_for_it(routes):
    seed, tile, pad, blur = 12, 256, 32, 8
    img = make_input("noise", 6, 1, 720, 1280)
    model, result = BlockingT0Model(), {}

    def job():
        try:
            result["out"] = _usdu(img, model, seed, tile, pad, blur)
        except BaseException as e:      # noqa: BLE001 -- handed to the test
            result["error"] = e
    t = threading.Thread(target=job, daemon=True)
    t.start()
    try:
        assert model.entered.wait(300)
        busy = _caches()
        assert routes.clear_memory() == (200, {"status": "success", "message": "GPU memory cleared."})
        assert _caches() == busy and busy["HostPipeline"] == 1 and engine._release_pending
    finally:
        model.go.set()
        t.join(300)
    assert not t.is_alive() and "error" not in result, result.get("error")
    assert _caches() == EMPTY and not engine._release_pending
    assert np.array_equal(result["out"], orc.process_single(img, orc.make_t0_denoiser(seed, 0.5), tile, tile, pad,
                                                            blur, True))


# --------------------------------------------------------------------------------------
# the orchestrator's fleet, its workers served by these routes and dispatched over worker_ws
# --------------------------------------------------------------------------------------
def _dispatch_message(**fields) -> dict:
    """The reference's dispatch_prompt message: the golden file's "dispatch" case with these fields."""
    case = next(c for c in GOLDEN["cases"]["worker_ws"] if c["name"] == "dispatch")
    msg = json.loads(case["messages"][0]["text"])
    assert set(fields) <= set(msg)
    return {**msg, **fields}


@pytest.fixture
def ws_fleet(tmp_path):
    """tgo.Fleet whose two workers serve GET /prompt and these routes, and whose orchestrator sends each worker prompt
    as one dispatch_prompt message on the worker's /distributed/worker_ws."""
    from aiohttp import web
    f = tgo.Fleet(tmp_path)
    ports = {}
    for wid in ("w1", "w2"):
        part = tgo.Participant()
        server = rw.reset_server(ro.PromptServer())
        server.prompt_queue.put = lambda item, part=part: part.put(item[2])
        routes = web.RouteTableDef()

        @routes.get("/prompt")
        async def probe(request):
            return web.json_response({"exec_info": {"queue_remaining": 0}})
        assert len(wr.register(routes, server, ro.validator(False), module_state=False)) == 5
        ports[wid] = f.lp.serve(routes)
        f.workers[wid] = part
    (tmp_path / "ws_config.json").write_text(json.dumps({
        "workers": [{"id": w, "host": "127.0.0.1", "port": p, "type": "local", "enabled": True}
                    for w, p in ports.items()], "settings": {"websocket_orchestration": False}}))
    f.orch.config = orchestrator.Config(str(tmp_path / "ws_config.json"))

    async def dispatch(session, worker, prompt, workflow_meta):
        msg = _dispatch_message(request_id=uuid.uuid4().hex, prompt=prompt, workflow=workflow_meta, client_id="c")
        async with session.ws_connect(f.orch.url(worker, "/distributed/worker_ws")) as ws:
            await ws.send_json(msg)
            ack = await ws.receive_json(timeout=60)
        assert ack["type"] == "dispatch_ack" and ack["request_id"] == msg["request_id"] and ack["ok"], ack
    f.orch.dispatch = dispatch
    yield f
    f.close()


@pytest.mark.timeout(900)
def test_usdu_prompt_over_worker_ws_equals_replay(ws_fleet):
    tgo.test_usdu_prompt_equals_replay(ws_fleet)


@pytest.mark.timeout(600)
def test_collector_prompt_over_worker_ws_gathers_seeds_in_order(ws_fleet):
    tgo.test_collector_prompt_gathers_seeds_in_order(ws_fleet)
