"""End to end on the GPU: one POST /distributed/queue to a master that serves this package's routes (orchestrator.py,
http_master.py, http_collector.py) on 127.0.0.1, with two in-process stand-ins for ComfyUI workers that run the prompt
they are posted.  Every participant runs this package's nodes (the T0 sampler double for the model) through a small
prompt executor in place of ComfyUI's; the master runs the prompt the orchestrator queues on its PromptServer stand-in.
The results are checked against oracle/usdu_oracle.py alone."""
import json
import threading

import numpy as np
import pytest
import torch

import ref_orchestration as ro
import usdu_oracle as orc
from __graft_entry__ import load_package
from inputs import make_input
from test_orchestrator import Loop, _free_port, _post_queue

load_package()
from comfyui_distributed_b200 import http_collector as hc  # noqa: E402
from comfyui_distributed_b200 import http_master as hm  # noqa: E402
from comfyui_distributed_b200 import orchestrator  # noqa: E402
from comfyui_distributed_b200.nodes import NODE_CLASS_MAPPINGS  # noqa: E402
from comfyui_distributed_b200.testing import T0Model  # noqa: E402


class NoiseImage:
    FUNCTION = "make"

    def make(self, kind, seed, B, H, W):
        return (torch.from_numpy(make_input(kind, int(seed), B, H, W)),)


class T0ModelNode:
    FUNCTION = "load"

    def load(self):
        return (T0Model(),)


class Output:
    FUNCTION = "save"

    def save(self, images):
        self.images = images
        return ()


CLASSES = {**NODE_CLASS_MAPPINGS, "NoiseImage": NoiseImage, "T0Model": T0ModelNode, "SaveImage": Output,
           "PreviewImage": Output}


class Participant:
    """Runs each prompt it is given on a thread of its own, as ComfyUI's executor would: the output nodes and what
    they need, links resolved to the upstream node's outputs.  `runs` holds (node instances by id, error) per prompt."""

    def __init__(self):
        self.runs, self.threads = [], []

    def put(self, prompt):
        run = {"nodes": {}, "error": None}
        self.runs.append(run)
        t = threading.Thread(target=self._execute, args=(prompt, run), daemon=True)
        self.threads.append(t)
        t.start()

    def _execute(self, prompt, run):
        outs = {}

        def value(nid):
            if nid not in outs:
                node = prompt[nid]
                inst = CLASSES[node["class_type"]]()
                run["nodes"][nid] = inst
                kw = {k: value(str(v[0]))[v[1]] if isinstance(v, list) and len(v) == 2 else v
                      for k, v in node["inputs"].items()}
                res = getattr(inst, inst.FUNCTION)(**kw)
                outs[nid] = res["result"] if isinstance(res, dict) else res
            return outs[nid]
        try:
            for nid in sorted(prompt, key=int):
                if prompt[nid]["class_type"] in ("SaveImage", "PreviewImage"):
                    value(nid)
        except BaseException as e:      # noqa: BLE001 -- handed to the test
            run["error"] = e

    def join(self, timeout=600):
        for t in self.threads:
            t.join(timeout)
        assert not any(t.is_alive() for t in self.threads), "a prompt did not finish"
        for run in self.runs:
            if run["error"] is not None:
                raise run["error"]


class Fleet:
    """The master (its routes, its PromptServer stand-in whose queue runs the prompt) and two workers on one loop."""

    def __init__(self, tmp_path):
        from aiohttp import web
        self.lp = Loop()
        self.master, self.workers = Participant(), {"w1": Participant(), "w2": Participant()}
        ports = {}
        for wid, part in self.workers.items():
            routes = web.RouteTableDef()

            @routes.get("/prompt")
            async def probe(request):
                return web.json_response({"exec_info": {"queue_remaining": 0}})

            @routes.post("/prompt")
            async def prompt(request, part=part):
                part.put((await request.json())["prompt"])
                return web.json_response({"prompt_id": "p", "number": 0, "node_errors": {}})
            ports[wid] = self.lp.serve(routes)
        (tmp_path / "gpu_config.json").write_text(json.dumps({
            "workers": [{"id": w, "host": "127.0.0.1", "port": p, "type": "local", "enabled": True}
                        for w, p in ports.items()], "settings": {"websocket_orchestration": False}}))
        hm.reset_for_tests()
        hc.reset_for_tests()
        port = _free_port()
        server = ro.PromptServer(port)
        server.prompt_queue.put = lambda item: self.master.put(item[2])
        self.orch = orchestrator.Orchestrator(server, validate=ro.validator(False),
                                              config=orchestrator.Config(str(tmp_path / "gpu_config.json")))
        routes = web.RouteTableDef()
        hm.register(routes, hm.STORE, self.lp.loop)
        hc.register(routes, hc.STORE, self.lp.loop)
        orchestrator.register(routes, self.orch, module_state=False)
        self.url = f"http://127.0.0.1:{self.lp.serve(routes, port)}"
        assert hm.serving() and hc.serving()

    def queue(self, prompt, **body):
        status, reply = _post_queue(self.url, {"prompt": prompt, "client_id": "c", "enabled_worker_ids": ["w1", "w2"],
                                               **body})
        assert status == 200 and reply["worker_count"] == 2, reply
        for part in [self.master, *self.workers.values()]:
            part.join()
        assert len(self.master.runs) == 1
        return self.master.runs[0]["nodes"]

    def close(self):
        try:
            self.lp.close()
        finally:
            hm.reset_for_tests()
            hc.reset_for_tests()


@pytest.fixture
def fleet(tmp_path):
    f = Fleet(tmp_path)
    yield f
    f.close()


def _n(ct, **inputs):
    return {"class_type": ct, "inputs": inputs}


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_usdu_prompt_equals_replay(fleet):
    B, H, W, tile, pad, blur, seed, denoise = 1, 300, 420, 128, 16, 8, 5, 0.5
    prompt = {"1": _n("NoiseImage", kind="noise", seed=3, B=B, H=H, W=W), "2": _n("T0Model"),
              "3": _n("UltimateSDUpscaleDistributed", upscaled_image=["1", 0], model=["2", 0], positive=None,
                      negative=None, vae=None, seed=seed, steps=20, cfg=8.0, sampler_name="euler", scheduler="normal",
                      denoise=denoise, tile_width=tile, tile_height=tile, padding=pad, mask_blur=blur,
                      force_uniform_tiles=True, tiled_decode=False),
              "4": _n("SaveImage", images=["3", 0])}
    nodes = fleet.queue(prompt)
    stats, got = nodes["3"].last_stats, nodes["4"].images
    asg = stats["assignment"]
    n_tiles = len(orc.make_plan(W, H, tile, tile, pad, True)[2])
    assert len(asg) == 3 and sorted(t for a in asg for t in a) == list(range(n_tiles))
    for wid, part in fleet.workers.items():                 # each worker ran the USDU node as an HTTP worker
        assert part.runs and part.runs[0]["nodes"]["3"].last_stats["pulled"] == asg[int(wid[1])]
    img = make_input("noise", 3, B, H, W)
    want = orc.replay_static(img, orc.make_t0_denoiser(seed, denoise), tile, tile, pad, blur, True, asg)
    assert np.array_equal(got.cpu().numpy(), want), asg


def _collector_prompt():
    return {"1": _n("DistributedSeed", seed=100), "2": _n("NoiseImage", kind="noise", seed=["1", 0], B=2, H=40, W=56),
            "3": _n("DistributedCollector", images=["2", 0]), "4": _n("SaveImage", images=["3", 0])}


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_collector_prompt_gathers_seeds_in_order(fleet):
    got = fleet.queue(_collector_prompt())["4"].images
    img = {s: make_input("noise", s, 2, 40, 56) for s in (100, 101, 102)}
    want = orc.collector_combine(img[100], {"w1": img[101], "w2": img[102]}, ["w1", "w2"])
    assert got.shape == (6, 40, 56, 3) and np.array_equal(got.cpu().numpy(), want)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_delegate_only_collector_prompt_returns_the_workers_images(fleet):
    nodes = fleet.queue(_collector_prompt(), delegate_master=True)
    assert "1" not in nodes and "2" not in nodes                # the master ran only the collector and its output
    img = {s: make_input("noise", s, 2, 40, 56) for s in (101, 102)}
    want = orc.collector_combine(None, {"w1": img[101], "w2": img[102]}, ["w1", "w2"], delegate_only=True)
    got = nodes["4"].images
    assert got.shape == (4, 40, 56, 3) and np.array_equal(got.cpu().numpy(), want)
