"""The orchestrator (orchestrator.py) against the reference's own: every case of tests/golden/orchestration.json
(oracle/ref_orchestration.py ran the reference's /distributed/queue handler on it) gives the same reply, worker POST
bodies, master queue item and collector queues; malformed bodies get the same status and error.  Then the network side
with stand-in workers on 127.0.0.1: probes, least-busy choice, dispatch bodies, media uploads, the websocket setting and
route registration."""
import asyncio
import json
import os
import socket
import sys
import threading
import types
import warnings

import pytest

import ref_orchestration as ro
from __graft_entry__ import load_package

load_package()
from comfyui_distributed_b200 import http_collector as hc  # noqa: E402
from comfyui_distributed_b200 import orchestrator as orc  # noqa: E402
from comfyui_distributed_b200.http_worker import _call  # noqa: E402

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "orchestration.json")))
CASES = {c["name"]: c for c in GOLDEN["cases"]}
QUEUE = ("POST", "/distributed/queue")


def _orch(tmp_path, config, server=None, invalid=False):
    path = tmp_path / "gpu_config.json"
    path.write_text(json.dumps(config))
    o = orc.Orchestrator(server or ro.PromptServer(), validate=ro.validator(invalid), store=hc.CollectorStore(),
                         config=orc.Config(str(path)))
    o.job_prefix = lambda: GOLDEN["prefix"]
    return o


@pytest.mark.parametrize("name", list(CASES))
def test_case_equals_reference(tmp_path, name):
    case = CASES[name]
    o = _orch(tmp_path, case["config"], invalid=case["invalid"])
    session = ro.FakeSession(case["queues"], case["seps"])
    o.session = lambda: session
    handler = orc.make_handlers(o)[QUEUE]
    resp = asyncio.run(handler(ro.FakeRequest(json.dumps(case["body"]))))
    got = ro.observed(resp, session, o.server, sorted(o.store.jobs))
    want = case["expect"]
    assert got["status"] == want["status"] and got["reply"] == want["reply"]
    assert [u for u, _ in got["posts"]] == [u for u, _ in want["posts"]]
    for (url, body), (_, ref) in zip(got["posts"], want["posts"]):
        assert body == ref, url                 # the pruned worker prompt with its hidden inputs, and extra_data
    assert got["queued"] == want["queued"]      # the master's prompt, extra_data (client_id, workflow) and outputs
    assert got["queues"] == want["queues"]      # the job-id map: one collector queue per distributed node


def test_golden_covers_the_rules():
    """The cases reach what the issue lists: collectors after USDU, delegate-only with and without collectors and with
    USDU, 0/1/3 workers, load_balance on a worker and on the master."""
    def master_prompt(n):
        return CASES[n]["expect"]["queued"][0]["prompt"]
    assert any(v["inputs"].get("pass_through") for v in master_prompt("collector_after_usdu").values())
    assert any(v["class_type"] == "DistributedEmptyImage" for v in master_prompt("delegate_collectors").values())
    assert master_prompt("delegate_usdu").keys() == CASES["delegate_usdu"]["prompt"].keys()
    assert master_prompt("delegate_no_collector") == CASES["delegate_no_collector"]["prompt"]
    assert [CASES[f"seed_value_{n}_workers"]["expect"]["reply"]["worker_count"] for n in (0, 1, 3)] == [0, 1, 3]
    assert CASES["load_balance_busy"]["expect"]["posts"][0][0].endswith(":9002/prompt")
    assert CASES["load_balance_master_idle"]["expect"]["posts"] == []


@pytest.mark.parametrize("i", range(len(GOLDEN["bad_bodies"])))
def test_request_validation_equals_reference(tmp_path, i):
    b = GOLDEN["bad_bodies"][i]
    if b["ok"]:
        got = orc.parse_queue_request(json.loads(b["raw"]))
        assert {k: getattr(got, k) for k in b["parsed"]} == b["parsed"]
        return
    o = _orch(tmp_path, {})
    o.session = lambda: pytest.fail("a refused body reached the orchestration")
    resp = asyncio.run(orc.make_handlers(o)[QUEUE](ro.FakeRequest(b["raw"])))
    assert {"status": resp.status, "reply": ro.reply_json(resp)} == b["expect"]


def test_config_defaults_cache_and_reload(tmp_path):
    path = tmp_path / "gpu_config.json"
    cfg = orc.Config(str(path))
    assert cfg.load() == orc.default_config()
    path.write_text(json.dumps({"workers": [{"id": "a"}], "settings": {"master_delegate_only": True}, "extra": 1}))
    os.utime(path, (1000, 1000))
    cfg = orc.Config(str(path))
    got = cfg.load()
    assert got["workers"] == [{"id": "a"}] and got["extra"] == 1 and got["master"] == {"host": ""}
    assert got["settings"]["master_delegate_only"] and got["settings"]["worker_probe_concurrency"] == 8
    path.write_text(json.dumps({"workers": []}))
    os.utime(path, (1000, 1000))
    assert cfg.load() is got                    # same mtime: the cached config
    os.utime(path, (2000, 2000))
    assert cfg.load()["workers"] == []
    path.write_text("{not json")
    os.utime(path, (3000, 3000))
    with pytest.warns(RuntimeWarning, match="using the defaults"):
        assert cfg.load() == orc.default_config()


def test_resolve_workers():
    cfg = {"workers": [{"id": " a ", "listen_port": "9000", "enabled": True}, {"id": "b", "port": "x"},
                       {"id": ""}, {"id": "c", "port": 0, "enabled": False, "type": "cloud", "host": "h"}]}
    assert orc.resolve_workers(cfg) == [{"id": "a", "name": "a", "host": None, "port": 9000, "type": "local"}]
    assert [(w["id"], w["port"]) for w in orc.resolve_workers(cfg, ["b", "c"])] == [("b", 8188), ("c", 8188)]


# --------------------------------------------------------------------------------------
# stand-in workers and master on 127.0.0.1
# --------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


class Loop:
    """An event loop on its own thread, for the servers of one test."""

    def __init__(self):
        self.loop = asyncio.new_event_loop()
        self.thread = threading.Thread(target=self.loop.run_forever, daemon=True)
        self.thread.start()
        self.runners = []

    def call(self, coro, timeout=60):
        return asyncio.run_coroutine_threadsafe(coro, self.loop).result(timeout)

    def serve(self, routes, port=None):
        from aiohttp import web
        app = web.Application(client_max_size=1 << 28)
        app.add_routes(routes)
        runner = web.AppRunner(app)
        self.call(runner.setup())
        port = port or _free_port()
        self.call(web.TCPSite(runner, "127.0.0.1", port).start())
        self.runners.append(runner)
        return port

    def close(self):
        try:
            for r in self.runners:
                self.call(r.cleanup())
        finally:
            self.loop.call_soon_threadsafe(self.loop.stop)
            self.thread.join(10)


class Worker:
    """A ComfyUI worker's routes the orchestrator calls: GET /prompt (after `delay` s) answers `queue_remaining`;
    POST /prompt, /distributed/check_file and /upload/image are recorded."""

    def __init__(self, lp: Loop, queue_remaining=0, delay=0.0, sep=None, have=()):
        from aiohttp import web
        self.prompts, self.checks, self.uploads = [], [], []
        routes = web.RouteTableDef()

        @routes.get("/prompt")
        async def probe(request):
            await asyncio.sleep(delay)
            return web.json_response({"exec_info": {"queue_remaining": queue_remaining}})

        @routes.post("/prompt")
        async def prompt(request):
            self.prompts.append(await request.json())
            return web.json_response({"prompt_id": "p", "number": 0, "node_errors": {}})

        @routes.get("/distributed/system_info")
        async def system_info(request):
            if sep is None:
                return web.json_response({}, status=404)
            return web.json_response({"platform": {"path_separator": sep}})

        @routes.post("/distributed/check_file")
        async def check_file(request):
            body = await request.json()
            self.checks.append(body)
            return web.json_response({"status": "success", "exists": body["filename"] in have, "hash_matches": True})

        @routes.post("/upload/image")
        async def upload(request):
            form = await request.post()
            f = form["image"]
            self.uploads.append({"name": f.filename, "bytes": f.file.read(), "type": form["type"],
                                 "subfolder": form["subfolder"], "overwrite": form["overwrite"],
                                 "content_type": f.content_type})
            return web.json_response({"name": "up_" + f.filename, "subfolder": "sync", "type": "input"})

        self.port = lp.serve(routes)


@pytest.fixture
def lp():
    loop = Loop()
    yield loop
    loop.close()


def _post_queue(url, body):
    status, text = _call(url + "/distributed/queue", "POST", json.dumps(body).encode(), "application/json", timeout=60)
    return status, json.loads(text)


def _master(lp, tmp_path, config, port=None, extra=None):
    """The orchestrator's routes served on 127.0.0.1 -> (url, orchestrator).  Its PromptServer reports `port`, the
    port it is served on, or ro.MASTER_PORT (the reference's runs) when None."""
    from aiohttp import web
    o = _orch(tmp_path, config, server=ro.PromptServer(port or ro.MASTER_PORT))
    routes = web.RouteTableDef()
    assert orc.register(routes, o, module_state=False) == {QUEUE, ("GET", "/distributed/queue_status/{job_id}")}
    if extra:
        extra(routes)
    return f"http://127.0.0.1:{lp.serve(routes, port)}", o


def _live_config(case, ports, **settings):
    cfg = json.loads(json.dumps(case["config"]))
    for w in cfg["workers"]:
        w["port"] = ports.get(w["id"], w.get("port"))
    cfg["settings"] = {**cfg.get("settings", {}), **settings}
    return cfg


def test_dispatch_bodies_equal_reference(lp, tmp_path):
    case = CASES["workflow:distributed-txt2img.json"]      # a workflow and a client_id: extra_data on the wire
    w1, w2 = Worker(lp), Worker(lp)
    url, o = _master(lp, tmp_path, _live_config(case, {"w1": w1.port, "w2": w2.port}))
    status, reply = _post_queue(url, case["body"])
    reply.pop("prompt_id")
    assert (status, reply) == (200, case["expect"]["reply"])
    assert [w1.prompts, w2.prompts] == [[b] for _, b in case["expect"]["posts"]]
    assert ro.queued_items(o.server) == case["expect"]["queued"]


def test_offline_and_slow_workers_are_dropped(lp, tmp_path, monkeypatch):
    """A worker whose probe is slower than PROBE_TIMEOUT counts as offline, like one that does not listen."""
    monkeypatch.setattr(orc, "PROBE_TIMEOUT", 0.5)
    case = CASES["seed_value_one_offline"]                  # w2 offline in the reference's run
    w1, w2, w3 = Worker(lp), Worker(lp, delay=3.0), Worker(lp)
    url, _ = _master(lp, tmp_path, _live_config(case, {"w1": w1.port, "w2": w2.port, "w3": w3.port}))
    assert _post_queue(url, case["body"])[1]["worker_count"] == 2
    assert w2.prompts == [] and [w1.prompts, w3.prompts] == [[b] for _, b in case["expect"]["posts"]]

    case = CASES["delegate_all_offline"]                    # nobody answers: the master runs the whole prompt
    slow = Worker(lp, delay=3.0)
    url, o = _master(lp, tmp_path, _live_config(case, {"w1": _free_port(), "w2": slow.port}))
    assert _post_queue(url, case["body"])[1]["worker_count"] == 0
    assert o.server.queued[0][2] == case["expect"]["queued"][0]["prompt"]


def test_least_busy_choice(lp, tmp_path):
    """load_balance: the shortest queue among the workers and the master; idle candidates take turns."""
    from aiohttp import web
    case = CASES["load_balance_busy"]
    qs = {int(k): v for k, v in case["queues"].items()}
    ws = {f"w{i}": Worker(lp, qs[9000 + i]) for i in (1, 2, 3)}

    def master_probe(routes):
        @routes.get("/prompt")
        async def probe(request):
            return web.json_response({"exec_info": {"queue_remaining": qs[ro.MASTER_PORT]}})
    port = _free_port()
    url, o = _master(lp, tmp_path, _live_config(case, {k: w.port for k, w in ws.items()}), port, master_probe)
    assert _post_queue(url, case["body"])[1]["worker_count"] == 1
    want = json.loads(json.dumps(case["expect"]["posts"][0][1]).replace(f":{ro.MASTER_PORT}", f":{port}"))
    assert [len(w.prompts) for w in ws.values()] == [0, 1, 0] and ws["w2"].prompts[0] == want
    # every candidate idle (the master too): the choice moves one candidate per request
    idle = [Worker(lp, 0), Worker(lp, 0)]
    (tmp_path / "idle.json").write_text(json.dumps({"workers": [{"id": f"i{k}", "host": "127.0.0.1", "port": w.port}
                                                                 for k, w in enumerate(idle)],
                                                    "settings": {"websocket_orchestration": False}}))
    o.config = orc.Config(str(tmp_path / "idle.json"))
    qs[ro.MASTER_PORT] = 0
    body = {**case["body"], "enabled_worker_ids": ["i0", "i1"]}
    counts = [_post_queue(url, body)[1]["worker_count"] for _ in range(3)]
    assert counts == [1, 1, 0] and [len(w.prompts) for w in idle] == [1, 1]     # i0, i1, then the master


def test_remote_worker_gets_media_and_paths(lp, tmp_path, monkeypatch):
    pic, clip = tmp_path / "pic.png", tmp_path / "clip.mp4"
    pic.write_bytes(b"\x89PNG fake")
    clip.write_bytes(b"fake video")
    files = {"sub/pic.png": str(pic), "clip.mp4": str(clip)}
    monkeypatch.setitem(sys.modules, "folder_paths", types.SimpleNamespace(
        get_annotated_filepath=lambda name: files.get(name, str(tmp_path / "missing"))))
    prompt = {"1": {"class_type": "LoadImage", "inputs": {"image": "sub\\pic.png [input]"}},
              "2": {"class_type": "LoadVideo", "inputs": {"file": "clip.mp4", "path": "models/a/b.safetensors"}},
              "3": {"class_type": "LoadImage", "inputs": {"image": "gone.png"}},
              "4": {"class_type": "Combine", "inputs": {"a": ["1", 0], "b": ["2", 0], "c": ["3", 0]}},
              "5": {"class_type": "DistributedCollector", "inputs": {"images": ["4", 0]}}}
    remote = Worker(lp, sep="\\", have=("clip.mp4",))
    local = Worker(lp)
    cfg = {"workers": [{"id": "r", "host": "127.0.0.1", "port": remote.port, "type": "remote"},
                       {"id": "l", "host": "127.0.0.1", "port": local.port, "type": "local"}],
           "settings": {"websocket_orchestration": False}}
    url, _ = _master(lp, tmp_path, cfg)
    assert _post_queue(url, {"prompt": prompt, "client_id": "c", "enabled_worker_ids": ["r", "l"]})[0] == 200
    assert [c["filename"] for c in remote.checks] == ["clip.mp4", "sub/pic.png"]
    assert remote.uploads == [{"name": "pic.png", "bytes": b"\x89PNG fake", "type": "input", "subfolder": "sub",
                               "overwrite": "true", "content_type": "image/png"}]
    got = remote.prompts[0]["prompt"]
    assert got["1"]["inputs"]["image"] == "sync/up_pic.png"          # the worker's name for the upload
    assert got["2"]["inputs"] == {"file": "clip.mp4", "path": "models\\a\\b.safetensors"}
    assert got["3"]["inputs"]["image"] == "gone.png"
    assert local.checks == [] and local.uploads == []
    assert local.prompts[0]["prompt"]["2"]["inputs"]["path"] == "models/a/b.safetensors"


def test_websocket_setting_warns_once_and_uses_http(lp, tmp_path):
    orc.reset_for_tests()
    case = CASES["workflow:distributed-txt2img.json"]
    w1, w2 = Worker(lp), Worker(lp)
    url, _ = _master(lp, tmp_path, _live_config(case, {"w1": w1.port, "w2": w2.port}, websocket_orchestration=True))
    with warnings.catch_warnings(record=True) as seen:
        warnings.simplefilter("always")
        for _ in range(2):
            assert _post_queue(url, case["body"])[0] == 200
    assert sum("websocket_orchestration" in str(w.message) for w in seen) == 1
    assert len(w1.prompts) == len(w2.prompts) == 2
    orc.reset_for_tests()


def test_queue_route_taken_by_another_package_is_skipped(tmp_path):
    from aiohttp import web
    orc.reset_for_tests()
    routes = web.RouteTableDef()

    @routes.post("/distributed/queue")
    async def theirs(request):
        return web.json_response({})
    o = _orch(tmp_path, {})
    with pytest.warns(RuntimeWarning, match="/distributed/queue is already served"):
        served = orc.register(routes, o)
    assert served == {("GET", "/distributed/queue_status/{job_id}")} and not orc.serving()
    orc.reset_for_tests()
    assert orc.register(web.RouteTableDef(), o) and orc.serving()
    orc.reset_for_tests()


def test_queue_status_reports_collector_queues(lp, tmp_path):
    case = CASES["seed_value_0_workers"]
    url, o = _master(lp, tmp_path, case["config"])
    assert _post_queue(url, case["body"])[0] == 200
    job = case["expect"]["queues"][0]
    for jid, exists in ((job, True), ("nope", False)):
        status, text = _call(f"{url}/distributed/queue_status/{jid}", "GET")
        assert (status, json.loads(text)) == (200, {"exists": exists, "job_id": jid})
