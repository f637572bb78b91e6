"""The reference's orchestrator (api/job_routes.py:206-236 and what it calls: api/queue_request.py,
api/queue_orchestration.py, api/orchestration/, utils/network.py, utils/async_helpers.py), run for real under stubs --
TEST INFRASTRUCTURE ONLY; generating needs the reference tree or the bundle oracle/make_ref.py packs.

`python oracle/ref_orchestration.py` posts every case of `cases()` to the reference's `/distributed/queue` handler, with
the network replaced by `FakeSession` (the workers' answers are the case's), ComfyUI's PromptServer and
execution.validate_prompt by stand-ins, and the job-id prefix fixed, and writes what the reference derived to
tests/golden/orchestration.json: the reply, the POST /prompt body each worker got, the master's queue item and the
collector queues it opened.  Only derived prompts and verdicts are written, no reference source.  The shipped workflows
(workflows/*.json, the UI's graph format) are turned into API prompts by `api_prompt` first.

`FakeSession` and `FakeRequest` are shared with tests/test_orchestrator.py, which runs this package's orchestrator on
the same cases.
"""
from __future__ import annotations

import asyncio
import copy
import dataclasses
import importlib.util
import json
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(os.path.dirname(HERE), "tests", "golden", "orchestration.json")
PKG = "reforch"
MASTER_PORT = 8188
FIXED_MS = 1700000000000                # the job-id prefix of every case: exec_<FIXED_MS>_<FIXED_HEX>
FIXED_HEX = "a1b2c3"
WORKFLOWS = ("distributed-txt2img.json", "distributed-upscale-video.json", "distributed-upscale.json",
             "distributed-wan-2.2_14b_t2v.json", "distributed-wan.json")


# --------------------------------------------------------------------------------------
# stand-ins shared with the tests
# --------------------------------------------------------------------------------------
class _Resp:
    def __init__(self, status, payload, url):
        self.status, self._payload, self.url = status, payload, url

    async def json(self):
        return self._payload

    def raise_for_status(self):
        if self.status >= 400:
            raise RuntimeError(f"HTTP {self.status} from {self.url}")

    async def __aenter__(self):
        return self

    async def __aexit__(self, *exc):
        return False


class FakeSession:
    """An aiohttp ClientSession stand-in for the workers of a case.  `queues` {port: queue_remaining, or None for a
    worker that does not answer}; `seps` {port: path separator a worker reports}.  `posts` records every POST as
    (url, json body)."""

    def __init__(self, queues, seps=None):
        self.queues = {int(k): v for k, v in queues.items()}
        self.seps = {int(k): v for k, v in (seps or {}).items()}
        self.posts = []

    @staticmethod
    def _port(url):
        rest = url.split("://", 1)[1]
        host = rest.split("/", 1)[0]
        return int(host.rsplit(":", 1)[1]) if ":" in host else 80

    def get(self, url, timeout=None):
        port = self._port(url)
        if self.queues.get(port) is None:
            raise asyncio.TimeoutError()
        if url.endswith("/distributed/system_info"):
            sep = self.seps.get(port)
            return _Resp(200 if sep else 404, {"platform": {"path_separator": sep}} if sep else None, url)
        return _Resp(200, {"exec_info": {"queue_remaining": self.queues[port]}}, url)

    def post(self, url, json=None, data=None, timeout=None):
        self.posts.append((url, copy.deepcopy(json)))
        return _Resp(200, {}, url)

    async def __aenter__(self):
        return self

    async def __aexit__(self, *exc):
        return False

    @property
    def closed(self):
        return False


class FakeRequest:
    """What a route handler reads of an aiohttp request: the body as JSON."""

    def __init__(self, raw: str, match_info=None):
        self.raw, self.match_info = raw, match_info or {}

    async def json(self):
        return json.loads(self.raw)


class PromptServer:
    """The parts of ComfyUI's PromptServer the orchestrator touches."""

    def __init__(self, port=MASTER_PORT):
        self.address, self.port, self.number, self.loop = "127.0.0.1", port, 0, None
        self.queued = []
        self.prompt_queue = types.SimpleNamespace(put=self.queued.append)

    def trigger_on_prompt(self, payload):
        return payload


def validator(invalid: bool):
    """execution.validate_prompt stand-in: accepts every prompt, or refuses it with one node error."""
    async def validate_prompt(prompt_id, prompt, partial):
        if invalid:
            return (False, {"type": "prompt_outputs_failed_validation", "message": "Prompt outputs failed validation",
                            "details": "", "extra_info": {}}, [],
                    {"9": {"class_type": "SaveImage", "errors": [{"message": "Required input is missing",
                                                                  "details": "images"}]}})
        outs = sorted(k for k, v in prompt.items() if v.get("class_type") in ("PreviewImage", "SaveImage"))
        return (True, None, outs, {})
    return validate_prompt


def reply_json(resp) -> dict:
    return json.loads(resp.body)


# --------------------------------------------------------------------------------------
# the cases
# --------------------------------------------------------------------------------------
def api_prompt(ui: dict) -> dict:
    """A UI workflow graph -> an API prompt: links become [source id, slot] (through Reroutes), widget values become
    inputs named widget_<i> (`image` for LoadImage), notes are dropped."""
    nodes = {n["id"]: n for n in ui["nodes"]}
    links = {l[0]: (l[1], l[2]) for l in ui["links"]}

    def source(link):
        src, slot = links[link]
        while nodes[src]["type"] == "Reroute":
            src, slot = links[nodes[src]["inputs"][0]["link"]]
        return [str(src), slot]

    out = {}
    for nid, n in nodes.items():
        if n["type"] in ("Reroute", "Note", "MarkdownNote"):
            continue
        inputs = {}
        wv = n.get("widgets_values")
        if isinstance(wv, dict):
            inputs.update({k: v for k, v in wv.items() if not isinstance(v, (dict, list))})
        elif isinstance(wv, list):
            for i, v in enumerate(wv):
                inputs["image" if n["type"] == "LoadImage" and i == 0 else f"widget_{i}"] = v
        for inp in n.get("inputs") or []:
            if inp.get("link") is not None:
                inputs[inp["name"]] = source(inp["link"])
        out[str(nid)] = {"inputs": inputs, "class_type": n["type"], "_meta": {"title": n.get("title", n["type"])}}
    return out


def _n(ct, **inputs):
    return {"class_type": ct, "inputs": inputs}


def synthetic() -> dict:
    """Prompts that reach each rule of the rewriting."""
    img = _n("LoadImage", image="sub\\dir/pic.png [input]")
    base = {"1": img, "2": _n("CheckpointLoaderSimple", ckpt_name="models\\sd\\x.safetensors")}
    usdu = _n("UltimateSDUpscaleDistributed", upscaled_image=["1", 0], model=["2", 0], positive=["2", 1],
              negative=["2", 1], vae=["2", 2], seed=["5", 0], steps=20, tile_width=512, tile_height=512)
    return {
        "collector_after_usdu": {**base, "5": _n("DistributedSeed", seed=7), "3": usdu,
                                 "4": _n("DistributedCollector", images=["3", 0]), "9": _n("SaveImage", images=["4", 0])},
        "collectors_two": {**base, "5": _n("DistributedSeed", seed=11), "6": _n("KSampler", seed=["5", 0], model=["2", 0]),
                           "7": _n("VAEDecode", samples=["6", 0], vae=["2", 2]),
                           "4": _n("DistributedCollector", images=["7", 0], load_balance=False),
                           "8": _n("ImageScale", image=["4", 0]), "9": _n("SaveImage", images=["8", 0]),
                           "12": _n("DistributedCollector", images=["1", 0]), "13": _n("PreviewImage", images=["12", 0])},
        "no_collector": {**base, "5": _n("DistributedSeed", seed=3), "6": _n("KSampler", seed=["5", 0]),
                         "9": _n("SaveImage", images=["6", 0])},
        "seed_value": {**base, "5": _n("DistributedSeed", seed=100), "10": _n("DistributedValue", default_value="a",
                                                                               worker_values='{"1": "b", "2": "c"}'),
                       "6": _n("KSampler", seed=["5", 0], cfg=["10", 0]), "4": _n("DistributedCollector", images=["6", 0]),
                       "9": _n("SaveImage", images=["4", 0])},
        "usdu_only": {**base, "5": _n("DistributedSeed", seed=1), "3": usdu, "9": _n("SaveImage", images=["3", 0])},
        "load_balance": {**base, "6": _n("KSampler", seed=5), "4": _n("DistributedCollector", images=["6", 0],
                                                                      load_balance="yes"),
                         "9": _n("SaveImage", images=["4", 0])},
    }


def _workers(n, **extra):
    return [{"id": f"w{i + 1}", "name": f"Worker {i + 1}", "host": "127.0.0.1", "port": 9001 + i, "type": "local",
             "enabled": True, **extra} for i in range(n)]


def cases(workflows: dict) -> list:
    """-> [{name, prompt, config, body, queues, seps, invalid}]: the request each case posts and what its workers
    answer (queues: {port: queue_remaining or None when offline}; the master is MASTER_PORT)."""
    s = synthetic()
    settings = {"websocket_orchestration": False}
    two = {"workers": _workers(2), "settings": settings}
    three = {"workers": _workers(3), "settings": settings}
    up = {9001: 0, 9002: 0, 9003: 0, MASTER_PORT: 0}
    out = []

    def case(name, prompt, config, ids=("w1", "w2"), delegate=None, queues=None, seps=None, invalid=False,
             workflow=None, body=None):
        b = body if body is not None else {"prompt": prompt, "client_id": "client-1", "enabled_worker_ids": list(ids)}
        if delegate is not None:
            b["delegate_master"] = delegate
        if workflow is not None:
            b["workflow"] = workflow
        out.append({"name": name, "prompt": prompt, "config": config, "body": b,
                    "queues": {str(k): v for k, v in (queues or up).items()}, "seps": seps or {}, "invalid": invalid})

    for wf, prompt in workflows.items():
        case(f"workflow:{wf}", prompt, two, workflow={"note": wf})
        case(f"workflow:{wf}:delegate", prompt, two, delegate=True)
    case("collector_after_usdu", s["collector_after_usdu"], two)
    case("delegate_collectors", s["collectors_two"], two, delegate=True)
    case("delegate_no_collector", s["no_collector"], two, delegate=True)
    case("delegate_usdu", s["collector_after_usdu"], two, delegate=True)
    case("delegate_usdu_only", s["usdu_only"], two, delegate=True)
    case("delegate_from_config", s["collectors_two"], {"workers": _workers(2), "settings": {
        "websocket_orchestration": False, "master_delegate_only": True}})
    case("delegate_all_offline", s["collectors_two"], two, delegate=True, queues={9001: None, 9002: None})
    case("delegate_no_workers", s["collectors_two"], two, ids=(), delegate=True)
    for n in (0, 1, 3):
        case(f"seed_value_{n}_workers", s["seed_value"], three, ids=[f"w{i + 1}" for i in range(n)])
    case("seed_value_one_offline", s["seed_value"], three, ids=("w1", "w2", "w3"), queues={9001: 0, 9002: None, 9003: 0})
    case("enabled_from_config", s["seed_value"], {"workers": _workers(2) + [{"id": "w3", "port": 9003, "enabled": False}],
                                                  "settings": settings}, body={"prompt": s["seed_value"],
                                                                               "client_id": "c", "workers": [
                                                                                   {"id": "w2"}, "w1", None]})
    # load_balance: idle workers in turn, else the shortest queue; the master competes unless delegate-only
    case("load_balance_busy", s["load_balance"], three, ids=("w1", "w2", "w3"), queues={9001: 4, 9002: 2, 9003: 3,
                                                                                       MASTER_PORT: 5})
    case("load_balance_master_idle", s["load_balance"], three, ids=("w1", "w2", "w3"),
         queues={9001: 4, 9002: 2, 9003: 3, MASTER_PORT: 0})
    case("load_balance_idle", s["load_balance"], three, ids=("w1", "w2", "w3"), queues={9001: 1, 9002: 0, 9003: 0,
                                                                                       MASTER_PORT: 0})
    case("load_balance_delegate", s["load_balance"], three, ids=("w1", "w2", "w3"), delegate=True,
         queues={9001: 3, 9002: 1, 9003: 2, MASTER_PORT: 0})
    case("load_balance_no_workers", s["load_balance"], three, ids=(), queues={MASTER_PORT: 2})
    # remote workers: paths converted for the worker's separator; callbacks at the configured master host
    remote = {"master": {"host": "master.example:8190"}, "settings": settings,
              "workers": [{"id": "r1", "host": "10.0.0.5", "port": 9001, "type": "remote", "enabled": True},
                          {"id": "r2", "host": "10.0.0.6", "port": 9002, "type": "remote", "enabled": True}]}
    case("remote_paths", s["collectors_two"], remote, ids=("r1", "r2"), seps={9001: "\\", 9002: "/"})
    case("invalid_master_prompt", s["collectors_two"], two, invalid=True)
    return out


# malformed bodies of POST /distributed/queue (each a raw text)
BAD_BODIES = [
    "", "{", "[]", "null", "3", '"x"',
    '{"prompt": {}, "client_id": "c", "enabled_worker_ids": [], "auto_prepare": "yes"}',
    '{"client_id": "c", "enabled_worker_ids": []}',
    '{"prompt": [], "client_id": "c", "enabled_worker_ids": []}',
    '{"workflow": {"prompt": []}, "client_id": "c", "enabled_worker_ids": []}',
    '{"workflow": "x", "client_id": "c", "enabled_worker_ids": []}',
    '{"prompt": {}, "client_id": "c"}',
    '{"prompt": {}, "client_id": "c", "workers": "w1"}',
    '{"prompt": {}, "client_id": "c", "enabled_worker_ids": "w1"}',
    '{"prompt": {}, "client_id": "c", "enabled_worker_ids": {"w1": 1}}',
    '{"prompt": {}, "client_id": "c", "enabled_worker_ids": [], "delegate_master": 1}',
    '{"prompt": {}, "client_id": "c", "enabled_worker_ids": [], "delegate_master": "true"}',
    '{"prompt": {}, "enabled_worker_ids": []}',
    '{"prompt": {}, "client_id": "   ", "enabled_worker_ids": []}',
    '{"prompt": {}, "client_id": 5, "enabled_worker_ids": []}',
    '{"prompt": {}, "client_id": "c", "enabled_worker_ids": [], "trace_execution_id": 5}',
    '{"prompt": {}, "client_id": "c", "enabled_worker_ids": ["  "], "trace_execution_id": "  "}',
    '{"prompt": {}, "client_id": "c", "enabled_worker_ids": [], "auto_prepare": null}',
    '{"prompt": null, "workflow": {"prompt": {}}, "client_id": "c", "workers": [{"id": 1}, {"x": 1}, 2]}',
]


# --------------------------------------------------------------------------------------
# the reference, loaded under stubs
# --------------------------------------------------------------------------------------
def _mod(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


def _load(root, name, rel):
    spec = importlib.util.spec_from_file_location(f"{PKG}.{name}", os.path.join(root, rel))
    m = importlib.util.module_from_spec(spec)
    sys.modules[f"{PKG}.{name}"] = m
    spec.loader.exec_module(m)
    return m


def load_reference(root: str):
    """-> (job_routes module, the stub PromptServer, the stub execution module, the reference's modules by name)."""
    from aiohttp import web
    inst = PromptServer()
    inst.routes = web.RouteTableDef()
    _mod("server", PromptServer=types.SimpleNamespace(instance=inst))
    execution = _mod("execution", validate_prompt=validator(False))
    mm = _mod("comfy.model_management", processing_interrupted=lambda: False,
              throw_exception_if_processing_interrupted=lambda: None)
    cu = _mod("comfy.utils", ProgressBar=lambda *a, **k: types.SimpleNamespace(update=lambda *a, **k: None))
    _mod("comfy", model_management=mm, utils=cu)
    for p in (PKG, PKG + ".utils", PKG + ".api", PKG + ".api.orchestration"):
        _mod(p).__path__ = []
    noop = lambda *a, **k: None  # noqa: E731
    _mod(PKG + ".utils.logging", debug_log=noop, log=noop)
    _mod(PKG + ".utils.trace_logger", trace_debug=noop, trace_info=noop)
    mods = {}
    for name, rel in (("utils.constants", "utils/constants.py"), ("utils.config", "utils/config.py"),
                      ("utils.network", "utils/network.py"), ("utils.async_helpers", "utils/async_helpers.py"),
                      ("utils.image", "utils/image.py"), ("api.schemas", "api/schemas.py"),
                      ("api.orchestration.prompt_transform", "api/orchestration/prompt_transform.py"),
                      ("api.orchestration.dispatch", "api/orchestration/dispatch.py"),
                      ("api.orchestration.media_sync", "api/orchestration/media_sync.py"),
                      ("api.queue_request", "api/queue_request.py"),
                      ("api.queue_orchestration", "api/queue_orchestration.py"),
                      ("api.job_routes", "api/job_routes.py")):
        mods[name] = _load(root, name, rel)
    return mods["api.job_routes"], inst, execution, mods


def run_reference_case(mods, inst, execution, case) -> dict:
    qo, disp = mods["api.queue_orchestration"], mods["api.orchestration.dispatch"]
    session = FakeSession(case["queues"], case["seps"])

    async def get_session():
        return session

    async def no_media(*a, **k):
        return None
    for m in (mods["utils.network"], disp, mods["api.orchestration.media_sync"]):
        m.get_client_session = get_session
    cfg = json.loads(json.dumps(case["config"]))
    merged = mods["utils.config"]._merge_with_defaults(cfg, mods["utils.config"].get_default_config())
    qo.load_config = lambda: merged
    qo.sync_worker_media = no_media
    qo.time = types.SimpleNamespace(time=lambda: FIXED_MS / 1000)
    qo.uuid = types.SimpleNamespace(uuid4=lambda: types.SimpleNamespace(hex=FIXED_HEX + "000000"))
    disp._least_busy_rr_index = 0
    inst.number, inst.distributed_pending_jobs = 0, {}
    inst.queued.clear()
    execution.validate_prompt = validator(case["invalid"])
    handler = mods["api.job_routes"].distributed_queue_endpoint

    async def go():
        inst.distributed_jobs_lock = asyncio.Lock()
        return await handler(FakeRequest(json.dumps(case["body"])))
    resp = asyncio.run(go())
    return observed(resp, session, inst, sorted(inst.distributed_pending_jobs))


def observed(resp, session, server, queues) -> dict:
    """What a case's run shows: the reply (without the random prompt_id), the POST bodies by URL, the master's queue
    items (without create_time and prompt_id) and the collector queues opened."""
    body = reply_json(resp)
    body.pop("prompt_id", None)
    return {"status": resp.status, "reply": body, "posts": [[u, b] for u, b in session.posts],
            "queued": queued_items(server), "queues": queues}


def queued_items(server) -> list:
    return [{"number": number, "prompt": prompt, "extra_data": {k: v for k, v in extra.items() if k != "create_time"},
             "outputs": outputs, "sensitive": sensitive}
            for number, _pid, prompt, extra, outputs, sensitive in server.queued]


def run_reference_bad_body(mods, raw: str) -> dict:
    async def go():
        return await mods["api.job_routes"].distributed_queue_endpoint(FakeRequest(raw))
    resp = asyncio.run(go())
    return {"status": resp.status, "reply": reply_json(resp)}


def main():
    sys.path.insert(0, HERE)
    import make_ref
    root = make_ref.staged_root()
    if not root:
        raise SystemExit("ref_orchestration: the reference tree or its bundle is needed")
    wf_dir = os.path.join(make_ref.SRC, "workflows")
    workflows = {wf: api_prompt(json.load(open(os.path.join(wf_dir, wf)))) for wf in WORKFLOWS}
    _, inst, execution, mods = load_reference(root)
    out_cases = []
    for c in cases(workflows):
        c["expect"] = run_reference_case(mods, inst, execution, c)
        out_cases.append(c)
    # bad bodies: the orchestration is never reached; a body that parses is marked ok
    bad = []
    for raw in BAD_BODIES:
        try:
            parsed = mods["api.queue_request"].parse_queue_request_payload(json.loads(raw))
            bad.append({"raw": raw, "ok": True, "parsed": dataclasses.asdict(parsed)})
        except Exception:
            bad.append({"raw": raw, "ok": False, "expect": run_reference_bad_body(mods, raw)})
    with open(GOLDEN, "w") as f:
        json.dump({"prefix": f"exec_{FIXED_MS}_{FIXED_HEX}", "cases": out_cases, "bad_bodies": bad}, f)
    print(f"ref_orchestration: {len(out_cases)} cases, {len(bad)} bodies -> {GOLDEN}")


if __name__ == "__main__":
    main()
