"""The worker routes (worker_routes.py) against the reference's own: every case of tests/golden/worker_routes.json
(oracle/ref_worker_routes.py ran the reference's handlers on it) gets the same status and body, and on worker_ws the
same acks in the same order and the same close code.  Then check_file's one difference, route registration, and --
where the reference tree is present -- the reference's own client code against these routes on 127.0.0.1."""
import asyncio
import json
import os
import sys
import types
import warnings

import pytest

import ref_orchestration as ro
import ref_worker_routes as rw
from __graft_entry__ import load_package
from test_orchestrator import Loop

load_package()
from comfyui_distributed_b200 import worker_routes as wr  # noqa: E402

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "worker_routes.json")))
CASES = [(kind, c["name"]) for kind, cs in GOLDEN["cases"].items() for c in cs]
BY_NAME = {(kind, c["name"]): c for kind, cs in GOLDEN["cases"].items() for c in cs}


@pytest.fixture
def files(tmp_path):
    return rw.make_files(str(tmp_path))


@pytest.mark.parametrize("kind,name", CASES)
def test_reply_equals_reference(monkeypatch, files, kind, name):
    monkeypatch.setattr(wr, "MEMORY_CLEAR_DELAY", 0)
    case = BY_NAME[(kind, name)]
    server = ro.PromptServer()
    route = {"worker_ws": ("GET", "/distributed/worker_ws"), "system_info": ("GET", "/distributed/system_info"),
             "check_file": ("POST", "/distributed/check_file"), "clear_memory": ("POST", "/distributed/clear_memory"),
             "local_log": ("GET", "/distributed/local_log")}[kind]
    handler = wr.make_handlers(server, ro.validator(bool(case.get("invalid"))))[route]
    assert rw.run_case(kind, case, {kind: handler}, server, root=files) == case["expect"]


def test_golden_covers_the_cases():
    ws = {c["name"]: c["expect"] for c in GOLDEN["cases"]["worker_ws"]}
    assert ws["probe"] == {"frames": [], "close": 1000, "queued": []}
    assert [f["request_id"] for f in ws["several"]["frames"]] == [None, 7, "a", "b", "c"]       # binary: no ack
    assert ws["several"]["queued"][0]["extra_data"] == {"extra_pnginfo": {"workflow": {"w": 1}}, "client_id": "c"}
    assert ws["array_closes"]["close"] == ws["null_closes"]["close"] == 1006                  # dropped, no close frame
    assert ws["validation_failure"]["frames"][0]["node_errors"]
    clear = {c["name"]: c["expect"]["body"]["message"] for c in GOLDEN["cases"]["clear_memory"]}
    assert clear["unload_runtime_ok"] == "GPU memory cleared (with warnings)" and clear["both_ok"] == "GPU memory cleared."
    assert {c["expect"]["body"]["is_docker"] for c in GOLDEN["cases"]["system_info"]} == {False, True, "yes", "1"}


@pytest.mark.parametrize("name", ["../outside.png", "../input/../outside.png", "/{root}/outside.png",
                                  "escape.png", "escape.png [output]"])
def test_check_file_outside_comfy_directories_is_missing_and_unread(monkeypatch, files, name):
    """The reference hashes any file the name reaches; here a name outside input/output/temp answers exists: false
    without the file being opened (the master then uploads it as usual)."""
    outside = os.path.join(files, "outside.png")
    with open(outside, "wb") as f:
        f.write(b"secret")
    os.symlink(outside, os.path.join(files, "input", "escape.png"))
    os.symlink(outside, os.path.join(files, "output", "escape.png"))
    monkeypatch.setattr(wr, "open", lambda *a, **k: pytest.fail("a file outside the directories was opened"),
                        raising=False)
    monkeypatch.setitem(sys.modules, "folder_paths", rw.folder_paths(files))
    got = wr.check_file(name.replace("/{root}", files), rw.md5(b"secret"))
    assert got == {"status": "success", "exists": False}


def test_route_taken_by_another_package_is_skipped():
    from aiohttp import web
    wr.reset_for_tests()

    def theirs():
        routes = web.RouteTableDef()

        @routes.get("/distributed/system_info")
        async def system_info(request):
            return web.json_response({})
        return routes
    with warnings.catch_warnings(record=True) as seen:
        warnings.simplefilter("always")
        served = wr.register(theirs(), ro.PromptServer())
        wr.register(web.RouteTableDef(), ro.PromptServer(), module_state=False)
        wr.register(theirs(), ro.PromptServer(), module_state=False)          # warned once already
    assert [str(w.message) for w in seen] == [
        "comfyui-distributed_b200: GET /distributed/system_info is already served by another package; "
        "this package's handler stays off"]
    assert ("GET", "/distributed/system_info") not in served and len(served) == 4 and wr.serving()
    wr.reset_for_tests()
    assert not wr.serving()


# --------------------------------------------------------------------------------------
# the reference's client code against these routes (needs the reference tree)
# --------------------------------------------------------------------------------------
def _reference_root():
    import make_ref
    root = make_ref.staged_root()
    ok = root and all(os.path.isfile(os.path.join(root, p)) for p in (
        "api/orchestration/dispatch.py", "api/orchestration/media_sync.py", "workers/detection.py",
        "api/worker_routes.py"))
    return root if ok else None


REF_ROOT = _reference_root()
needs_reference = pytest.mark.skipif(not REF_ROOT, reason="reference tree not present")


@pytest.fixture(scope="module")
def ref():
    """The reference loaded under stubs; the ComfyUI stand-ins it puts in sys.modules are taken out again after."""
    names = ("server", "execution", "comfy", "comfy.model_management", "comfy.utils")
    saved = {k: sys.modules.get(k) for k in names}
    try:
        _, inst, _, mods = rw.load_reference(REF_ROOT)
        yield types.SimpleNamespace(inst=inst, mods=mods)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


class Worker:
    """This package's worker routes on 127.0.0.1 over a PromptServer stand-in; `invalid` makes validation refuse."""

    def __init__(self, lp: Loop):
        from aiohttp import web
        self.server, self.invalid = rw.reset_server(ro.PromptServer()), False

        async def validate(pid, prompt, partial):
            return await ro.validator(self.invalid)(pid, prompt, partial)
        routes = web.RouteTableDef()
        wr.register(routes, self.server, validate, module_state=False)
        self.port = lp.serve(routes)
        self.config = {"id": f"w{self.port}", "name": "Worker", "host": "127.0.0.1", "port": self.port,
                       "type": "local"}


@pytest.fixture
def lp():
    loop = Loop()
    yield loop
    loop.close()


def _run(ref, coro):
    """Run a coroutine of the reference's client code, then close its shared session."""
    async def go():
        try:
            return await coro
        finally:
            await ref.mods["utils.network"].cleanup_client_session()
    return asyncio.run(go())


@needs_reference
def test_reference_clients_against_these_routes(ref, lp, files, monkeypatch, caplog):
    disp = ref.mods["api.orchestration.dispatch"]
    media = ref.mods["api.orchestration.media_sync"]
    detection = ref.mods["workers.detection"]
    monkeypatch.setitem(sys.modules, "folder_paths", rw.folder_paths(files))
    w = Worker(lp)
    # the probe opens worker_ws and closes it at once: active, and nothing logged as an error
    assert _run(ref, disp.select_active_workers([w.config], True, False)) == ([w.config], False)
    assert not [r for r in caplog.records if r.levelname in ("ERROR", "CRITICAL")]
    # a prompt with its workflow and client id lands in the worker's queue
    _run(ref, disp.dispatch_worker_prompt(w.config, rw.PROMPT, {"w": 1}, client_id="cid", use_websocket=True))
    assert ro.queued_items(w.server) == [{"number": 0, "prompt": rw.PROMPT, "outputs": ["9"], "sensitive": {},
                                          "extra_data": {"extra_pnginfo": {"workflow": {"w": 1}}, "client_id": "cid"}}]
    # a validation failure raises the reference's message, built from the ack the golden file records
    w.invalid = True
    ack = BY_NAME[("worker_ws", "validation_failure")]["expect"]["frames"][0]
    want = f"{ack['error']} | validation_error={ack['validation_error']} | node_errors={ack['node_errors']}"
    with pytest.raises(RuntimeError) as err:
        _run(ref, disp.dispatch_worker_prompt(w.config, rw.PROMPT, None, client_id="c", use_websocket=True))
    assert str(err.value) == want and len(w.server.queued) == 1
    # system_info: this machine's separator, and the worker is recognised as being on this machine
    assert _run(ref, media.fetch_worker_path_separator(w.config)) == os.sep
    assert _run(ref, detection.is_same_physical_host(w.config)) is True
    # check_file: a file the worker has is not uploaded again; one whose hash differs goes on to the upload
    assert _run(ref, media._upload_media_to_worker(w.config, "sub\\clip.mp4", b"a clip", rw.md5(b"a clip"),
                                                    "video/mp4")) == (False, "sub/clip.mp4")
    import aiohttp
    with pytest.raises(aiohttp.ClientResponseError) as err:         # this stand-in serves no /upload/image
        _run(ref, media._upload_media_to_worker(w.config, "pic.png", b"new", rw.md5(b"new"), "image/png"))
    assert err.value.request_info.url.path == "/upload/image"


@needs_reference
def test_reference_queue_at_default_config_dispatches_to_these_workers(ref, lp):
    """The reference's whole /distributed/queue handler with websocket_orchestration left at its default (true):
    both workers are probed and sent their prompts over worker_ws, and each prompt is the one the reference's HTTP
    dispatch posts (tests/golden/orchestration.json)."""
    golden = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "orchestration.json")))
    case = next(c for c in golden["cases"] if c["name"] == "workflow:distributed-upscale.json")
    workers = {"w1": Worker(lp), "w2": Worker(lp)}
    cfg = json.loads(json.dumps(case["config"]))
    for w in cfg["workers"]:
        w["port"] = workers[w["id"]].port
    cfg["settings"].pop("websocket_orchestration")
    mods, inst = ref.mods, ref.inst
    conf = mods["utils.config"]
    merged = conf._merge_with_defaults(cfg, conf.get_default_config())
    assert merged["settings"]["websocket_orchestration"] is True
    qo = mods["api.queue_orchestration"]
    saved = qo.load_config, qo.time, qo.uuid
    qo.load_config = lambda: merged
    qo.time = types.SimpleNamespace(time=lambda: ro.FIXED_MS / 1000)
    qo.uuid = types.SimpleNamespace(uuid4=lambda: types.SimpleNamespace(hex=ro.FIXED_HEX + "000000"))
    mods["api.orchestration.dispatch"]._least_busy_rr_index = 0
    sys.modules["execution"].validate_prompt = ro.validator(False)
    rw.reset_server(inst)
    inst.distributed_pending_jobs = {}

    async def queue():
        inst.distributed_jobs_lock = asyncio.Lock()
        return await mods["api.job_routes"].distributed_queue_endpoint(ro.FakeRequest(json.dumps(case["body"])))
    try:
        resp = _run(ref, queue())
    finally:
        qo.load_config, qo.time, qo.uuid = saved
    body = ro.reply_json(resp)
    assert resp.status == 200 and body["worker_count"] == 2, body
    for (_, posted), wid in zip(case["expect"]["posts"], ("w1", "w2")):
        got = ro.queued_items(workers[wid].server)
        assert len(got) == 1 and got[0]["prompt"] == posted["prompt"]
        assert got[0]["extra_data"] == {**posted.get("extra_data", {}), "client_id": case["body"]["client_id"]}
    assert ro.queued_items(inst) == case["expect"]["queued"]
