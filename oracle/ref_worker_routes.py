"""The reference's worker routes (api/worker_routes.py: worker_ws, system_info, local_log; api/job_routes.py: check_file,
clear_memory), run for real under stubs -- TEST INFRASTRUCTURE ONLY; generating needs the reference tree or the bundle
oracle/make_ref.py packs.

`python oracle/ref_worker_routes.py` runs every case of `cases()` through the reference's handlers and writes what they
answered to tests/golden/worker_routes.json: the status and JSON body of each request, and for worker_ws the frames the
client received in order and the close code it saw.  The stand-ins: the PromptServer (ref_orchestration.PromptServer
with a queue that records its flags), execution.validate_prompt, folder_paths over a scratch directory, app.logger,
comfy.model_management, uuid.getnode, socket.gethostname, platform and the environment.  The prompt id of an ack (a
uuid4) is written as the index of the queue item it names.  Only replies are written, no reference source.

The same stand-ins and drivers run this package's worker_routes.py in tests/test_worker_routes.py.
"""
from __future__ import annotations

import asyncio
import contextlib
import hashlib
import json
import os
import platform
import shutil
import socket
import sys
import tempfile
import types
import uuid
from unittest import mock

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(os.path.dirname(HERE), "tests", "golden", "worker_routes.json")
sys.path.insert(0, HERE)
import ref_orchestration as ro  # noqa: E402

FILES = {"input/pic.png": b"a picture", "input/sub/clip.mp4": b"a clip", "output/result.png": b"a result",
         "temp/t.png": b"a temp file"}


def md5(data: bytes) -> str:
    return hashlib.md5(data).hexdigest()


# --------------------------------------------------------------------------------------
# stand-ins
# --------------------------------------------------------------------------------------
def reset_server(server, queue: str = "ok"):
    """`server` (a ref_orchestration.PromptServer) with an empty queue: "ok", "raises" (put raises) or "none" (no
    prompt_queue attribute).  server.flags records set_flag calls."""
    server.number, server.queued, server.flags = 0, [], []
    if queue == "none":
        if hasattr(server, "prompt_queue"):
            del server.prompt_queue
        return server

    def put(item):
        if queue == "raises":
            raise RuntimeError("the prompt queue is closed")
        server.queued.append(item)
    server.prompt_queue = types.SimpleNamespace(put=put, set_flag=lambda k, v: server.flags.append([k, v]))
    return server


def folder_paths(root: str):
    """ComfyUI's folder_paths over root/{input,output,temp}: "name [output]" and "name [temp]" name those directories,
    any other name the input directory."""
    dirs = {k: os.path.join(root, k) for k in ("input", "output", "temp")}

    def get_annotated_filepath(name, default_dir=None):
        for kind in ("input", "output", "temp"):
            if name.endswith(f"[{kind}]"):
                return os.path.join(dirs[kind], name[:-len(kind) - 2].strip())
        return os.path.join(default_dir or dirs["input"], name)
    return types.SimpleNamespace(get_annotated_filepath=get_annotated_filepath,
                                 get_input_directory=lambda: dirs["input"], get_output_directory=lambda: dirs["output"],
                                 get_temp_directory=lambda: dirs["temp"])


def make_files(root: str):
    for rel, data in FILES.items():
        path = os.path.join(root, rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "wb") as f:
            f.write(data)
    return root


@contextlib.contextmanager
def system_patched(case: dict):
    """uuid.getnode, socket.gethostname, platform.* and /.dockerenv fixed; the environment's Docker and RunPod
    variables as the case sets them."""
    real_exists = os.path.exists
    env = {k: v for k, v in os.environ.items() if k not in ("DOCKER_CONTAINER", "RUNPOD_POD_ID", "RUNPOD_API_KEY")}
    env.update(case.get("env", {}))
    with mock.patch.object(uuid, "getnode", lambda: 0x0242AC110002), \
            mock.patch.object(socket, "gethostname", lambda: "gpu-host-7"), \
            mock.patch.object(platform, "system", lambda: "Linux"), \
            mock.patch.object(platform, "machine", lambda: "x86_64"), \
            mock.patch.object(platform, "node", lambda: case.get("node", "gpu-host-7")), \
            mock.patch.object(os.path, "exists", lambda p: False if p == "/.dockerenv" else real_exists(p)), \
            mock.patch.dict(os.environ, env, clear=True):
        yield


def model_management(mode: str, calls: list):
    """comfy.model_management whose unload_all_models / soft_empty_cache record their calls and raise as `mode` says:
    "ok", "unload_attr" (AttributeError), "unload_runtime", "soft_runtime", "both"."""
    def unload():
        calls.append("unload_all_models")
        if mode in ("unload_attr", "both"):
            raise AttributeError("'NoneType' object has no attribute 'model_unload'")
        if mode == "unload_runtime":
            raise RuntimeError("CUDA error: out of memory")

    def soft():
        calls.append("soft_empty_cache")
        if mode in ("soft_runtime", "both"):
            raise RuntimeError("soft_empty_cache failed")
    return types.ModuleType("comfy.model_management"), unload, soft


@contextlib.contextmanager
def modules_patched(case: dict, root: str, calls: list):
    """folder_paths, app.logger and comfy.model_management in sys.modules for one case; restored after."""
    names = ("folder_paths", "app.logger", "comfy", "comfy.model_management")
    saved = {k: sys.modules.get(k) for k in names}
    try:
        sys.modules["folder_paths"] = folder_paths(root)
        logs = case.get("logs", "absent")
        if logs == "absent":
            sys.modules["app.logger"] = None            # import of app.logger halted; None in sys.modules
        else:
            if isinstance(logs, dict):
                logs = [{"m": f"{k}\n"} for k in range(logs["generated"])]
            sys.modules["app.logger"] = types.SimpleNamespace(get_logs=lambda: logs)
        mm, unload, soft = model_management(case.get("mm", "ok"), calls)
        mm.unload_all_models, mm.soft_empty_cache = unload, soft
        sys.modules["comfy.model_management"] = mm
        sys.modules["comfy"] = types.SimpleNamespace(model_management=mm)
        yield
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


class Request:
    """What the handlers read of an aiohttp request: the body as JSON and the query."""

    def __init__(self, raw: str = "", query=None):
        self.raw, self.query = raw, dict(query or {})

    async def json(self):
        return json.loads(self.raw)


# --------------------------------------------------------------------------------------
# the cases
# --------------------------------------------------------------------------------------
PROMPT = {"1": {"class_type": "LoadImage", "inputs": {"image": "pic.png"}},
          "9": {"class_type": "SaveImage", "inputs": {"images": ["1", 0]}}}


def _dispatch(rid, prompt=PROMPT, **extra):
    return {"text": json.dumps({"type": "dispatch_prompt", "request_id": rid, "prompt": prompt, **extra})}


def cases() -> dict:
    ws = [
        {"name": "probe", "messages": []},
        {"name": "invalid_json", "messages": [{"text": "{not json"}]},
        {"name": "empty_text", "messages": [{"text": ""}]},
        {"name": "unsupported_type", "messages": [{"text": json.dumps({"type": "ping", "request_id": "r1"})}]},
        {"name": "prompt_missing", "messages": [{"text": json.dumps({"type": "dispatch_prompt", "request_id": "r1"})}]},
        {"name": "prompt_not_object", "messages": [_dispatch("r1", prompt=[1, 2])]},
        {"name": "dispatch", "messages": [_dispatch("r1", workflow={"nodes": [1]}, client_id="client-1")]},
        {"name": "dispatch_bare", "messages": [_dispatch(None)]},
        {"name": "several", "messages": [
            {"text": "{"}, {"binary": "00ff"}, {"text": json.dumps({"type": "other", "request_id": 7})},
            _dispatch("a", workflow={"w": 1}, client_id="c"), _dispatch("b", client_id="c2"),
            _dispatch("c", prompt="x")]},
        {"name": "validation_failure", "invalid": True, "messages": [_dispatch("r1", client_id="c")]},
        {"name": "queue_raises", "queue": "raises", "messages": [_dispatch("r1")]},
        {"name": "array_closes", "messages": [_dispatch("r1"), {"text": "[1, 2]"}, _dispatch("r2")]},
        {"name": "null_closes", "messages": [{"text": "null"}]},
    ]
    check = [{"name": n, "raw": raw} for n, raw in (
        ("bad_json", "{"), ("not_object", "[]"), ("number", "3"), ("empty", "{}"),
        ("no_hash", json.dumps({"filename": "pic.png"})), ("no_filename", json.dumps({"hash": md5(b"a picture")})),
        ("empty_filename", json.dumps({"filename": "", "hash": "x"})),
        ("missing_file", json.dumps({"filename": "gone.png", "hash": "x"})),
        ("match", json.dumps({"filename": "pic.png", "hash": md5(b"a picture")})),
        ("mismatch", json.dumps({"filename": "pic.png", "hash": md5(b"another picture")})),
        ("subfolder", json.dumps({"filename": "sub/clip.mp4", "hash": md5(b"a clip")})),
        ("input_annotated", json.dumps({"filename": "pic.png [input]", "hash": md5(b"a picture")})),
        ("output_annotated", json.dumps({"filename": "result.png [output]", "hash": md5(b"a result")})),
        ("temp_annotated", json.dumps({"filename": "t.png [temp]", "hash": md5(b"a temp")})))]
    system = [{"name": "plain"}, {"name": "docker_env", "env": {"DOCKER_CONTAINER": "yes"}},
              {"name": "docker_node", "node": "Docker-Desktop"},
              {"name": "runpod", "env": {"RUNPOD_POD_ID": "pod-42"}},
              {"name": "runpod_key", "env": {"RUNPOD_API_KEY": "k"}},
              {"name": "docker_and_runpod", "env": {"DOCKER_CONTAINER": "1", "RUNPOD_POD_ID": "pod-7"}}]
    mixed = [{"m": "first\n"}, "second\n", {"t": 1.5}, {"m": "a\nb\n"}, 17, {"m": "last"}]
    many = {"generated": 3005}                  # {"m": "<k>\n"} for k < 3005
    log = [{"name": "no_logger", "logs": "absent"}, {"name": "none", "logs": None}, {"name": "empty", "logs": []}]
    for q in (None, "0", "abc", "5000", "2", "-3", "1.5"):
        log.append({"name": f"mixed_lines_{q}", "logs": mixed, "query": {} if q is None else {"lines": q}})
    for q in (None, "5000", "3000"):
        log.append({"name": f"many_lines_{q}", "logs": many, "query": {} if q is None else {"lines": q}})
    clear = [{"name": f"{mm}_{queue}", "mm": mm, "queue": queue}
             for queue in ("ok", "none") for mm in ("ok", "unload_attr", "unload_runtime", "soft_runtime", "both")]
    return {"worker_ws": ws, "check_file": check, "system_info": system, "local_log": log, "clear_memory": clear}


# --------------------------------------------------------------------------------------
# drivers, for the reference's handlers and for this package's
# --------------------------------------------------------------------------------------
def reply(resp) -> dict:
    return {"status": resp.status, "body": json.loads(resp.body)}


async def ws_exchange(handler, messages) -> dict:
    """Serve `handler` at /ws on 127.0.0.1, send `messages` one by one (a TEXT message waits for its answer) and
    -> {"frames": [JSON of each TEXT frame received], "close": the close code the client saw}."""
    import aiohttp
    from aiohttp import web
    app = web.Application()
    app.router.add_get("/ws", handler)
    runner = web.AppRunner(app)
    await runner.setup()
    site = web.TCPSite(runner, "127.0.0.1", 0)
    await site.start()
    port = site._server.sockets[0].getsockname()[1]
    frames = []
    try:
        async with aiohttp.ClientSession() as session:
            ws = await session.ws_connect(f"http://127.0.0.1:{port}/ws")
            for m in messages:
                if "binary" in m:
                    await ws.send_bytes(bytes.fromhex(m["binary"]))
                    continue
                await ws.send_str(m["text"])
                msg = await ws.receive(timeout=30)
                if msg.type != aiohttp.WSMsgType.TEXT:
                    break
                frames.append(json.loads(msg.data))
            if not ws.closed:
                await ws.close()
            return {"frames": frames, "close": ws.close_code}
    finally:
        await runner.cleanup()


def mask_prompt_ids(frames, server) -> list:
    """An ack's prompt_id (a uuid4) -> "queued[k]", k the queue item it names."""
    ids = [item[1] for item in server.queued]
    out = []
    for f in frames:
        f = dict(f)
        if "prompt_id" in f:
            assert str(uuid.UUID(f["prompt_id"], version=4)) == f["prompt_id"]
            f["prompt_id"] = f"queued[{ids.index(f['prompt_id'])}]"
        out.append(f)
    return out


def run_ws(handler, server, case) -> dict:
    got = asyncio.run(ws_exchange(handler, case["messages"]))
    return {"frames": mask_prompt_ids(got["frames"], server), "close": got["close"],
            "queued": ro.queued_items(server)}


def run_case(kind: str, case: dict, handlers: dict, server, execution=None, root: str = "") -> dict:
    """One case through `handlers` ({"worker_ws": fn, ...}).  `execution`: the module whose validate_prompt the
    handler calls (the reference's); this package's handlers are made with ro.validator(case["invalid"]) instead."""
    reset_server(server, case.get("queue", "ok"))
    if execution is not None:
        execution.validate_prompt = ro.validator(bool(case.get("invalid")))
    calls = []
    with modules_patched(case, root, calls), system_patched(case):
        if kind == "worker_ws":
            return run_ws(handlers[kind], server, case)
        req = Request(case.get("raw", ""), case.get("query"))
        out = reply(asyncio.run(handlers[kind](req)))
    if kind == "clear_memory":
        out["flags"], out["calls"] = server.flags, calls
    return out


# --------------------------------------------------------------------------------------
# the reference, loaded under stubs
# --------------------------------------------------------------------------------------
def load_reference(root: str):
    """-> (the reference's five handlers by kind, its PromptServer stand-in, its execution stand-in).  The
    reference's own network clients are in mods (ro.load_reference) and mods["workers.detection"]."""
    job_routes, inst, execution, mods = ro.load_reference(root)
    ro._mod(ro.PKG + ".workers", get_worker_manager=lambda: None).__path__ = []
    mods["workers.detection"] = ro._load(root, "workers.detection", "workers/detection.py")
    wr = ro._load(root, "api.worker_routes", "api/worker_routes.py")
    mods["api.worker_routes"] = wr
    job_routes.MEMORY_CLEAR_DELAY = 0
    handlers = {"worker_ws": wr.worker_ws_endpoint, "system_info": wr.get_system_info_endpoint,
                "local_log": wr.get_local_log_endpoint, "check_file": job_routes.check_file_endpoint,
                "clear_memory": job_routes.clear_memory_endpoint}
    return handlers, inst, execution, mods


def main():
    import make_ref
    root = make_ref.staged_root()
    if not root:
        raise SystemExit("ref_worker_routes: the reference tree or its bundle is needed")
    handlers, inst, execution, _ = load_reference(root)
    scratch = make_files(tempfile.mkdtemp(prefix="worker_routes_"))
    try:
        out = {kind: [{**c, "expect": run_case(kind, c, handlers, inst, execution, scratch)} for c in cs]
               for kind, cs in cases().items()}
    finally:
        shutil.rmtree(scratch, ignore_errors=True)
    with open(GOLDEN, "w") as f:
        json.dump({"files": {k: v.decode() for k, v in FILES.items()}, "cases": out}, f)
    print(f"ref_worker_routes: {sum(len(v) for v in out.values())} cases -> {GOLDEN}")


if __name__ == "__main__":
    main()
