"""The routes a reference master and the reference's web UI call on each worker: `GET /distributed/worker_ws` (prompt
dispatch over a WebSocket, api/worker_routes.py:43-112), `GET /distributed/system_info` (:408-430),
`POST /distributed/check_file` (api/job_routes.py:79-101, :255-270), `POST /distributed/clear_memory` (:160-203) and
`GET /distributed/local_log` (api/worker_routes.py:328-390), with the reference's status codes and JSON bodies.

A master at the reference's default `websocket_orchestration: true` probes its workers by opening worker_ws and skips
those that refuse it; with these routes a worker running this package takes part.  Prompts arriving on the socket are
queued as ComfyUI's POST /prompt queues them (orchestrator.queue_prompt).

Differences from the reference (INTEGRATION.md, "Workers of a reference master"):
* check_file answers `exists: false` for a name that resolves outside ComfyUI's input, output and temp directories,
  without reading it (the master then uploads the file as usual); the reference hashes any file on the machine;
* clear_memory also releases this package's device caches (engine.release_device_caches), which ComfyUI's
  unload_all_models and soft_empty_cache do not reach.
"""
from __future__ import annotations

import asyncio
import gc
import hashlib
import json
import logging
import os
import platform
import socket
import uuid
import warnings

MEMORY_CLEAR_DELAY = 0.5        # utils/constants.py:40: s for the queue to act on its flags
LOG_LINES, LOG_LINES_MAX = 300, 3000

log = logging.getLogger(__name__)


def _error(error, status):
    from aiohttp import web
    if isinstance(error, list):
        return web.json_response({"errors": [str(e) for e in error]}, status=status)
    return web.json_response({"error": str(error)}, status=status)


def _ack(request_id, ok: bool, **fields) -> dict:
    return {"type": "dispatch_ack", "request_id": request_id, "ok": ok, **fields}


async def dispatch_ack(server, validate, data) -> dict:
    """The answer to one decoded worker_ws message (a JSON object)."""
    from .orchestrator import PromptValidationError, queue_prompt
    rid = data.get("request_id")
    if data.get("type") != "dispatch_prompt":
        return _ack(rid, False, error="Unsupported websocket message type.")
    prompt = data.get("prompt")
    if not isinstance(prompt, dict):
        return _ack(rid, False, error="Field 'prompt' must be an object.")
    try:
        queued = await queue_prompt(server, prompt, data.get("workflow"), data.get("client_id"), validate)
        return _ack(rid, True, prompt_id=queued["prompt_id"])
    except PromptValidationError as exc:
        return _ack(rid, False, error=str(exc), validation_error=exc.validation_error, node_errors=exc.node_errors)
    except Exception as exc:
        return _ack(rid, False, error=str(exc))


def machine_id() -> str:
    """workers/detection.py:49-62."""
    try:
        return str(uuid.getnode())
    except Exception:
        try:
            return f"{platform.machine()}_{socket.gethostname()}"
        except Exception:
            return platform.machine()


def system_info() -> dict:
    """The reference's expressions (workers/detection.py:64-73): is_docker can be the DOCKER_CONTAINER string."""
    return {
        "status": "success",
        "hostname": socket.gethostname(),
        "machine_id": machine_id(),
        "platform": {"system": platform.system(), "machine": platform.machine(), "node": platform.node(),
                     "path_separator": os.sep, "os_name": os.name},
        "is_docker": (os.path.exists("/.dockerenv") or os.environ.get("DOCKER_CONTAINER", False)
                      or "docker" in platform.node().lower()),
        "is_runpod": os.environ.get("RUNPOD_POD_ID") is not None or os.environ.get("RUNPOD_API_KEY") is not None,
        "runpod_pod_id": os.environ.get("RUNPOD_POD_ID"),
    }


def _inside(path: str, dirs) -> bool:
    path = os.path.realpath(path)
    for d in dirs:
        d = os.path.realpath(d)
        try:
            if os.path.commonpath([path, d]) == d:
                return True
        except ValueError:                      # another drive
            pass
    return False


def check_file(filename, expected_hash) -> dict:
    """Whether this ComfyUI has `filename` (a name as its LoadImage takes, annotations included) with MD5
    `expected_hash`.  A name outside the input, output and temp directories counts as missing and is not read."""
    import folder_paths
    path = folder_paths.get_annotated_filepath(filename)
    roots = (folder_paths.get_input_directory(), folder_paths.get_output_directory(), folder_paths.get_temp_directory())
    if not _inside(path, roots) or not os.path.exists(path):
        return {"status": "success", "exists": False}
    md5 = hashlib.md5()
    with open(path, "rb") as f:
        for chunk in iter(lambda: f.read(4096), b""):
            md5.update(chunk)
    return {"status": "success", "exists": True, "hash_matches": md5.hexdigest() == expected_hash}


def _lines_query(value) -> int:
    """_parse_positive_int_query (api/worker_routes.py:328-337) with the local_log bounds."""
    try:
        return min(LOG_LINES_MAX, max(1, int(value)))
    except (TypeError, ValueError):
        return LOG_LINES


def make_handlers(server, validate=None):
    """The five handlers -> {(method, path): handler}.  `server`: ComfyUI's PromptServer (trigger_on_prompt, number,
    prompt_queue); `validate`: execution.validate_prompt when None."""
    from aiohttp import WSMsgType, web

    async def worker_ws(request):
        ws = web.WebSocketResponse(heartbeat=30)
        await ws.prepare(request)
        async for msg in ws:
            if msg.type == WSMsgType.TEXT:
                try:
                    data = json.loads(msg.data or "{}")
                except json.JSONDecodeError:
                    await ws.send_json(_ack(None, False, error="Invalid JSON payload."))
                    continue
                if not isinstance(data, dict):
                    # the reference's handler fails on such a message and aiohttp drops the connection
                    raise TypeError(f"worker_ws: a message must be a JSON object, got {type(data).__name__}")
                await ws.send_json(await dispatch_ack(server, validate, data))
            elif msg.type == WSMsgType.ERROR:
                log.warning("comfyui-distributed_b200: worker websocket error: %s", ws.exception())
        return ws

    async def system_info_route(request):
        try:
            return web.json_response(system_info())
        except Exception as exc:
            return _error(exc, 500)

    async def check_file_route(request):
        try:
            data = await request.json()
            filename, expected = data.get("filename"), data.get("hash")
            if not filename or not expected:
                return _error("Missing filename or hash", 400)
            reply = await asyncio.get_running_loop().run_in_executor(None, check_file, filename, expected)
            return web.json_response(reply)
        except Exception as exc:
            return _error(exc, 500)

    async def clear_memory(request):
        import torch
        try:
            if hasattr(server, "prompt_queue"):
                server.prompt_queue.set_flag("unload_models", True)
                server.prompt_queue.set_flag("free_memory", True)
            await asyncio.sleep(MEMORY_CLEAR_DELAY)
            import comfy.model_management as mm
            try:
                mm.unload_all_models()
            except AttributeError as exc:
                log.debug("clear_memory: model unload: %s", exc)
            try:
                mm.soft_empty_cache()
            except Exception as exc:
                log.debug("clear_memory: cache clear: %s", exc)
            from .engine import release_device_caches
            release_device_caches()
            for _ in range(3):
                gc.collect()
            if torch.cuda.is_available():
                torch.cuda.empty_cache()
                torch.cuda.ipc_collect()
            return web.json_response({"status": "success", "message": "GPU memory cleared."})
        except Exception as exc:
            gc.collect()
            if torch.cuda.is_available():
                torch.cuda.empty_cache()
            log.debug("clear_memory: partial clear: %s", exc)
            return web.json_response({"status": "success", "message": "GPU memory cleared (with warnings)"})

    async def local_log(request):
        try:
            from app.logger import get_logs
        except Exception as exc:
            return _error(f"Failed to import app.logger: {exc}", 500)
        try:
            lines = _lines_query(request.query.get("lines"))
            logs = get_logs()
            if logs is None:
                return web.json_response({"status": "success", "content": "", "entries": 0, "source": "memory",
                                          "truncated": False, "lines_shown": 0})
            entries = list(logs)
            shown = entries[-lines:]
            content = "".join(e.get("m", "") if isinstance(e, dict) else str(e) for e in shown)
            return web.json_response({"status": "success", "content": content, "entries": len(shown),
                                      "source": "memory", "truncated": len(entries) > len(shown),
                                      "lines_shown": content.count("\n") + (1 if content else 0)})
        except Exception as exc:
            return _error(exc, 500)

    return {("GET", "/distributed/worker_ws"): worker_ws, ("GET", "/distributed/system_info"): system_info_route,
            ("POST", "/distributed/check_file"): check_file_route, ("POST", "/distributed/clear_memory"): clear_memory,
            ("GET", "/distributed/local_log"): local_log}


WS_ROUTE = ("GET", "/distributed/worker_ws")
_served: set = set()
_warned: set = set()


def register(routes, server, validate=None, module_state: bool = True) -> set:
    """Add the handlers to an aiohttp RouteTableDef, skipping, with one warning each, every path another package
    already serves.  -> the (method, path) pairs served."""
    taken = {(getattr(r, "method", None), getattr(r, "path", None)) for r in routes}
    served = set()
    for (method, path), fn in make_handlers(server, validate).items():
        if (method, path) in taken:
            if (method, path) not in _warned:
                _warned.add((method, path))
                warnings.warn(f"comfyui-distributed_b200: {method} {path} is already served by another package; "
                              "this package's handler stays off", RuntimeWarning, stacklevel=2)
            continue
        routes.route(method, path)(fn)
        served.add((method, path))
    if module_state:
        _served.update(served)
    return served


def install(server):
    """Register on ComfyUI's PromptServer once (http_master.install_in_comfyui)."""
    if not _served:
        register(server.routes, server)


def serving() -> bool:
    """This process serves GET /distributed/worker_ws."""
    return WS_ROUTE in _served


def reset_for_tests():
    """Forget the registration (test harnesses that start and stop their own server)."""
    _served.clear()
    _warned.clear()
