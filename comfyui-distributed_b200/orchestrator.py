"""The master's orchestrator: the reference's public `POST /distributed/queue` route (api/job_routes.py:206-236) and
`GET /distributed/queue_status/{job_id}` (api/config_routes.py:147-163), with the worker config, the prompt rewriting and
the dispatch behind them (api/queue_request.py, api/queue_orchestration.py, api/orchestration/, utils/config.py).

One POST takes a workflow's API prompt and the ids of the workers to use.  The orchestrator probes those workers
(`GET /prompt`), picks one participant when a DistributedCollector asks for load_balance, gives every distributed node a
job id, opens the collector queues in http_collector's store, writes each participant's prompt (the worker prompts are
pruned to the distributed nodes and what feeds them; every prompt gets the hidden inputs of DistributedSeed,
DistributedValue, DistributedCollector and UltimateSDUpscaleDistributed for its role), uploads the media a remote worker
lacks, posts each worker its prompt and queues the master's own prompt on this ComfyUI.  The nodes then run the master
roles of http_master.py and http_collector.py.  No pixel work happens here.

HTTP goes through one aiohttp session per request that reads no proxy from the environment (as http_worker.py).

Differences from the reference (INTEGRATION.md, "The orchestrator"):
* `websocket_orchestration: true` (the reference's default) probes and dispatches over `/distributed/worker_ws`; workers
  running this package serve it (worker_routes.py), but this orchestrator still probes and dispatches over HTTP and
  warns once;
* the config file is only read: its editing routes belong to the reference's web UI.
"""
from __future__ import annotations

import asyncio
import dataclasses
import hashlib
import json
import mimetypes
import os
import re
import time
import uuid
import warnings
from collections import deque
from typing import Dict, List, Optional

CONFIG_FILE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "gpu_config.json")

# utils/constants.py:57-68
PROBE_CONCURRENCY = int(os.environ.get("COMFYUI_ORCHESTRATION_WORKER_PROBE_CONCURRENCY", "8"))
PREP_CONCURRENCY = int(os.environ.get("COMFYUI_ORCHESTRATION_WORKER_PREP_CONCURRENCY", "4"))
MEDIA_SYNC_CONCURRENCY = int(os.environ.get("COMFYUI_ORCHESTRATION_MEDIA_SYNC_CONCURRENCY", "2"))
MEDIA_SYNC_TIMEOUT = float(os.environ.get("COMFYUI_ORCHESTRATION_MEDIA_SYNC_TIMEOUT", "120"))
PROBE_TIMEOUT = 3.0                 # dispatch.py:34, :229
DISPATCH_TIMEOUT = 60.0             # dispatch.py:139
SYSTEM_INFO_TIMEOUT = 5.0           # media_sync.py:132
CHECK_FILE_TIMEOUT = 6.0            # media_sync.py:156
UPLOAD_TIMEOUT = 30.0               # media_sync.py:182

COLLECTOR, USDU = "DistributedCollector", "UltimateSDUpscaleDistributed"


# --------------------------------------------------------------------------------------
# gpu_config.json (utils/config.py:22-97), read only
# --------------------------------------------------------------------------------------
def default_config() -> dict:
    return {
        "master": {"host": ""},
        "workers": [],
        "settings": {
            "debug": False,
            "auto_launch_workers": False,
            "stop_workers_on_master_exit": True,
            "master_delegate_only": False,
            "websocket_orchestration": True,
            "worker_probe_concurrency": 8,
            "worker_prep_concurrency": 4,
            "media_sync_concurrency": 2,
            "media_sync_timeout_seconds": 120,
        },
        "tunnel": {"status": "stopped", "public_url": "", "pid": None, "log_file": "", "previous_master_host": ""},
    }


def _merge(data, defaults):
    """The file's values over the defaults, key by key into nested objects; keys the defaults lack are kept."""
    if not isinstance(data, dict):
        return defaults
    out = {}
    for key, dflt in defaults.items():
        value = data.get(key, dflt)
        out[key] = _merge(value, dflt) if isinstance(dflt, dict) and isinstance(value, dict) else value
    for key, value in data.items():
        out.setdefault(key, value)
    return out


class Config:
    """gpu_config.json, re-read when its mtime changes; the defaults when it is missing or unreadable."""

    def __init__(self, path: str = CONFIG_FILE):
        self.path, self._cache, self._mtime = path, None, 0.0

    def load(self) -> dict:
        try:
            mtime = os.path.getmtime(self.path)
        except OSError:
            if self._cache is None:
                self._cache = default_config()
            return self._cache
        if self._cache is None or mtime != self._mtime:
            try:
                with open(self.path, "r", encoding="utf-8") as f:
                    self._cache = _merge(json.load(f), default_config())
            except Exception as exc:
                warnings.warn(f"comfyui-distributed_b200: cannot read {self.path} ({exc}); using the defaults",
                              RuntimeWarning, stacklevel=2)
                self._cache = default_config()
            self._mtime = mtime
        return self._cache


def positive_int(value, default: int) -> int:
    try:
        return max(1, int(value))
    except (TypeError, ValueError):
        return max(1, int(default))


def positive_float(value, default: float) -> float:
    try:
        return max(0.0, float(value))
    except (TypeError, ValueError):
        return max(0.0, float(default))


def resolve_workers(config: dict, requested_ids=None) -> List[dict]:
    """The participating workers: those named in `requested_ids`, or the enabled ones when it is None."""
    workers = []
    for w in config.get("workers", []):
        wid = str(w.get("id") or "").strip()
        if not wid:
            continue
        if requested_ids is not None:
            if wid not in requested_ids:
                continue
        elif not w.get("enabled", False):
            continue
        raw = w.get("port", w.get("listen_port", 8188))
        try:
            port = int(raw or 8188)
        except (TypeError, ValueError):
            port = 8188
        workers.append({"id": wid, "name": w.get("name", wid), "host": w.get("host"), "port": port,
                        "type": w.get("type", "local")})
    return workers


# --------------------------------------------------------------------------------------
# the request body (api/queue_request.py)
# --------------------------------------------------------------------------------------
@dataclasses.dataclass(frozen=True)
class QueueRequest:
    prompt: dict
    workflow_meta: object
    client_id: str
    delegate_master: Optional[bool]
    enabled_worker_ids: List[str]
    auto_prepare: bool
    trace_execution_id: Optional[str]


def parse_queue_request(data) -> QueueRequest:
    """The POST body -> QueueRequest, or ValueError with the reference's message."""
    if not isinstance(data, dict):
        raise ValueError("Expected a JSON object body")
    auto_prepare = data.get("auto_prepare", True)
    if not isinstance(auto_prepare, bool):
        raise ValueError("auto_prepare must be a boolean when provided")
    prompt = data.get("prompt")
    if prompt is None and isinstance(data.get("workflow"), dict) and isinstance(data["workflow"].get("prompt"), dict):
        prompt = data["workflow"]["prompt"]
    if not isinstance(prompt, dict):
        raise ValueError("Field 'prompt' must be an object")
    ids = data.get("enabled_worker_ids")
    workers = data.get("workers")
    if ids is None and workers is not None:
        if not isinstance(workers, list):
            raise ValueError("Field 'workers' must be a list when provided")
        ids = []
        for entry in workers:
            wid = entry.get("id") if isinstance(entry, dict) else entry
            if wid is not None:
                ids.append(str(wid))
    if ids is None:
        raise ValueError("enabled_worker_ids required")
    if not isinstance(ids, list):
        raise ValueError("enabled_worker_ids must be a list of worker IDs")
    ids = [str(w).strip() for w in ids if str(w).strip()]
    delegate = data.get("delegate_master")
    if delegate is not None and not isinstance(delegate, bool):
        raise ValueError("delegate_master must be a boolean when provided")
    client_id = data.get("client_id")
    if not isinstance(client_id, str) or not client_id.strip():
        raise ValueError("client_id required")
    trace = data.get("trace_execution_id")
    if trace is not None:
        if not isinstance(trace, str):
            raise ValueError("trace_execution_id must be a string when provided")
        trace = trace.strip() or None
    return QueueRequest(prompt=prompt, workflow_meta=data.get("workflow"), client_id=client_id.strip(),
                        delegate_master=delegate, enabled_worker_ids=ids, auto_prepare=auto_prepare,
                        trace_execution_id=trace)


# --------------------------------------------------------------------------------------
# prompt rewriting (api/orchestration/prompt_transform.py)
# --------------------------------------------------------------------------------------
def _nodes(prompt: dict):
    return ((str(k), v) for k, v in prompt.items() if isinstance(v, dict))


def _links(node: dict):
    """The source node ids of a node's linked inputs ([source id, output index])."""
    return [str(v[0]) for v in (node.get("inputs", {}) or {}).values() if isinstance(v, list) and len(v) == 2]


def nodes_of_class(prompt: dict, class_type: str) -> List[str]:
    return [nid for nid, node in _nodes(prompt) if node.get("class_type") == class_type]


def _copy(obj):
    return json.loads(json.dumps(obj))


class PromptIndex:
    """The submitted prompt, frozen: a fresh copy per participant, and its nodes by class and their inputs."""

    def __init__(self, prompt: dict):
        self._json = json.dumps(prompt)
        self.by_class: Dict[str, List[str]] = {}
        self.class_of: Dict[str, Optional[str]] = {}
        self.inputs: Dict[str, dict] = {}
        for nid, node in _nodes(prompt):
            ct = node.get("class_type")
            if ct:
                self.by_class.setdefault(ct, []).append(nid)
            self.class_of[nid] = ct
            self.inputs[nid] = node.get("inputs", {})
        self._upstream: Dict[tuple, bool] = {}

    def copy(self) -> dict:
        return json.loads(self._json)

    def of_class(self, class_type: str) -> List[str]:
        return self.by_class.get(class_type, [])

    def has_upstream(self, nid: str, class_type: str) -> bool:
        """A node of `class_type` feeds `nid`, directly or through other nodes."""
        key = (str(nid), class_type)
        if key not in self._upstream:
            self._upstream[key] = self._search_upstream(str(nid), class_type)
        return self._upstream[key]

    def _search_upstream(self, start: str, class_type: str) -> bool:
        seen, stack = set(), [start]
        while stack:
            nid = stack.pop()
            if nid in seen:
                continue
            seen.add(nid)
            for src in _links({"inputs": self.inputs.get(nid, {})}):
                if self.class_of.get(src) == class_type:
                    return True
                if src in self.inputs:
                    stack.append(src)
        return False


def downstream_of(prompt: dict, start_ids) -> set:
    consumers: Dict[str, set] = {}
    for nid, node in _nodes(prompt):
        for src in _links(node):
            consumers.setdefault(src, set()).add(nid)
    found, todo = set(start_ids), deque(start_ids)
    while todo:
        for nxt in consumers.get(todo.popleft(), ()):
            if nxt not in found:
                found.add(nxt)
                todo.append(nxt)
    return found


def upstream_of(prompt: dict, start_ids) -> set:
    found = {str(n) for n in start_ids}
    todo = deque(found)
    while todo:
        for src in _links(prompt.get(todo.popleft()) or {}):
            if src in prompt and src not in found:
                found.add(src)
                todo.append(src)
    return found


def _id_counter(prompt: dict):
    """New node ids above every numeric id of `prompt`."""
    top = 0
    for nid in prompt:
        try:
            top = max(top, int(nid))
        except (TypeError, ValueError):
            pass

    def next_id():
        nonlocal top
        top += 1
        return str(top)
    return next_id


def prune_for_worker(prompt: dict) -> dict:
    """The distributed nodes and everything upstream of them; a PreviewImage on each distributed node whose consumers
    were cut away, so the worker's ComfyUI still has an output to run."""
    dist = nodes_of_class(prompt, COLLECTOR) + nodes_of_class(prompt, USDU)
    if not dist:
        return prompt
    out = {nid: _copy(prompt[nid]) for nid in upstream_of(prompt, dist) if prompt.get(nid) is not None}
    next_id = _id_counter(prompt)
    for nid in dist:
        if nid in out and any(d != nid for d in downstream_of(prompt, [nid])):
            out[next_id()] = {"inputs": {"images": [nid, 0]}, "class_type": "PreviewImage",
                              "_meta": {"title": "Preview Image (auto-added)"}}
    return out


def delegate_master_prompt(prompt: dict, collector_ids: List[str]) -> dict:
    """The collectors and what runs after them, each collector fed a 64x64 DistributedEmptyImage in place of its
    upstream: the master of a delegate-only run only gathers."""
    keep = set(collector_ids) | downstream_of(prompt, collector_ids)
    out = {nid: _copy(prompt[nid]) for nid in keep if prompt.get(nid) is not None}
    for node in out.values():
        inputs = node.get("inputs")
        if not inputs:
            continue
        for name, value in list(inputs.items()):
            if isinstance(value, list) and len(value) == 2 and str(value[0]) not in out:
                inputs.pop(name, None)
    next_id = _id_counter(prompt)
    for cid in collector_ids:
        entry = out.get(cid)
        if not entry:
            continue
        pid = next_id()
        out[pid] = {"class_type": "DistributedEmptyImage", "inputs": {"height": 64, "width": 64, "channels": 3},
                    "_meta": {"title": "Distributed Empty Image (auto-added)"}}
        entry.setdefault("inputs", {})["images"] = [pid, 0]
    return out


def job_id_map(index: PromptIndex, prefix: str) -> Dict[str, str]:
    return {nid: f"{prefix}_{nid}" for nid in index.of_class(COLLECTOR) + index.of_class(USDU)}


def apply_overrides(prompt: dict, participant: str, enabled_ids: List[str], jobs: Dict[str, str], master_url: str,
                    delegate_master: bool, index: PromptIndex) -> dict:
    """Set the hidden inputs of every distributed node of `prompt` (in place) for `participant`: "master" or a worker
    id.  Worker k of `enabled_ids` is "worker_k" to DistributedSeed and DistributedValue.  A collector downstream of an
    UltimateSDUpscaleDistributed only passes its images through."""
    master = participant == "master"
    position = {wid: k for k, wid in enumerate(enabled_ids)}
    enabled_json = json.dumps(enabled_ids)

    def targets(class_type):
        return [(nid, prompt[nid]) for nid in index.of_class(class_type) if isinstance(prompt.get(nid), dict)]

    for class_type in ("DistributedSeed", "DistributedValue"):
        for _, node in targets(class_type):
            inputs = node.setdefault("inputs", {})
            inputs["is_worker"] = not master
            inputs["worker_id"] = "" if master else f"worker_{position.get(participant, 0)}"
    for class_type in (COLLECTOR, USDU):
        for nid, node in targets(class_type):
            if class_type == COLLECTOR and index.has_upstream(nid, USDU):
                node.setdefault("inputs", {})["pass_through"] = True
                continue
            inputs = node.setdefault("inputs", {})
            inputs["multi_job_id"] = jobs.get(nid, nid)
            inputs["is_worker"] = not master
            inputs["enabled_worker_ids"] = enabled_json
            if master:
                inputs.pop("master_url", None)
                inputs.pop("worker_id", None)
            else:
                inputs["master_url"] = master_url
                inputs["worker_id"] = participant
            if class_type == COLLECTOR:
                inputs["delegate_only"] = bool(delegate_master) if master else False
    return prompt


def load_balance_requested(index: PromptIndex) -> bool:
    for nid in index.of_class(COLLECTOR):
        value = index.inputs.get(nid, {}).get("load_balance", False)
        if isinstance(value, bool):
            on = value
        elif isinstance(value, (int, float)):
            on = bool(value)
        elif isinstance(value, str):
            on = value.strip().lower() in {"1", "true", "yes", "on"}
        else:
            on = False
        if on:
            return True
    return False


# --------------------------------------------------------------------------------------
# paths and media of remote workers (api/orchestration/media_sync.py)
# --------------------------------------------------------------------------------------
_EXT_ANY = (r"ckpt|safetensors|pt|pth|bin|yaml|json|png|jpg|jpeg|webp|gif|bmp|mp4|avi|mov|mkv|webm|"
            r"wav|mp3|flac|m4a|aac|ogg|opus|aiff|aif|wma|latent|txt|vae|lora|embedding")
_EXT_MEDIA = r"png|jpg|jpeg|webp|gif|bmp|mp4|avi|mov|mkv|webm|wav|mp3|flac|m4a|aac|ogg|opus|aiff|aif|wma"
FILENAME_RE = re.compile(rf"\.({_EXT_ANY})(\s*\[\w+\])?$", re.IGNORECASE)
MEDIA_RE = re.compile(rf"\.({_EXT_MEDIA})(\s*\[\w+\])?$", re.IGNORECASE)
MEDIA_KEYS = ("image", "video", "audio", "file")
VIDEO_EXTS = {".mp4", ".avi", ".mov", ".mkv", ".webm"}


def media_reference(value) -> Optional[str]:
    """A media input's file name, without a trailing " [input]"-style annotation and with forward slashes."""
    if not isinstance(value, str):
        return None
    cleaned = re.sub(r"\s*\[\w+\]$", "", value).strip().replace("\\", "/")
    return cleaned if MEDIA_RE.search(cleaned) else None


def convert_paths(obj, sep: str):
    """Every string that looks like a file path, with `sep` as its separator; relative media paths and URLs keep
    their forward slashes."""
    if sep not in ("/", "\\"):
        return obj
    if isinstance(obj, str):
        if ("/" in obj or "\\" in obj) and FILENAME_RE.search(obj):
            s = obj.strip()
            drive = bool(re.match(r"^[A-Za-z]:(\\\\|/)", s))
            absolute = s.startswith("/") or s.startswith("\\\\")
            if re.match(r"^\w+://", s):
                return s
            if not drive and not absolute and MEDIA_RE.search(s):
                return re.sub(r"[\\]+", "/", s)
            return re.sub(r"[\\/]+", r"\\" if sep == "\\" else "/", s)
        return obj
    if isinstance(obj, list):
        return [convert_paths(v, sep) for v in obj]
    if isinstance(obj, dict):
        return {k: convert_paths(v, sep) for k, v in obj.items()}
    return obj


def media_references(prompt: dict) -> List[str]:
    refs = set()
    for node in prompt.values():
        if isinstance(node, dict):
            inputs = node.get("inputs", {})
            for key in MEDIA_KEYS:
                ref = media_reference(inputs.get(key))
                if ref:
                    refs.add(ref)
    return sorted(refs)


def read_media(filename: str):
    """-> (bytes, md5 hex, mime type) of an input file of this ComfyUI."""
    import folder_paths
    path = folder_paths.get_annotated_filepath(filename)
    if not os.path.exists(path):
        raise FileNotFoundError(filename)
    with open(path, "rb") as f:
        data = f.read()
    mime = mimetypes.guess_type(path)[0]
    if not mime:
        mime = "video/mp4" if os.path.splitext(path)[1].lower() in VIDEO_EXTS else "image/png"
    return data, hashlib.md5(data).hexdigest(), mime


# --------------------------------------------------------------------------------------
# URLs (utils/network.py)
# --------------------------------------------------------------------------------------
_HTTPS_SUFFIXES = (".proxy.runpod.net", ".ngrok-free.app", ".ngrok-free.dev", ".ngrok.io", ".trycloudflare.com",
                   ".cloudflare.dev")
_LOCAL_HOSTS = {"", "localhost", "127.0.0.1", "::1", "[::1]", "0.0.0.0"}


def _base(scheme: str, host: str, port: int) -> str:
    return f"{scheme}://{host}" + ("" if port == (443 if scheme == "https" else 80) else f":{port}")


def worker_url(worker: dict, endpoint: str = "", default_host: str = "127.0.0.1") -> str:
    host = (worker.get("host") or "").strip() or default_host
    port = int(worker.get("port", worker.get("listen_port", 8188)) or 8188)
    if host.startswith(("http://", "https://")):
        return host.rstrip("/") + endpoint
    cloud = worker.get("type") == "cloud" or host.endswith(".proxy.runpod.net") or port == 443
    return _base("https" if cloud else "http", host, port) + endpoint


def _split_host_port(host: str):
    if host.startswith("["):
        m = re.match(r"^(\[[^\]]+\])(?::(\d+))?$", host)
        return (m.group(1), int(m.group(2)) if m.group(2) else None) if m else (host, None)
    if host.count(":") == 1:
        h, p = host.rsplit(":", 1)
        if p.isdigit():
            return h, int(p)
    return host, None


def master_url(config: dict, address: str, port: int) -> str:
    """The URL workers reach this master at: the config's master host, else this server's address."""
    host = ((config or {}).get("master", {}) or {}).get("host") or ""
    host = host.strip()
    if host:
        if host.startswith(("http://", "https://")):
            return host.rstrip("/")
        host, explicit = _split_host_port(host)
        https_host = host.lower().endswith(_HTTPS_SUFFIXES)
        p = explicit if explicit is not None else int(port)
        scheme = "https" if https_host or p == 443 else "http"
        if explicit is None and scheme == "https" and https_host:
            p = 443
        return _base(scheme, host, p)
    if address in ("0.0.0.0", "::"):
        address = "127.0.0.1"
    return _base("https" if int(port) == 443 else "http", address, int(port))


def callback_url(worker: dict, config: dict, address: str, port: int) -> str:
    """A local worker calls back on 127.0.0.1; any other at master_url()."""
    wtype = str(worker.get("type") or "").strip().lower()
    host = worker.get("host")
    if isinstance(host, str):
        host = re.sub(r"^https?://", "", host.strip(), flags=re.IGNORECASE).split("/")[0] if host.strip() else ""
    if wtype == "local" or host in _LOCAL_HOSTS:
        return _base("https" if int(port) == 443 else "http", "127.0.0.1", int(port))
    return master_url(config, address, port)


# --------------------------------------------------------------------------------------
# the master's own prompt (utils/async_helpers.py:60-149)
# --------------------------------------------------------------------------------------
def _summary(node_errors) -> str:
    if not isinstance(node_errors, dict):
        return ""
    parts = []
    for nid, entry in node_errors.items():
        if not isinstance(entry, dict):
            continue
        ct = str(entry.get("class_type") or "UnknownNode")
        for err in entry.get("errors", []):
            if not isinstance(err, dict):
                continue
            details = str(err.get("details") or "").strip()
            parts.append(f"{ct}#{nid}: {str(err.get('message') or 'validation error')}"
                         + (f" ({details})" if details else ""))
            if len(parts) >= 5:
                return " | ".join(parts)
    return " | ".join(parts)


class PromptValidationError(RuntimeError):
    """ComfyUI refused the master's prompt; the message carries its error and node_errors as the reference's does."""

    def __init__(self, error, node_errors=None):
        self.validation_error = dict(error) if isinstance(error, dict) else {
            "type": "prompt_validation_failed", "message": str(error), "details": "", "extra_info": {}}
        self.node_errors = node_errors if isinstance(node_errors, dict) else {}
        if self.node_errors and not str(self.validation_error.get("details") or "").strip():
            summary = _summary(self.node_errors)
            if summary:
                self.validation_error["details"] = summary
        merged = dict(self.validation_error)
        if self.node_errors:
            merged["node_errors"] = self.node_errors
        super().__init__(f"Invalid prompt: {merged}")


async def queue_prompt(server, prompt: dict, workflow_meta, client_id, validate=None) -> dict:
    """Validate and queue a prompt on this ComfyUI, as its POST /prompt does -> {prompt_id, number, node_errors}.
    `server`: the PromptServer (trigger_on_prompt, number, prompt_queue); `validate`: execution.validate_prompt when
    None.  A refused prompt raises PromptValidationError."""
    if validate is None:
        import execution
        validate = execution.validate_prompt
    prompt = server.trigger_on_prompt({"prompt": prompt})["prompt"]
    prompt_id = str(uuid.uuid4())
    valid = await validate(prompt_id, prompt, None)
    if not valid[0]:
        raise PromptValidationError(valid[1] if len(valid) > 1 else "Prompt outputs failed validation",
                                    valid[3] if len(valid) > 3 else {})
    extra = {"create_time": int(time.time() * 1000)}
    if workflow_meta:
        extra["extra_pnginfo"] = {"workflow": workflow_meta}
    if client_id:
        extra["client_id"] = client_id
    sensitive = {}
    try:
        import execution
        keys = getattr(execution, "SENSITIVE_EXTRA_DATA_KEYS", [])
    except ImportError:
        keys = []
    for key in keys:
        if key in extra:
            sensitive[key] = extra.pop(key)
    number = getattr(server, "number", 0)
    server.number = number + 1
    server.prompt_queue.put((number, prompt_id, prompt, extra, valid[2], sensitive))
    return {"prompt_id": prompt_id, "number": number, "node_errors": {}}


# --------------------------------------------------------------------------------------
# the orchestration (api/queue_orchestration.py, api/orchestration/dispatch.py)
# --------------------------------------------------------------------------------------
_ws_warned = False


def _warn_websocket_once():
    global _ws_warned
    if not _ws_warned:
        _ws_warned = True
        warnings.warn("comfyui-distributed_b200: websocket_orchestration is set, but this package dispatches worker "
                      "prompts over HTTP (POST /prompt)", RuntimeWarning, stacklevel=3)


class Orchestrator:
    """The orchestration of one ComfyUI server.  `server`: its PromptServer (address, port, number, prompt_queue,
    trigger_on_prompt); `validate`: execution.validate_prompt; `store`: the collector store the queues go in."""

    def __init__(self, server, validate=None, store=None, config: Optional[Config] = None):
        from . import http_collector
        self.server, self.store = server, store if store is not None else http_collector.STORE
        self._validate = validate
        self.config = config if config is not None else Config()
        self.rr = 0                 # the round-robin position among idle load-balance candidates (dispatch.py:28)

    # ---- the network
    async def probe(self, session, worker: dict) -> Optional[dict]:
        """GET <worker>/prompt -> its JSON object, or None when it does not answer 200 with one in PROBE_TIMEOUT s."""
        import aiohttp
        url = self.url(worker).strip().rstrip("/")
        if not url:
            return None
        url = url if url.endswith("/prompt") else url + "/prompt"
        try:
            async with session.get(url, timeout=aiohttp.ClientTimeout(total=PROBE_TIMEOUT)) as resp:
                if resp.status != 200:
                    return None
                payload = await resp.json()
                return payload if isinstance(payload, dict) else None
        except Exception:
            return None

    async def dispatch(self, session, worker: dict, prompt: dict, workflow_meta):
        """POST <worker>/prompt; an error status raises (aiohttp.ClientResponseError)."""
        import aiohttp
        payload = {"prompt": prompt}
        if workflow_meta:
            payload["extra_data"] = {"extra_pnginfo": {"workflow": workflow_meta}}
        async with session.post(self.url(worker, "/prompt"), json=payload,
                                timeout=aiohttp.ClientTimeout(total=DISPATCH_TIMEOUT)) as resp:
            resp.raise_for_status()

    async def path_separator(self, session, worker: dict) -> Optional[str]:
        import aiohttp
        try:
            async with session.get(self.url(worker, "/distributed/system_info"),
                                   timeout=aiohttp.ClientTimeout(total=SYSTEM_INFO_TIMEOUT)) as resp:
                if resp.status != 200:
                    return None
                sep = (((await resp.json()) or {}).get("platform") or {}).get("path_separator")
                return sep if sep in ("/", "\\") else None
        except Exception:
            return None

    async def upload_media(self, session, worker: dict, filename: str, data: bytes, md5: str, mime: str):
        """-> (uploaded, the worker's name for the file): skipped when the worker has it with the same MD5."""
        import aiohttp
        name = filename.replace("\\", "/")
        try:
            async with session.post(self.url(worker, "/distributed/check_file"), json={"filename": name, "hash": md5},
                                    timeout=aiohttp.ClientTimeout(total=CHECK_FILE_TIMEOUT)) as resp:
                if resp.status == 200:
                    got = await resp.json()
                    if got.get("exists") and got.get("hash_matches"):
                        return False, name
        except Exception:
            pass
        parts = name.split("/")
        form = aiohttp.FormData()
        form.add_field("image", data, filename=parts[-1], content_type=mime)
        form.add_field("type", "input")
        form.add_field("subfolder", "/".join(parts[:-1]))
        form.add_field("overwrite", "true")
        async with session.post(self.url(worker, "/upload/image"), data=form,
                                timeout=aiohttp.ClientTimeout(total=UPLOAD_TIMEOUT)) as resp:
            resp.raise_for_status()
            try:
                got = await resp.json()
            except Exception:
                got = {}
        base = str((got or {}).get("name") or parts[-1]).strip()
        sub = str((got or {}).get("subfolder") or "").strip().replace("\\", "/").strip("/")
        return True, f"{sub}/{base}" if sub else base

    async def sync_media(self, session, worker: dict, prompt: dict):
        """Upload the prompt's media inputs the remote worker lacks and point the inputs at the worker's copies."""
        loop = asyncio.get_running_loop()
        renamed = {}
        for filename in media_references(prompt):
            try:
                data, md5, mime = await loop.run_in_executor(None, read_media, filename)
            except Exception:
                continue                            # missing here: the worker may have it
            try:
                _, there = await self.upload_media(session, worker, filename, data, md5, mime)
                if there:
                    renamed[filename] = there
            except Exception:
                continue
        for node in prompt.values():
            inputs = node.get("inputs", {}) if isinstance(node, dict) else None
            if not isinstance(inputs, dict):
                continue
            for key in MEDIA_KEYS:
                ref = media_reference(inputs.get(key))
                if ref and renamed.get(ref):
                    inputs[key] = renamed[ref]

    # ---- the steps
    def url(self, worker: dict, endpoint: str = "") -> str:
        return worker_url(worker, endpoint, getattr(self.server, "address", "127.0.0.1") or "127.0.0.1")

    def _port(self) -> int:
        return int(getattr(self.server, "port", 8188) or 8188)

    def job_prefix(self) -> str:
        return f"exec_{int(time.time() * 1000)}_{uuid.uuid4().hex[:6]}"

    async def select_active(self, session, workers, delegate_master, concurrency):
        """The workers that answer the probe; delegate-only is dropped when none does."""
        sem = asyncio.Semaphore(positive_int(concurrency, 8))

        async def one(w):
            async with sem:
                return w, await self.probe(session, w) is not None
        active = [w for w, ok in await asyncio.gather(*[one(w) for w in workers]) if ok]
        return active, (delegate_master and bool(active))

    async def least_busy(self, session, candidates, concurrency) -> Optional[dict]:
        """The idle candidates in turn, else the one with the shortest queue; None when no probe answers."""
        sem = asyncio.Semaphore(positive_int(concurrency, 8))

        async def one(w):
            async with sem:
                payload = await self.probe(session, w)
            if payload is None:
                return None
            try:
                remaining = int(payload.get("exec_info", {}).get("queue_remaining", 0))
            except (TypeError, ValueError, AttributeError):
                remaining = 0
            return w, max(remaining, 0)
        statuses = [s for s in await asyncio.gather(*[one(w) for w in candidates]) if s is not None]
        if not statuses:
            return None
        idle = [w for w, n in statuses if n == 0]
        if idle:
            chosen = idle[self.rr % len(idle)]
            self.rr += 1
            return chosen
        return min(statuses, key=lambda s: s[1])[0]

    def session(self):
        """The HTTP client of one request (aiohttp reads no proxy from the environment unless told to)."""
        import aiohttp
        return aiohttp.ClientSession(connector=aiohttp.TCPConnector(limit=100, limit_per_host=30))

    async def run(self, prompt: dict, workflow_meta, client_id, enabled_worker_ids=None, delegate_master=None):
        """The whole orchestration -> (prompt_id, number, workers dispatched, node_errors)."""
        async with self.session() as session:
            return await self._run(session, prompt, workflow_meta, client_id, enabled_worker_ids, delegate_master)

    async def _run(self, session, prompt, workflow_meta, client_id, enabled_worker_ids, delegate_master):
        config = self.config.load()
        settings = config.get("settings", {}) or {}
        if settings.get("websocket_orchestration", False):
            _warn_websocket_once()
        address, port = getattr(self.server, "address", "127.0.0.1") or "127.0.0.1", self._port()
        master = master_url(config, address, port)
        probe_n = positive_int(settings.get("worker_probe_concurrency"), PROBE_CONCURRENCY)
        prep_n = positive_int(settings.get("worker_prep_concurrency"), PREP_CONCURRENCY)
        media_n = positive_int(settings.get("media_sync_concurrency"), MEDIA_SYNC_CONCURRENCY)
        media_timeout = positive_float(settings.get("media_sync_timeout_seconds"), MEDIA_SYNC_TIMEOUT)
        workers = resolve_workers(config, enabled_worker_ids)
        index = PromptIndex(prompt)

        if delegate_master is None:
            delegate_master = bool(settings.get("master_delegate_only", False))
        if not workers:
            delegate_master = False
        active, delegate_master = await self.select_active(session, workers, delegate_master, probe_n)

        if load_balance_requested(index):
            candidates = list(active)
            if not delegate_master:         # the master competes only when it takes part
                candidates.append({"id": "master", "name": "Master", "host": master, "type": "local"})
            chosen = await self.least_busy(session, candidates, probe_n) if candidates else None
            if chosen is None and candidates:
                chosen = candidates[0]
            if chosen is None or str(chosen.get("id")) == "master":
                active, delegate_master = [], False
            else:
                active, delegate_master = [chosen], True

        enabled_ids = [w["id"] for w in active]
        jobs = job_id_map(index, self.job_prefix())
        if not jobs:
            queued = await queue_prompt(self.server, prompt, workflow_meta, client_id, self._validate)
            return queued["prompt_id"], queued["number"], 0, queued.get("node_errors", {})
        for job in jobs.values():
            await self.store.prepare(job)

        master_prompt = apply_overrides(index.copy(), "master", enabled_ids, jobs, master, delegate_master, index)
        if delegate_master:
            collectors = nodes_of_class(master_prompt, COLLECTOR)
            # a USDU prompt runs whole on the master, as the reference's does (its delegate mode lacks USDU)
            if collectors and not nodes_of_class(master_prompt, USDU):
                master_prompt = delegate_master_prompt(master_prompt, collectors)

        prep_sem, media_sem = asyncio.Semaphore(prep_n), asyncio.Semaphore(media_n)

        async def prepare(w):
            async with prep_sem:
                wp = index.copy()
                remote = bool(w.get("host")) and str(w.get("type") or "local").strip().lower() != "local"
                if remote:
                    sep = await self.path_separator(session, w)
                    if sep:
                        wp = convert_paths(wp, sep)
                wp = apply_overrides(prune_for_worker(wp), w["id"], enabled_ids, jobs,
                                     callback_url(w, config, address, port), delegate_master, index)
                if remote:
                    async with media_sem:
                        try:
                            await asyncio.wait_for(self.sync_media(session, w, wp), timeout=media_timeout)
                        except asyncio.TimeoutError:
                            pass            # dispatch anyway, as the reference does
                return w, wp
        prepared = await asyncio.gather(*[prepare(w) for w in active]) if active else []
        if prepared:
            await asyncio.gather(*[self.dispatch(session, w, wp, workflow_meta) for w, wp in prepared])
        queued = await queue_prompt(self.server, master_prompt, workflow_meta, client_id, self._validate)
        return queued["prompt_id"], queued["number"], len(prepared), queued.get("node_errors", {})


# --------------------------------------------------------------------------------------
# routes
# --------------------------------------------------------------------------------------
def _error(error, status):
    from aiohttp import web
    if isinstance(error, list):
        return web.json_response({"errors": [str(e) for e in error]}, status=status)
    return web.json_response({"error": str(error)}, status=status)


def make_handlers(orch: Orchestrator):
    """The two route handlers over `orch` -> {(method, path): handler}."""
    from aiohttp import web

    async def queue(request):
        try:
            raw = await request.json()
        except Exception as exc:
            return _error(f"Invalid JSON payload: {exc}", 400)
        try:
            req = parse_queue_request(raw)
        except ValueError as exc:
            return _error(exc, 400)
        try:
            prompt_id, number, count, node_errors = await orch.run(
                req.prompt, req.workflow_meta, req.client_id, enabled_worker_ids=req.enabled_worker_ids,
                delegate_master=req.delegate_master)
            return web.json_response({"prompt_id": prompt_id, "number": number, "node_errors": node_errors,
                                      "worker_count": count, "auto_prepare_supported": True})
        except Exception as exc:
            return _error(exc, 500)

    async def queue_status(request):
        try:
            job_id = request.match_info["job_id"]
            async with orch.store.lock:
                exists = job_id in orch.store.jobs
            return web.json_response({"exists": exists, "job_id": job_id})
        except Exception as exc:
            return _error(exc, 500)

    return {("POST", "/distributed/queue"): queue, ("GET", "/distributed/queue_status/{job_id}"): queue_status}


QUEUE_ROUTE = ("POST", "/distributed/queue")
_served: set = set()
_warned: set = set()


def register(routes, orch: Orchestrator, module_state: bool = True) -> set:
    """Add the handlers to an aiohttp RouteTableDef, skipping, with one warning each, every path another package
    already serves.  -> the (method, path) pairs served."""
    taken = {(getattr(r, "method", None), getattr(r, "path", None)) for r in routes}
    served = set()
    for (method, path), fn in make_handlers(orch).items():
        if (method, path) in taken:
            if (method, path) not in _warned:
                _warned.add((method, path))
                warnings.warn(f"comfyui-distributed_b200: {method} {path} is already served by another package; "
                              "this package's orchestrator stays off", RuntimeWarning, stacklevel=2)
            continue
        routes.route(method, path)(fn)
        served.add((method, path))
    if module_state:
        _served.update(served)
    return served


def install(server):
    """Register on ComfyUI's PromptServer once (http_master.install_in_comfyui)."""
    if not _served:
        register(server.routes, Orchestrator(server))


def serving() -> bool:
    """This process serves POST /distributed/queue."""
    return QUEUE_ROUTE in _served


def reset_for_tests():
    """Forget the registration (test harnesses that start and stop their own server)."""
    global _ws_warned
    _served.clear()
    _warned.clear()
    _ws_warned = False
