"""The reference's collector master, run for real in this process -- TEST INFRASTRUCTURE ONLY.

`Master` serves the reference's job_complete route (api/job_routes.py:273-343) on an in-process aiohttp app on 127.0.0.1
and runs `DistributedCollectorNode.execute(is_worker=False)` (nodes/collector.py) on the same event loop, so that HTTP
workers -- the reference's own or this package's -- can post to it.  The reference's modules come from
oracle/ref_collector.py's loader: from /root/reference where it exists, else from the bundle oracle/make_ref.py staged
(make_ref.staged_root()), as oracle/ref_static_run.py does.
"""
from __future__ import annotations

import asyncio
import json
import os
import socket
import sys
import threading
from typing import Sequence

import torch

import make_ref
import ref_collector
from ref_collector import PKG


def available() -> bool:
    return ref_collector.available() or bool(make_ref.staged_root())


def load():
    """ref_collector.load(), from the staged bundle when the reference tree is absent.  ref_collector's root is only
    pointed at the bundle for the load itself: its modules stay cached, and its own availability check is unchanged."""
    if ref_collector._loaded is None and not ref_collector.available():
        root = make_ref.staged_root()
        if root:
            saved = ref_collector.REF_ROOT
            ref_collector.REF_ROOT = root
            try:
                return ref_collector.load()
            finally:
                ref_collector.REF_ROOT = saved
    return ref_collector.load()


class Master:
    """The reference's collector master on 127.0.0.1: `url` takes job_complete POSTs; `collect(...)` runs
    DistributedCollectorNode.execute as the master (is_worker=False) in the server's loop and returns a future of its
    (combined images, combined audio).  `worker_timeout`: seconds the master waits without a POST before it gives up
    on the workers still missing (the reference's unified worker timeout).  `keep_bodies`: keep every accepted POST
    body in `received`."""

    def __init__(self, worker_timeout: float = 60.0, keep_bodies: bool = True):
        from aiohttp import web
        collector, routes, _ = load()
        self.collector, self.routes = collector, routes
        self.received = []                                   # every POST body the route accepted, in arrival order
        self.loop = asyncio.new_event_loop()
        self.thread = threading.Thread(target=self._run, daemon=True)
        self.thread.start()
        inst = collector.prompt_server
        # stand-ins for what ComfyUI's PromptServer holds; the route and the master share them
        inst.distributed_pending_jobs = {}
        self._lock_ready = threading.Event()
        self.loop.call_soon_threadsafe(self._make_lock, inst)
        self._lock_ready.wait(10)
        cfg = sys.modules[f"{PKG}.utils.config"]
        cfg.CONFIG_FILE = os.path.join("/nonexistent", "gpu_config.json")   # defaults; never the reference's tree
        collector.get_worker_timeout_seconds = lambda: max(1, int(worker_timeout))
        handler = next(r.handler for r in inst.routes if getattr(r, "path", "") == "/distributed/job_complete")

        async def job_complete(request):
            body = await request.read()
            response = await handler(request)
            if response.status < 400 and keep_bodies:
                self.received.append(body)
            return response

        app = web.Application(client_max_size=1 << 30)
        app.router.add_post("/distributed/job_complete", job_complete)
        self.runner = web.AppRunner(app)
        self._call(self.runner.setup())
        s = socket.socket()
        s.bind(("127.0.0.1", 0))
        self.port = s.getsockname()[1]
        s.close()
        self._call(web.TCPSite(self.runner, "127.0.0.1", self.port).start())
        self.url = f"http://127.0.0.1:{self.port}"

    def _make_lock(self, inst):
        inst.distributed_jobs_lock = asyncio.Lock()
        self._lock_ready.set()

    def _run(self):
        asyncio.set_event_loop(self.loop)
        self.loop.run_forever()

    def _call(self, coro, timeout=60):
        return asyncio.run_coroutine_threadsafe(coro, self.loop).result(timeout)

    def collect(self, images: torch.Tensor, job_id: str, enabled_worker_ids: Sequence[str], audio=None,
                delegate_only: bool = False):
        node = self.collector.DistributedCollectorNode()
        coro = node.execute(images, audio, False, job_id, False, "", json.dumps(list(enabled_worker_ids)), 1, "",
                            bool(delegate_only))
        return asyncio.run_coroutine_threadsafe(coro, self.loop)

    def worker_send(self, images: torch.Tensor, audio, job_id: str, worker_id: str):
        """The reference's worker side (send_batch_to_master, collector.py:84-119), blocking until it has posted."""
        node = self.collector.DistributedCollectorNode()
        self._call(node.send_batch_to_master(images, audio, job_id, self.url, worker_id), timeout=300)

    def close(self):
        try:
            net = sys.modules.get(f"{PKG}.utils.network")
            if net is not None and hasattr(net, "cleanup_client_session"):
                self._call(net.cleanup_client_session())
            self._call(self.runner.cleanup())
        finally:
            self.loop.call_soon_threadsafe(self.loop.stop)
            self.thread.join(timeout=10)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
