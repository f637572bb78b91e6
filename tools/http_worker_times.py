"""Per-tile time of a static-mode HTTP worker on cfg2 (7680x4320, 512 px tiles, padding 32, T0 sampler), split into
its phases, for this package's worker (engine.WorkerJob + http_worker.HttpStaticWorker) and for the reference's worker,
all posting to the reference's master routes on 127.0.0.1 in this process.  This package's worker runs twice over the
same tiles: once with the PNGs encoded on the GPU (WorkerJob.step_png, the node's worker role) and once PIL-encoded on
the host (WorkerJob.step + http_worker.encode_png), so both encodes are timed on one card in one run.

The master here only serves the queue: the job is created through the reference's own `init_static_job_batched` and
nobody else pulls, so each worker gets every tile the queue holds.  The reference's worker takes seconds per tile at 8K
on the CPU, so it is given the first --ref-tiles tiles of the grid (its masks are built for those only; the per-tile work
does not depend on how many there are).

    python tools/http_worker_times.py [--ref-tiles 3] [--out results/http_worker_times.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import torch  # noqa: E402

import ref_static_run  # noqa: E402
from __graft_entry__ import load_package  # noqa: E402
from inputs import make_input  # noqa: E402

W, H, TILE, PAD, BLUR = 7680, 4320, 512, 32, 8
SEED, DENOISE = 11, 0.5


def card() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=60)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def start_job(env, job_id: str, n_tiles: int):
    env._call(env.mods["upscale.job_store"].init_static_job_batched(job_id, 1, n_tiles, [job_id]))


def gpu_worker(env, url: str, img, encode: str) -> dict:
    """encode = "gpu": the node's worker role (WorkerJob.step_png); "pil": WorkerJob.step, PNGs from PIL on the host."""
    load_package()
    from comfyui_distributed_b200.denoise import T0Denoiser
    from comfyui_distributed_b200.engine import WorkerJob
    from comfyui_distributed_b200.http_worker import HttpStaticWorker

    x = torch.from_numpy(img)
    warm = WorkerJob(x, T0Denoiser(SEED, DENOISE), TILE, TILE, PAD, BLUR, True)   # module loads, noise, work lists
    for t in range(len(warm.plan.tiles)):
        warm.step_png(t) if encode == "gpu" else warm.step(t)                    # and the PNG layout check
    del warm
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    job = WorkerJob(x, T0Denoiser(SEED, DENOISE), TILE, TILE, PAD, BLUR, True)
    setup = time.perf_counter() - t0
    n = len(job.plan.tiles)
    job_id = "gpu-" + encode
    start_job(env, job_id, n)
    w = HttpStaticWorker(url, job_id, job_id, PAD, [(t.x1, t.y1, t.ew, t.eh) for t in job.plan.tiles], 1)
    t0 = time.perf_counter()
    assert w.run(job.step_png if encode == "gpu" else job.step)
    wall = time.perf_counter() - t0
    assert sorted(w.pulled) == list(range(n)), "the GPU worker did not get every tile"
    ms = lambda s: round(1e3 * s / n, 3)   # noqa: E731
    return {"tiles": n, "setup_ms": round(1e3 * setup, 1), "per_tile_ms": {
        "device_step": round(job.times["device_ms"] / n, 3), "gpu_png_encode": round(job.times["encode_ms"] / n, 3),
        "d2h": round(job.times["d2h_ms"] / n, 3), "step_host_wall": ms(w.times["step_s"]),
        "pil_png_encode": ms(w.times["encode_s"]), "post": ms(w.times["post_s"]),
        "heartbeat": ms(w.times["heartbeat_s"]), "tile_request": ms(w.times["request_s"]), "total_wall": ms(wall)},
        "uploads": w.chunks}


def ref_worker(env, url: str, img, n_tiles: int) -> dict:
    from PIL import Image

    acc = {k: 0.0 for k in ("canvas_to_fp32", "crop", "sampler", "blend", "png_encode", "send", "heartbeat", "tile_request")}

    def timed(fn, key):
        def f(*a, **k):
            t = time.perf_counter()
            try:
                return fn(*a, **k)
            finally:
                acc[key] += time.perf_counter() - t
        return f

    def timed_async(fn, key):
        async def f(*a, **k):
            t = time.perf_counter()
            try:
                return await fn(*a, **k)
            finally:
                acc[key] += time.perf_counter() - t
        return f

    node = env.node_cls()
    full = node.calculate_tiles
    node.calculate_tiles = lambda *a, **k: full(*a, **k)[:n_tiles]
    node.extract_batch_tile_with_padding = timed(node.extract_batch_tile_with_padding, "crop")
    node.process_tiles_batch = timed(node.process_tiles_batch, "sampler")
    node.blend_tile = timed(node.blend_tile, "blend")
    node.send_tiles_batch_to_master = timed_async(node.send_tiles_batch_to_master, "send")
    node._send_heartbeat_to_master = timed_async(node._send_heartbeat_to_master, "heartbeat")
    node._request_tile_from_master = timed_async(node._request_tile_from_master, "tile_request")
    static = env.mods["upscale.modes.static"]
    saved = static.pil_to_tensor, Image.Image.save
    static.pil_to_tensor = timed(static.pil_to_tensor, "canvas_to_fp32")
    Image.Image.save = timed(Image.Image.save, "png_encode")      # only the worker's tile PNGs are saved in this process
    start_job(env, "ref", n_tiles)
    cond = [[torch.zeros(1, 77, 8), {}]]
    try:
        t0 = time.perf_counter()
        node.run(torch.from_numpy(img), None, cond, cond, None, SEED, 20, 8.0, "euler", "normal", DENOISE, TILE, TILE,
                 PAD, BLUR, True, False, multi_job_id="ref", is_worker=True, master_url=url, worker_id="ref",
                 enabled_worker_ids='["ref"]')
        wall = time.perf_counter() - t0
    finally:
        static.pil_to_tensor, Image.Image.save = saved
    per = {k: round(1e3 * v / n_tiles, 1) for k, v in acc.items()}
    per["post"] = round(per.pop("send") - per["png_encode"], 1)
    return {"tiles": n_tiles, "per_tile_ms": per, "total_wall_ms_incl_setup": round(1e3 * wall, 1)}


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--ref-tiles", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("http_worker_times: needs a CUDA device")
    if not ref_static_run.available():
        raise SystemExit("http_worker_times: reference bundle (oracle/_ref) not present: run build() first")
    img = make_input("noise", 3, 1, H, W)
    env = ref_static_run._Env()
    try:
        env.sampler = ref_static_run.torch_t0
        url = f"http://127.0.0.1:{env.port}"
        res = {"card": card(), "cfg": f"{W}x{H} tile {TILE} padding {PAD} mask_blur {BLUR}, B=1, T0 sampler",
               "gpu_worker_gpu_png": gpu_worker(env, url, img, "gpu"), "gpu_worker_pil_png": gpu_worker(env, url, img, "pil"),
               "reference_worker": ref_worker(env, url, img, args.ref_tiles)}
    finally:
        env.close()
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
