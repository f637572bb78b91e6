"""The static-mode master's cost per received worker tile at cfg2 geometry (7680x4320, 512 px tiles, padding 32, blur 8:
576x576 processing tiles, 135 of them), for this package's master (http_master.HttpStaticMaster) and for the reference's.

This package: host validation (`parse_png`, time.perf_counter), the pinned upload and the decode kernel (CUDA events on
the side stream, in drained batches of COMFYUI_MAX_BATCH = 20 tiles), and the final composite of all tiles with one blend
launch (CUDA events) divided by the tile count.  The reference: PIL's open().convert("RGB") of the tile and its
`blend_tile` onto the 8K canvas (time.perf_counter), from the staged reference bundle (oracle/_ref), on --ref-tiles
tiles.  The tiles are level-0 PIL PNGs of noise, what both workers send.  Each number is the median of --reps runs after
a warm-up run.

    python tools/master_tile_cost.py [--reps 5] [--ref-tiles 3] [--out results/master_tile_cost.json]
"""
from __future__ import annotations

import argparse
import io
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from __graft_entry__ import load_package  # noqa: E402

W, H, TILE, PAD, BLUR = 7680, 4320, 512, 32, 8
BATCH = 20


def card() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=60)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def tiles_png(plan, seed=0):
    from comfyui_distributed_b200.http_worker import encode_png
    rng = np.random.default_rng(seed)
    return [encode_png(rng.integers(0, 256, (t.ph, t.pw, 3), dtype=np.uint8)) for t in plan.tiles]


def ours(pngs, reps):
    load_package()
    from comfyui_distributed_b200 import http_master as hm
    from comfyui_distributed_b200.denoise import T0Denoiser
    from comfyui_distributed_b200.engine import WorkerJob
    img = torch.rand(1, H, W, 3, generator=torch.Generator().manual_seed(1))
    runs = []
    for rep in range(reps + 1):
        job = WorkerJob(img, T0Denoiser(1, 0.5), TILE, TILE, PAD, BLUR, True)
        m = hm.HttpStaticMaster(job, "cost", ["w1"], loop=object())      # no routes: the store is not touched
        t0 = time.perf_counter()
        entries = []
        for t, data in enumerate(pngs):
            entries.append((t, {"png": data, "info": hm.parse_png(data), "tile_idx": t, "batch_idx": 0,
                                "global_idx": t, "worker_id": "w1"}))
        t1 = time.perf_counter()
        for i in range(0, len(entries), BATCH):
            m._decode(entries[i: i + BATCH])
        t2 = time.perf_counter()
        m._composite(dict(entries))
        t3 = time.perf_counter()
        n = len(pngs)
        runs.append({"validate_ms": 1e3 * (t1 - t0) / n, "stage_enqueue_ms": 1e3 * (t2 - t1) / n,
                     "upload_ms": m.stats["upload_ms"] / n, "decode_ms": m.stats["decode_ms"] / n,
                     "blend_ms": m.stats["blend_ms"] / n, "composite_wall_ms": 1e3 * (t3 - t2) / n,
                     "bytes_per_tile": m.stats["bytes_received"] / n})
        del m, job
    runs = runs[1:]
    return {k: statistics.median(r[k] for r in runs) for k in runs[0]}


def reference(pngs, plan, n_tiles):
    import ref_static_run
    from PIL import Image
    env = ref_static_run._Env()
    try:
        node = env.node_cls()
        canvas = Image.fromarray(np.random.default_rng(2).integers(0, 256, (H, W, 3), dtype=np.uint8))
        dec, blend = [], []
        for t in plan.tiles[:n_tiles]:
            mask = node.create_tile_mask(W, H, t.x, t.y, TILE, TILE, BLUR)
            t0 = time.perf_counter()
            im = Image.open(io.BytesIO(pngs[t.idx])).convert("RGB")
            t1 = time.perf_counter()
            canvas = node.blend_tile(canvas, im, t.x1, t.y1, (t.ew, t.eh), mask, PAD)
            t2 = time.perf_counter()
            dec.append(t1 - t0)
            blend.append(t2 - t1)
        return {"decode_ms": 1e3 * statistics.median(dec), "blend_tile_ms": 1e3 * statistics.median(blend),
                "tiles": n_tiles}
    finally:
        env.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ref-tiles", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    load_package()
    from comfyui_distributed_b200.planner import get_plan
    plan = get_plan(W, H, TILE, TILE, PAD, BLUR, True)
    pngs = tiles_png(plan)
    res = {"card": card(), "geometry": f"{W}x{H} tile {TILE} pad {PAD} blur {BLUR}", "tiles": len(plan.tiles),
           "ours_per_tile": ours(pngs, a.reps)}
    o = res["ours_per_tile"]
    o["total_ms"] = o["validate_ms"] + o["upload_ms"] + o["decode_ms"] + o["blend_ms"]
    try:
        res["reference_per_tile"] = reference(pngs, plan, a.ref_tiles)
    except Exception as e:      # noqa: BLE001 -- the bundle is optional for the device numbers
        res["reference_per_tile"] = {"error": repr(e)}
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
