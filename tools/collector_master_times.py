"""Per-image cost of DistributedCollector as the master of HTTP workers (http_collector.py), for 1280x720 x 81,
1920x1080 x 9 and 3840x2160 x 1 RGB frames per worker.  Workers are this package's (usdu_png_base64_u8 on the GPU,
http_worker.send_collector_batch) and post on 127.0.0.1 in this process.

Reported per image:
* the job_complete handler's host time, split into JSON parse, base64 decode, parse_png and the audio envelope
  (a 1 s stereo 48 kHz envelope, which rides on the last image only; its time is shown per envelope);
* upload and decode of each frame as it arrives (CUDA events in GpuFrames, one decode launch per frame);
* the final usdu_gather_unpack_f32 into pinned host memory as achieved GB/s of fp32 written, against
  usdu_unpack_tiles_f32 into device memory plus a cudaMemcpy to pinned memory of the same bytes (CUDA events);
* a worker's POST round trip against this master and against the reference's master (tests/collector_master.Master).

    python tools/collector_master_times.py [--reps 3] [--out results/collector_master_times.json]
"""
from __future__ import annotations

import argparse
import base64
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import torch  # noqa: E402

import collector_master  # noqa: E402
from __graft_entry__ import load_package  # noqa: E402

CASES = [(81, 720, 1280), (9, 1080, 1920), (1, 2160, 3840)]
JOB = "times"


def card() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=60)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def bodies(x_dev: torch.Tensor, audio_env: dict):
    """The job_complete bodies this package's worker sends for x_dev (the last one with the audio envelope)."""
    load_package()
    from comfyui_distributed_b200.nodes.collector import _native_pack, _native_png_b64
    B = x_dev.shape[0]
    out = []
    for i, text in enumerate(_native_png_b64(_native_pack(x_dev))):
        d = {"job_id": JOB, "worker_id": "w1", "batch_idx": i, "image": "data:image/png;base64," + bytes(text).decode(),
             "is_last": i == B - 1}
        if i == B - 1:
            d["audio"] = audio_env
        out.append(json.dumps(d).encode())
    return out


def handler_times(raws, reps: int) -> dict:
    """The handler's host steps, in its order, best of `reps` per image."""
    from comfyui_distributed_b200 import http_collector as hc
    from comfyui_distributed_b200.http_master import parse_png
    best = {}
    for _ in range(reps):
        t = {"json_s": 0.0, "base64_s": 0.0, "parse_png_s": 0.0, "audio_s": 0.0}
        for raw in raws:
            t0 = time.perf_counter()
            d = json.loads(raw)
            hc.field_errors(d)
            t1 = time.perf_counter()
            png = base64.b64decode(d["image"].partition(",")[2], validate=True)
            t2 = time.perf_counter()
            parse_png(png)
            t3 = time.perf_counter()
            if d.get("audio") is not None:
                hc.audio_of_payload(d["audio"])
            t4 = time.perf_counter()
            t["json_s"] += t1 - t0
            t["base64_s"] += t2 - t1
            t["parse_png_s"] += t3 - t2
            t["audio_s"] += t4 - t3
        for k, v in t.items():
            best[k] = min(best.get(k, v), v)
    n = len(raws)
    return {"json_s_per_image": best["json_s"] / n, "base64_s_per_image": best["base64_s"] / n,
            "parse_png_s_per_image": best["parse_png_s"] / n, "audio_s_per_envelope": best["audio_s"]}


def decode_and_gather(raws, B, H, W, reps: int) -> dict:
    """Decode each frame as it arrives (GpuFrames.add per image), then the gather into pinned memory, against unpack
    plus cudaMemcpy of the same bytes."""
    from comfyui_distributed_b200 import _native as nat
    from comfyui_distributed_b200 import http_collector as hc
    items = []
    for raw in raws:
        d = json.loads(raw)
        png, info = hc.png_of_payload(d["image"])
        items.append({"png": png, "info": info})
    frames = hc.GpuFrames(torch.device("cuda", torch.cuda.current_device()))
    for it in items:
        frames.add([it])
    torch.cuda.synchronize()
    up, dec = frames.decoder.times()
    e = H * W * 3
    out = torch.empty((B, H, W, 3), dtype=torch.float32, pin_memory=True)
    dev = torch.empty((B, e), dtype=torch.float32, device="cuda")
    ptrs = torch.tensor([b.data_ptr() + o for b, o in (it["frame"] for it in items)], dtype=torch.int64).cuda()
    packed = torch.empty((B, e), dtype=torch.uint8, device="cuda")
    for i, (b, o) in enumerate(it["frame"] for it in items):
        packed[i].copy_(b[o: o + e])
    s = torch.cuda.current_stream()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    g_best, u_best = None, None
    for _ in range(reps + 1):                                 # the first round warms up
        ev[0].record()
        nat.gather_unpack_f32(ptrs.data_ptr(), B, e, out.data_ptr(), s.cuda_stream)
        ev[1].record()
        nat.unpack_tiles_f32(packed.data_ptr(), dev.data_ptr(), B * e, s.cuda_stream)
        out.view(B, e).copy_(dev, non_blocking=True)
        ev[2].record()
        torch.cuda.synchronize()
        g, u = ev[0].elapsed_time(ev[1]) / 1e3, ev[1].elapsed_time(ev[2]) / 1e3
        g_best = g if g_best is None else min(g_best, g)
        u_best = u if u_best is None else min(u_best, u)
    frames.decoder.release()
    nbytes = B * e * 4
    return {"upload_s_per_image": up / 1e3 / B, "decode_s_per_image": dec / 1e3 / B,
            "gather_unpack_s_per_image": g_best / B, "gather_unpack_GBps": nbytes / g_best / 1e9,
            "unpack_memcpy_s_per_image": u_best / B, "unpack_memcpy_GBps": nbytes / u_best / 1e9,
            "png_bytes": len(items[0]["png"])}


def round_trips(x_dev, x_cpu, reps: int) -> dict:
    """This package's worker posting to this package's master node, and to the reference's master."""
    from comfyui_distributed_b200.nodes import collector
    from test_http_collector import Ours
    B = x_dev.shape[0]
    out = {}
    with Ours() as ours:
        for rep in range(reps + 1):
            res, posts = {}, []
            node = collector.DistributedCollectorNode()
            t = threading.Thread(target=lambda: res.update(r=node.run(x_cpu[:1], multi_job_id=f"{JOB}{rep}",
                                                                      enabled_worker_ids='["w1"]')))
            t.start()
            collector.send_to_master(x_dev, None, f"{JOB}{rep}", ours.url, "w1", post_times=posts)
            t.join(600)
            assert res["r"][0].shape[0] == 1 + B
            if rep:
                out.setdefault("ours_post_s_per_image", []).append(sum(posts) / B)
                out.setdefault("assembly_s_per_image", []).append(node.last_stats["assembly_ms"] / 1e3 / B)
    with collector_master.Master(keep_bodies=False) as m:
        for rep in range(reps + 1):
            fut = m.collect(x_cpu[:1], f"ref{rep}", ["w1"])
            posts = []
            collector.send_to_master(x_dev, None, f"ref{rep}", m.url, "w1", post_times=posts)
            assert fut.result(600)[0].shape[0] == 1 + B
            if rep:
                out.setdefault("ref_post_s_per_image", []).append(sum(posts) / B)
    return {k: min(v) for k, v in out.items()}


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    load_package()
    rows = {"card": card(), "cases": []}
    print("card:", rows["card"])
    wave = torch.rand(1, 2, 48000, generator=torch.Generator().manual_seed(0))
    audio_env = {"sample_rate": 48000, "shape": [1, 2, 48000], "dtype": "float32",
                 "data": base64.b64encode(wave.numpy().tobytes()).decode()}
    for B, H, W in CASES:
        g = torch.Generator().manual_seed(B * 7 + H)
        x_cpu = torch.rand((B, H, W, 3), generator=g)
        x_dev = x_cpu.cuda()
        raws = bodies(x_dev, audio_env)
        row = {"B": B, "H": H, "W": W, "body_bytes": len(raws[0])}
        row.update(handler_times(raws, a.reps))
        row.update(decode_and_gather(raws, B, H, W, a.reps))
        row.update(round_trips(x_dev, x_cpu, a.reps))
        rows["cases"].append(row)
        print(json.dumps(row))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
