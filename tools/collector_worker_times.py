"""Per-image time of DistributedCollector as an HTTP worker of the reference's master, for 1024x1024 x 1 and
1280x720 x 81 RGB frames: this package's worker (cast + stored-PNG + base64 on the GPU, usdu_png_base64_u8) against the
reference's worker (send_batch_to_master: tensor_to_pil, PIL PNG at level 0, base64, one POST per image), both posting
to the reference's job_complete route and collector master (tests/collector_master.Master) on 127.0.0.1 in this process.

Reported per image: pack + encode (CUDA events around the three passes and the cast, with the bytes the passes move
over that time), the D2H copy of the text (CUDA events), the POST (host clock), and the whole send for both workers.

    python tools/collector_worker_times.py [--reps 3] [--out results/collector_worker_times.json]
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

import collector_master  # noqa: E402
from __graft_entry__ import load_package  # noqa: E402

CASES = [(1, 1024, 1024), (81, 720, 1280)]


def card() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=60)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def device_times(x: torch.Tensor, reps: int) -> dict:
    """Events around the cast and the three passes over the whole batch, and around the D2H copy of its text."""
    load_package()
    from comfyui_distributed_b200 import _native as nat
    from comfyui_distributed_b200.nodes.collector import _native_pack
    B, H, W, C = x.shape
    png_len, text_len, staging_len = nat.png_sizes(H, W, C)
    staging = torch.empty(B * staging_len, dtype=torch.uint8, device="cuda")
    text = torch.empty(B * text_len, dtype=torch.uint8, device="cuda")
    host = torch.empty(B * text_len, dtype=torch.uint8, pin_memory=True)
    stream = torch.cuda.current_stream()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    best = None
    for _ in range(reps + 1):                                 # the first round warms up
        ev[0].record()
        q = _native_pack(x)
        ev[1].record()
        nat.png_base64_u8(q.data_ptr(), B, H, W, C, staging.data_ptr(), text.data_ptr(), stream.cuda_stream)
        ev[2].record()
        host.copy_(text, non_blocking=True)
        ev[3].record()
        torch.cuda.synchronize()
        t = [ev[i].elapsed_time(ev[i + 1]) / 1e3 for i in range(3)]
        best = t if best is None or sum(t) < sum(best) else best
    pack_s, enc_s, d2h_s = best
    raw = H * (1 + W * C)
    # pass A reads the frame and writes the chunks, pass C reads the PNG and writes the text; the cast reads fp32 and
    # writes u8 (pass B's few bytes per frame are left out)
    enc_bytes = B * (H * W * C + png_len + png_len + text_len)
    pack_bytes = B * H * W * C * 5
    return {"pack_s_per_image": pack_s / B, "encode_s_per_image": enc_s / B, "d2h_s_per_image": d2h_s / B,
            "encode_GBps": enc_bytes / enc_s / 1e9, "pack_GBps": pack_bytes / pack_s / 1e9,
            "png_bytes": png_len, "text_bytes": text_len, "raw_bytes": raw}


def send_times(x_dev: torch.Tensor, x_cpu: torch.Tensor, reps: int) -> dict:
    load_package()
    from comfyui_distributed_b200.nodes import collector
    B = x_dev.shape[0]
    out = {}
    with collector_master.Master(keep_bodies=False) as m:
        for rep in range(reps + 1):
            job = f"ours{rep}"
            fut = m.collect(x_cpu[:1], job, ["w1"])
            posts = []
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            collector.send_to_master(x_dev, None, job, m.url, "w1", post_times=posts)
            ours = time.perf_counter() - t0
            res = fut.result(600)
            assert res[0].shape[0] == 1 + B
            if rep:
                out.setdefault("ours_send_s_per_image", []).append(ours / B)
                out.setdefault("post_s_per_image", []).append(sum(posts) / B)
        node = m.collector.DistributedCollectorNode()
        for rep in range(reps):
            job = f"ref{rep}"
            fut = m.collect(x_cpu[:1], job, ["w1"])
            t0 = time.perf_counter()
            m._call(node.send_batch_to_master(x_cpu, None, job, m.url, "w1"), timeout=1200)
            ref = time.perf_counter() - t0
            res = fut.result(600)
            out.setdefault("ref_send_s_per_image", []).append(ref / B)
    return {k: min(v) for k, v in out.items()}


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    rows = {"card": card(), "cases": []}
    print("card:", rows["card"])
    for B, H, W in CASES:
        g = torch.Generator().manual_seed(B * 7 + H)
        x_cpu = torch.rand((B, H, W, 3), generator=g)
        x_dev = x_cpu.cuda()
        row = {"B": B, "H": H, "W": W}
        row.update(device_times(x_dev, a.reps))
        row.update(send_times(x_dev, x_cpu, a.reps))
        rows["cases"].append(row)
        print(json.dumps(row))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
