"""The baseline JPEG path per frame (http_master.parse_jpeg, usdu_jpeg_decode_u8) beside PIL:

* entropy: host time of parse_jpeg (marker parse and Huffman decode into int16 coefficients), median of --reps;
* kernel: device time of one usdu_jpeg_decode_u8 launch for the frame (CUDA events), median of --reps;
* pil: host time of PIL's Image.open(...).convert("RGB") on the same bytes, median of --reps;
* the card name and power limit, read in the same run.

Frames are 720p, 1080p and 4K pictures (gradients, edges and noise) written by Pillow at quality 75 and 95, in 4:2:0
and 4:4:4.

    python tools/jpeg_times.py [--reps 5] [--out results/jpeg_times.json]
"""
from __future__ import annotations

import argparse
import io
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402
from PIL import Image  # noqa: E402

from collector_master_times import card  # noqa: E402
from __graft_entry__ import load_package  # noqa: E402

SIZES = {"720p": (1280, 720), "1080p": (1920, 1080), "4k": (3840, 2160)}


def picture(W, H):
    rng = np.random.default_rng(W)
    y, x = np.mgrid[:H, :W]
    a = np.stack([x * 255 // (W - 1), y * 255 // (H - 1), ((x // 5 + y // 3) * 37) % 256], 2)
    return (a + rng.integers(-20, 21, a.shape)).clip(0, 255).astype(np.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    load_package()
    from comfyui_distributed_b200 import http_master as hm
    dev = torch.device("cuda")
    rows = {}
    for size, (W, H) in SIZES.items():
        img = Image.fromarray(picture(W, H))
        dst = torch.empty(H * W * 3, dtype=torch.uint8, device=dev)
        for q in (75, 95):
            for sub, tag in ((2, "420"), (0, "444")):
                b = io.BytesIO()
                img.save(b, "JPEG", quality=q, subsampling=sub)
                data = b.getvalue()
                entropy, kernel, pil = [], [], []
                for i in range(a.reps + 1):
                    t0 = time.perf_counter()
                    info = hm.parse_jpeg(data)
                    t1 = time.perf_counter()
                    ref = np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))
                    t2 = time.perf_counter()
                    dec = hm.PngDecoder(dev)
                    dec.decode_jpeg([(info, 0)], dst)
                    torch.cuda.synchronize()
                    if i:                             # the first run warms up
                        entropy.append((t1 - t0) * 1e3)
                        pil.append((t2 - t1) * 1e3)
                        kernel.append(dec.times()[1])
                    dec.release()
                assert np.array_equal(dst.cpu().numpy().reshape(H, W, 3), ref), (size, q, tag)
                name = f"{size}_q{q}_{tag}"
                rows[name] = {"jpeg_bytes": len(data), "entropy_ms": round(statistics.median(entropy), 2),
                              "kernel_ms": round(statistics.median(kernel), 3), "pil_ms": round(statistics.median(pil), 2)}
                r = rows[name]
                print(f"{name:16s} {len(data) / 1e6:6.2f} MB  entropy {r['entropy_ms']:7.2f} ms  kernel "
                      f"{r['kernel_ms']:7.3f} ms  PIL {r['pil_ms']:7.2f} ms", flush=True)
    out = {"card": card(), "reps": a.reps, "frames": rows}
    print(json.dumps(out))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
