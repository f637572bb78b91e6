"""The collector master's job_complete image checks per frame, host path against device path (http_collector.py), for
1280x720, 1920x1080 and 3840x2160 RGB frames as this package's worker sends them (level-0 PNG, base64 data URL).

Reported per frame (median of --reps runs, each after one warm-up):
* host: png_of_payload -- b64decode(validate=True) and parse_png, all on the event loop;
* device: DeviceChecks.png_of_payload -- wall time from call to answer, and the part of it the event loop is held
  (the wall time minus the awaited device wait): ASCII encode, pinned copy, four launches, the table walk.
The JSON parse, which both paths share, is not included.

    python tools/collector_b64_times.py [--reps 5] [--out results/collector_b64_times.json]
"""
from __future__ import annotations

import argparse
import asyncio
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)

import torch  # noqa: E402

from collector_master_times import bodies, card  # noqa: E402
from __graft_entry__ import load_package  # noqa: E402

SIZES = [(720, 1280), (1080, 1920), (2160, 3840)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    load_package()
    from comfyui_distributed_b200 import http_collector as hc
    checks = hc.device_checks()
    assert checks is not None
    waited = [0.0]
    real = hc.device_wait

    async def timed_wait(ev):
        t = time.perf_counter()
        await real(ev)
        waited[0] += time.perf_counter() - t
    hc.device_wait = timed_wait
    rows = []
    for H, W in SIZES:
        x = (torch.rand((1, H, W, 3), generator=torch.Generator().manual_seed(H))).cuda()
        img = json.loads(bodies(x, {})[0])["image"]
        host, wall, held = [], [], []
        for r in range(a.reps + 1):
            t = time.perf_counter()
            png, info = hc.png_of_payload(img)
            host.append(time.perf_counter() - t)
            waited[0] = 0.0
            t = time.perf_counter()
            dpng, dinfo = asyncio.run(checks.png_of_payload(img))
            wall.append(time.perf_counter() - t)
            held.append(wall[-1] - waited[0])
            assert isinstance(dpng, hc.DevicePng) and dpng == png and dinfo.segs == info.segs
            del dpng
        med = lambda v: round(1e3 * statistics.median(v[1:]), 3)
        rows.append({"H": H, "W": W, "png_bytes": len(png), "text_bytes": len(img), "host_ms": med(host),
                     "device_wall_ms": med(wall), "device_loop_held_ms": med(held), "runs": a.reps})
        print(json.dumps(rows[-1]), flush=True)
    res = {"card": card(), "rows": rows}
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
