"""Isolated launches of the two tile kernels on machine-filling work lists, per kernel path (tensor-core / integer-pipe):
CUDA events around each launch, inputs larger than L2 between launches (the 398 MB fp32 tile buffer is re-read).
  python tools/kernel_bench.py [workload]      -> one JSON line per (kernel, path)
What it launches: crop of ALL tiles of the canvas in one launch; blend of ALL tiles in one launch (the static-mode final
composite: every canvas block, ordered tile chains) from fp32 and from u8 sources; and one 8-tile wave of each."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from __graft_entry__ import load_package

load_package()
from comfyui_distributed_b200 import engine, planner

W = {"cfg2": (1, 4320, 7680, 512, 32, 8), "cfg4": (1, 8640, 15360, 256, 32, 8), "cfg5": (17, 2160, 3840, 512, 32, 8)}
name = sys.argv[1] if len(sys.argv) > 1 else "cfg2"
B, H, Wd, tile, pad, blur = W[name]
peak = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.isfile(
    os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")) else 3350.0   # H100 SXM data sheet
plan = planner.get_plan(Wd, H, tile, tile, pad, blur, True)
dev = torch.device("cuda", 0)
img = torch.rand(B, H, Wd, 3, device=dev)
ids = list(range(len(plan.tiles)))
wave = max(plan.waves(), key=len)


def timed(fn, reps=10):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    ts.sort()
    return ts[len(ts) // 2], ts[0]


for path_name, no_mma in (("mma", False), ("fast", True)):
    engine.FORCE_NO_MMA = no_mma
    dp = engine.DevicePlan.get(plan, dev)
    canvas = engine.Canvas(dp, B).load(img)
    for what, tiles in (("all tiles", ids), (f"{len(wave)}-tile wave", wave)):
        buf, offs = canvas.crop(tiles)
        wl = dp.crop_list(tuple(tiles), B, canvas.path_crop)[0]
        med, best = timed(lambda: canvas.crop(tiles, out=buf))
        nb = wl.algo_bytes * B
        print(json.dumps({"kernel": "crop_resize", "path": path_name, "launch": what, "grid": int(wl.items.shape[0]) * B, "us": round(med, 2),
                          "us_best": round(best, 2), "algo_MB": round(nb / 1e6, 1), "GBps": round(nb / med / 1e3, 1), "frac_of_hbm_peak": round(nb / med / 1e3 / peak, 3)}))
        src_f = torch.rand(buf.numel(), device=dev)
        src_u = (src_f * 255).to(torch.uint8)
        for sname, src in (("fp32", src_f), ("u8", src_u)):
            o = offs if sname == "fp32" else offs          # same element offsets: u8 buffer is indexed in elements too
            bl = dp.blend_list(tuple(tiles), o, sname == "u8", canvas.path_blend, B)[0]
            med, best = timed(lambda: canvas.blend(tiles, src, o))
            nb = bl.algo_bytes * B
            print(json.dumps({"kernel": "blend", "src": sname, "path": path_name, "launch": what, "grid": int(bl.n_launch) * B, "block_rows": bl.block_rows,
                              "us": round(med, 2), "us_best": round(best, 2), "algo_MB": round(nb / 1e6, 1), "GBps": round(nb / med / 1e3, 1),
                              "frac_of_hbm_peak": round(nb / med / 1e3 / peak, 3)}))
    del canvas
