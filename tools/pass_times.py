"""Eager quantise / dequantise passes of the bench workload (cfg2, 7680x4320), each alone: CUDA events around every
launch, median of many, with the achieved rate of the bytes the pass has to move (fp32 image + u8 canvas)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from __graft_entry__ import load_package
load_package()
from comfyui_distributed_b200 import engine, planner

B, H, W = 1, 4320, 7680
REPS = 50
img = torch.rand(B, H, W, 3, device="cuda")
plan = planner.get_plan(W, H, 512, 512, 32, 8, True)
cv = engine.Canvas(engine.DevicePlan.get(plan, img.device), B)
out = torch.empty_like(img)


def median_us(fn):
    for _ in range(5):
        fn()
    ts = []
    for _ in range(REPS):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    ts.sort()
    return ts[len(ts) // 2], ts[0], ts[-1]


nbytes = B * H * W * 3 * 5                  # 4 bytes of fp32 + 1 byte of u8 per channel value
for name, fn in (("quantize", lambda: cv.load(img)),
                 ("dequantize", lambda: engine.nat.dequantize_canvas(cv.buf.data_ptr(), out.data_ptr(), B, H, W, cv.pitch,
                                                                      engine._stream_ptr()))):
    med, lo, hi = median_us(fn)
    print(f"{name:10s} median {med:7.1f} us  (min {lo:.1f}, max {hi:.1f})  {nbytes / med / 1e3:7.1f} GB/s of {nbytes / 1e6:.1f} MB")
