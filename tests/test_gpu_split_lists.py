"""The split schedule's role-aware work lists on the GPU: the library's residency table equals the device's occupancy
calculator for every tensor-core list the schedule launches on bench.py's workloads, and the graphed job with tall early
crops, short late crops and the residency-sized blend still gives the reference's digests."""
import hashlib
import json
import os

import pytest
import torch

from __graft_entry__ import load_package

load_package()
from comfyui_distributed_b200 import _native as nat  # noqa: E402
from comfyui_distributed_b200 import engine, planner  # noqa: E402
from comfyui_distributed_b200.denoise import T0Denoiser  # noqa: E402

pytestmark = pytest.mark.gpu
DB = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "bench_digests.json")))["digests"]
WORKLOADS = {  # name: (B, H, W, tile, padding, blur)
    "cfg1_512_256px": (1, 512, 512, 256, 32, 8),
    "cfg2_4k_to_8k_sdxl_512px": (1, 4320, 7680, 512, 32, 8),
    "cfg5_video_17f_4k": (17, 2160, 3840, 512, 32, 8),
}


def _lists(name):
    B, H, W, tile, pad, blur = WORKLOADS[name]
    p = planner.Plan.build(W, H, tile, tile, pad, blur, True)
    waves = engine.split_waves(p, list(range(len(p.tiles))))
    out = []
    for k, w in enumerate(waves):
        offs, _ = p.slot_offsets(w, B)
        chain, side, _, _, bl = p.split_lists(w, offs, waves[k - 1] if k else None, B, 2)
        out.append((chain, side, bl))
    return B, out


@pytest.mark.parametrize("name", list(WORKLOADS))
def test_the_residency_table_equals_the_device(name):
    if nat.sm_count() != 132:
        pytest.skip("the table is the H100 SXM's (132 SMs)")
    torch.cuda.set_device(0)
    _, lists = _lists(name)
    seen = set()
    for chain, side, bl in lists:
        for cr in [chain] + ([side] if side is not None else []):
            for kernel in (nat.KERNEL_CROP_LDG, nat.KERNEL_CROP_TMA, nat.KERNEL_CROP_TMA | nat.KERNEL_LARGE):
                seen.add((kernel, cr.ks2, cr.patch_w, cr.patch_h, 0))
        seen.add((nat.KERNEL_BLEND, bl.ks2, bl.patch_w, bl.patch_h, bl.block_rows))
    for args in sorted(seen):
        assert nat.resident_ctas(*args, True) == nat.resident_ctas(*args, False), args


@pytest.mark.parametrize("name", list(WORKLOADS))
def test_role_aware_lists_give_the_reference_digest(name):
    B, H, W, tile, pad, blur = WORKLOADS[name]
    want = next(DB[f"{name}/n1/{s}"]["sha256"] for s in ("reference", "oracle") if f"{name}/n1/{s}" in DB)
    _, lists = _lists(name)
    if name != "cfg1_512_256px":                 # (cfg1's 16 tiles: every blend fits one round in 16-row blocks)
        assert any(side is not None and (side.items[:, nat.J_CY1] == 32).any() for _, side, _ in lists)
        assert {bl.block_rows for _, _, bl in lists} == {16, 32}
    g = torch.Generator().manual_seed(0)
    img = (torch.floor(torch.rand(B, H, W, 3, generator=g) * 255) / 255).cuda()
    for _ in range(2):                           # the second call replays the captured graph
        out = engine.upscale_single(img, T0Denoiser(123, 0.5), tile, tile, pad, blur, True)
        q = torch.round(out * 255).to(torch.uint8).cpu().contiguous()
        assert hashlib.sha256(q.numpy().tobytes()).hexdigest() == want
        del out
