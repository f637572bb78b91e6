"""Full-size parity on the BASELINE.json configurations: the CUDA path's result on bench.py's synthetic canvases
against the committed digests of the reference (tests/golden/bench_digests.json, oracle/gen_bench_digests.py: the REAL
reference's process_single_gpu for cfg2 and cfg5, the oracle for cfg4 / cfg4alt).  These are the sizes the small
parity cases do not reach: 31- and 126-wave progressive DAGs, TMA box clipping at W = 7680 / 15360, 17-frame batches,
64-bit offsets."""
import hashlib
import json
import os

import pytest
import torch

from __graft_entry__ import load_package

load_package()
from comfyui_distributed_b200 import engine  # noqa: E402
from comfyui_distributed_b200.denoise import T0Denoiser  # noqa: E402
from comfyui_distributed_b200.nodes import UltimateSDUpscaleDistributed  # noqa: E402
from comfyui_distributed_b200.testing import T0Model  # noqa: E402

pytestmark = pytest.mark.gpu
DB = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "bench_digests.json")))["digests"]
WORKLOADS = {
    "cfg2_4k_to_8k_sdxl_512px": (1, 4320, 7680, 512, 32, 8),
    "cfg1_512_256px": (1, 512, 512, 256, 32, 8),
    "cfg4_16k_256px": (1, 8640, 15360, 256, 32, 8),
    "cfg4alt_8k_256px": (1, 8192, 8192, 256, 32, 8),
    "cfg5_video_17f_4k": (17, 2160, 3840, 512, 32, 8),
}


def _canvas(B, H, W):
    g = torch.Generator().manual_seed(0)
    x = torch.rand(B, H, W, 3, generator=g)
    return torch.floor(x * 255) / 255


def _digest(out: torch.Tensor) -> str:
    q = torch.round(out.to(torch.float32) * 255).to(torch.uint8).cpu().contiguous()
    return hashlib.sha256(q.numpy().tobytes()).hexdigest()


def _expected(name):
    for src in ("reference", "oracle"):
        if f"{name}/n1/{src}" in DB:
            return DB[f"{name}/n1/{src}"]["sha256"]
    pytest.skip(f"no digest for {name}")


@pytest.mark.parametrize("name", list(WORKLOADS))
def test_device_resident_job_matches_the_reference_digest(name):
    B, H, W, tile, pad, blur = WORKLOADS[name]
    want = _expected(name)
    img = _canvas(B, H, W).cuda()
    for _ in range(2):                       # the second call replays the captured graph
        out = engine.upscale_single(img, T0Denoiser(123, 0.5), tile, tile, pad, blur, True)
        assert _digest(out) == want
        del out


@pytest.mark.parametrize("name", ["cfg2_4k_to_8k_sdxl_512px", "cfg5_video_17f_4k"])
def test_node_api_on_a_host_tensor_matches_the_reference_digest(name):
    B, H, W, tile, pad, blur = WORKLOADS[name]
    want = _expected(name)
    host = _canvas(B, H, W)
    node = UltimateSDUpscaleDistributed()
    for _ in range(2):
        (out,) = node.run(host, T0Model(), None, None, None, 123, 20, 8.0, "euler", "normal", 0.5, tile, tile, pad, blur,
                          True, False)
        assert not out.is_cuda and _digest(out) == want
        del out


@pytest.mark.parametrize("name,schedule", [("cfg2_4k_to_8k_sdxl_512px", "split_crop"), ("cfg2_4k_to_8k_sdxl_512px", "waves"),
                                           ("cfg5_video_17f_4k", "split_crop"), ("cfg5_video_17f_4k", "waves"),
                                           ("cfg1_512_256px", "split_crop")])
def test_every_level_schedule_gives_the_same_canvas(name, schedule):
    """engine.SCHEDULE: "split_crop" is the default (engine.run_split: the crop jobs of wave k+1 that do not read what wave
    k changes run on a second stream beside sampler(k) / blend(k)); "waves" is the plain level loop -- the same digest as
    the reference on every replay of both."""
    B, H, W, tile, pad, blur = WORKLOADS[name]
    want = _expected(name)
    img = _canvas(B, H, W).cuda()
    saved = engine.SCHEDULE
    engine.SCHEDULE = schedule
    try:
        for _ in range(3):
            out = engine.upscale_single(img, T0Denoiser(123, 0.5), tile, tile, pad, blur, True)
            assert _digest(out) == want
            del out
        if name != "cfg1_512_256px":                    # (cfg1 has 4 single-tile waves: run_split has nothing to split)
            gw = list(engine.GraphedWaves._cache.values())[-1]
            assert gw.split == (schedule == "split_crop")
    finally:
        engine.SCHEDULE = saved
