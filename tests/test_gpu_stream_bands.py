"""The canvas quantise / dequantise as row bands inside the wave graph (engine.CastBands): the same bytes as the eager
passes around the graph, for several grid caps, band counts and both priority settings, on cfg2 and cfg5; and one
captured graph serving different input and output tensors through its device-side argument block."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from __graft_entry__ import load_package

load_package()
from comfyui_distributed_b200 import engine  # noqa: E402
from comfyui_distributed_b200.denoise import T0Denoiser  # noqa: E402

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
WORKLOADS = {"cfg2_4k_to_8k_sdxl_512px": (1, 4320, 7680, 512, 32, 8), "cfg5_video_17f_4k": (17, 2160, 3840, 512, 32, 8)}


def _canvas(B, H, W):                         # bench.py's synthetic input
    g = torch.Generator().manual_seed(0)
    return torch.floor(torch.rand(B, H, W, 3, generator=g) * 255) / 255


def _digest(out: torch.Tensor) -> str:
    q = torch.round(out.to(torch.float32) * 255).to(torch.uint8).cpu().contiguous()
    return hashlib.sha256(q.numpy().tobytes()).hexdigest()


def _expected(name):
    return json.load(open(os.path.join(G, "bench_digests.json")))["digests"][f"{name}/n1/reference"]["sha256"]


class _Knobs:
    def __init__(self, **kw):
        self.kw = {k.upper(): v for k, v in kw.items()}

    def __enter__(self):
        self.saved = {k: getattr(engine, k) for k in self.kw}
        for k, v in self.kw.items():
            setattr(engine, k, v)

    def __exit__(self, *a):
        for k, v in self.saved.items():
            setattr(engine, k, v)


@pytest.mark.parametrize("name,ctas,bands,priority", [("cfg2_4k_to_8k_sdxl_512px", 16, 4, True), ("cfg2_4k_to_8k_sdxl_512px", 132, 8, False),
                                                      ("cfg2_4k_to_8k_sdxl_512px", 33, 12, True), ("cfg5_video_17f_4k", 66, 8, True),
                                                      ("cfg5_video_17f_4k", 16, 3, False)])
def test_cast_bands_give_the_eager_passes_bytes(name, ctas, bands, priority):
    B, H, W, tile, pad, blur = WORKLOADS[name]
    img = _canvas(B, H, W).cuda()
    with _Knobs(stream_overlap=False):
        ref = engine.upscale_single(img, T0Denoiser(123, 0.5), tile, tile, pad, blur, True)
    assert _digest(ref) == _expected(name)
    with _Knobs(stream_overlap=True, stream_ctas=ctas, stream_bands=bands, stream_priority=priority):
        for _ in range(2):
            out = engine.upscale_single(img, T0Denoiser(123, 0.5), tile, tile, pad, blur, True)
            assert torch.equal(out, ref)
            del out
        gw = list(engine.GraphedWaves._cache.values())[-1]
        assert gw.casts is not None and gw.exec
    assert _digest(ref) == _expected(name)


def test_one_graph_serves_different_images_and_results():
    """The argument block: two inputs and fresh outputs through ONE captured graph, back to back without a sync, each
    equal to the eager path's result for that input."""
    B, H, W, tile, pad, blur = 1, 1080, 1920, 256, 32, 8
    g = torch.Generator(device="cuda").manual_seed(7)
    a = torch.rand((B, H, W, 3), device="cuda", generator=g)
    b = torch.rand((B, H, W, 3), device="cuda", generator=g)
    den = T0Denoiser(5, 0.5)
    with _Knobs(stream_overlap=False):
        ra = engine.upscale_single(a, den, tile, tile, pad, blur, True)
        rb = engine.upscale_single(b, den, tile, tile, pad, blur, True)
    assert not torch.equal(ra, rb)
    with _Knobs(stream_overlap=True):
        engine.GraphedWaves._cache.clear()
        outs = [engine.upscale_single(x, den, tile, tile, pad, blur, True) for x in (a, b, a, b)]
        assert len(engine.GraphedWaves._cache) == 1
        gw = list(engine.GraphedWaves._cache.values())[0]
        assert gw.casts is not None
        assert len({o.data_ptr() for o in outs}) == 4
        for o, want in zip(outs, (ra, rb, ra, rb)):
            assert torch.equal(o, want)
    assert np.array_equal(outs[0].cpu().numpy(), ra.cpu().numpy())
