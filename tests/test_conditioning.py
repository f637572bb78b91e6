"""Per-tile conditioning cropping == the reference's utils/usdu_utils.py functions on the same inputs: run side by
side where the reference tree is present, against its recorded results (tests/recorded.py) everywhere."""
import copy

import pytest
import torch

import ref_loader
from __graft_entry__ import load_package
from recorded import digest, reference_digest

load_package()
from comfyui_distributed_b200 import conditioning as C  # noqa: E402

class FakeControl:
    def __init__(self, hint, prev=None):
        self.cond_hint_original = hint
        self.previous_controlnet = prev

    def copy(self):
        return copy.copy(self)

    def set_previous_controlnet(self, p):
        self.previous_controlnet = p


def _ref():
    ref_loader.load()
    import sys
    return sys.modules[ref_loader.PKG + ".utils.usdu_utils"]


REGIONS = [((480, 992, 1056, 1568), (7680, 4320), (544, 544)), ((0, 0, 544, 544), (1300, 1100), (544, 544)),
           ((724, 524, 1300, 1100), (1300, 1100), (544, 544)), ((10, 20, 170, 150), (300, 260), (160, 136))]


def _hints(c):
    out = []
    while c is not None:
        out.append(c.cond_hint_original)
        c = c.previous_controlnet
    return out


@pytest.mark.parametrize("region,canvas,tile", REGIONS)
def test_control_hint_crop_matches_reference(region, canvas, tile):
    g = torch.Generator().manual_seed(1)
    h1 = torch.rand(1, 3, canvas[1] // 4, canvas[0] // 4, generator=g)
    h2 = torch.rand(2, 3, canvas[1] // 8 + 3, canvas[0] // 8 + 1, generator=g)
    mine = {"control": FakeControl(h1.clone(), FakeControl(h2.clone()))}
    C.crop_control_hints(mine, region, canvas, tile)

    def reference():
        theirs = {"control": FakeControl(h1.clone(), FakeControl(h2.clone()))}
        _ref().crop_controlnet(theirs, region, canvas, canvas, tile, 0, 0)
        return _hints(theirs["control"])

    got = _hints(mine["control"])
    assert all(h.shape[-2:] == (tile[1], tile[0]) for h in got)
    assert digest(got) == reference_digest(f"conditioning/control_hints/{region}/{canvas}/{tile}", ref_loader.available(), reference)


@pytest.mark.parametrize("region,canvas,tile", REGIONS)
def test_area_gligen_reflatents_match_reference(region, canvas, tile):
    init = (canvas[0] // 2, canvas[1] // 2)
    areas = [(40, 60, 10, 20), (8, 8, 0, 0), (500, 500, 3, 7), (1, 1, 400, 400)]
    boxes = [("e1", 20, 30, 5, 6), ("e2", 64, 64, 60, 90), ("e3", 4, 4, 500, 500)]
    g = torch.Generator().manual_seed(2)
    lat = [torch.rand(1, 4, canvas[1] // 8, canvas[0] // 8, generator=g), torch.rand(1, 4, 1, 40, 50, generator=g)]

    def run(crop_area, crop_gligen, crop_reference_latents):
        out = []
        for area in areas:
            d = {"area": area, "strength": 1.0}
            crop_area(d, area)
            out.append(d)
        d = {"gligen": ("position", "m", list(boxes))}
        crop_gligen(d)
        out.append(d)
        d = {"reference_latents": [t.clone() for t in lat]}
        crop_reference_latents(d)
        out.append(d)
        return out

    mine = run(lambda d, a: C.crop_area(d, region, init, canvas, 0, 0),
               lambda d: C.crop_gligen(d, region, init, canvas, 0, 0),
               lambda d: C.crop_reference_latents(d, region, canvas, tile))

    def reference():
        u = _ref()
        return run(lambda d, a: u.crop_area(d, region, init, canvas, tile, 0, 0),
                   lambda d: u.crop_gligen(d, region, init, canvas, tile, 0, 0),
                   lambda d: u.crop_reference_latents(d, region, init, canvas, tile, 0, 0))

    assert digest(mine) == reference_digest(f"conditioning/area_gligen_reflatents/{region}/{canvas}/{tile}",
                                            ref_loader.available(), reference)


def test_crop_cond_and_clone_do_not_touch_the_originals():
    hint = torch.rand(1, 3, 64, 64)
    cond = [[torch.rand(1, 77, 8), {"control": FakeControl(hint), "area": (8, 8, 0, 0), "pooled_output": torch.rand(1, 8)}]]
    keep = hint.clone()
    out = C.crop_cond(C.clone_conditioning(cond), (0, 0, 128, 128), (256, 256), (256, 256), (128, 128))
    assert torch.equal(hint, keep) and cond[0][1]["control"].cond_hint_original is hint
    assert out[0][1]["control"].cond_hint_original.shape == (1, 3, 128, 128)
    if not torch.cuda.is_available():        # masks are cropped on the GPU only: loud failure, never a CPU path
        from comfyui_distributed_b200._native import NativeError
        with pytest.raises(NativeError):
            C.crop_cond([[None, {"mask": torch.rand(1, 8, 8)}]], (0, 0, 8, 8), (8, 8), (8, 8), (8, 8))
