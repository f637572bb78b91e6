"""The reference's float -> u8 cast pinned on the host: tests/u8_model.py's model_u8 (the rule the GPU tests compute
expected bytes with) against numpy's literal `(255 * arr).astype(np.uint8)` on every class of fp32 input, all fp16
patterns and seeded fp64 values; the oracle and casts.reference_f32 against the same; and, through the recordings
of tests/recorded.py, the oracle against the real reference's process_single_gpu on an fp16 image and on a sampler
whose output leaves [0, 1].  CPU only."""
import sys

import numpy as np
import pytest
import torch

import ref_loader
import usdu_oracle as orc
from __graft_entry__ import load_package
from inputs import make_input
from recorded import digest, reference_digest
from u8_model import WildSampler, edge_f32, model_u8, ref_u8, seeded_f32, special_f32

load_package()
from comfyui_distributed_b200.casts import reference_f32  # noqa: E402


def _x86_rule_holds() -> bool:
    probe = np.array([1.004, 2.0, -0.01, np.inf, 1e10, np.nan, -1e10], dtype=np.float32)
    return np.array_equal(ref_u8(probe), [0, 254, 254, 0, 0, 0, 0]) and ref_u8(np.array([3e9]))[0] == 0


pytestmark = pytest.mark.skipif(not _x86_rule_holds(), reason="this host's numpy does not cast out-of-range floats to "
                                "uint8 as on x86 (cvttss2si / cvttsd2si), the behaviour the reference was recorded with")


def _check(x: np.ndarray):
    want = ref_u8(x)
    got = model_u8(torch.from_numpy(x) * 255).numpy()
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, [(x.view(np.uint16 if x.itemsize == 2 else np.uint32 if x.itemsize == 4 else np.uint64)[i],
                            x[i], got[i], want[i]) for i in bad[:8]]


def test_model_matches_numpy_on_fp32_edges():
    x = edge_f32()
    assert x.size > 19000
    _check(x)


def test_model_matches_numpy_on_special_fp32_values():
    x = special_f32()
    _check(x)
    assert ref_u8(np.array([1.004, 1.01, 2.0, -0.01], dtype=np.float32)).tolist() == [0, 1, 254, 254]


def test_model_matches_numpy_on_seeded_fp32_patterns():
    for k in range(4):
        _check(seeded_f32(100 + k, 1 << 22))


def test_model_matches_numpy_on_every_fp16_pattern():
    _check(np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(np.float16))


def test_model_matches_numpy_on_seeded_fp64_values():
    rng = np.random.default_rng(7)
    bits = rng.integers(0, 1 << 63, 1 << 20, dtype=np.int64).view(np.float64) * rng.choice([-1, 1], 1 << 20)
    wide = rng.uniform(-1.2e10, 1.2e10, 1 << 20) / 255
    unit = rng.uniform(-2, 3, 1 << 20)
    bounds = np.array([2.0 ** 31, -2.0 ** 31, 2.0 ** 31 - 1, -2.0 ** 31 - 1, 2.0 ** 24, np.inf, -np.inf, np.nan]) / 255
    edges = np.concatenate([np.nextafter(bounds, np.inf), np.nextafter(bounds, -np.inf), bounds])
    _check(np.concatenate([bits, wide, unit, edges]))


def test_every_code_over_255_truncates_back_to_itself():
    """k / 255 in fp32 (IEEE division, what reference_f32 hands the kernels) casts back to k for all 256 codes."""
    codes = np.arange(256, dtype=np.float32) / np.float32(255)
    assert np.array_equal(ref_u8(codes), np.arange(256))
    assert np.array_equal(model_u8(torch.from_numpy(codes) * 255).numpy(), np.arange(256))


@pytest.mark.parametrize("dtype", [np.float16, np.float32, np.float64])
def test_oracle_quantises_in_the_input_dtype(dtype):
    x = np.concatenate([seeded_f32(3, 1 << 16).astype(dtype), (np.arange(256) / 255).astype(dtype),
                        np.random.default_rng(4).uniform(-1.5, 2.5, 1 << 16).astype(dtype)])
    assert np.array_equal(orc.quantize_u8(x), ref_u8(x))


def test_reference_f32_gives_the_reference_bytes():
    """fp16 (every pattern) and fp64: the fp32 values reference_f32 returns cast (as the kernels do, fp32) to the bytes
    the reference gets in the input's own dtype; fp32 passes through uncopied; bf16 is converted as it is."""
    x16 = torch.from_numpy(np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(np.float16))
    x64 = torch.from_numpy(np.random.default_rng(9).uniform(-3, 4, 1 << 20))
    for x in (x16, x64):
        y = reference_f32(x)
        assert y.dtype == torch.float32 and y.shape == x.shape
        assert np.array_equal(ref_u8(y.numpy()), ref_u8(x.numpy()))
    k = torch.arange(256, dtype=torch.float64) / 255
    assert np.array_equal(ref_u8(reference_f32(k.half()).numpy()), np.arange(256))        # fp16(k/255) -> k, all codes
    x32 = torch.rand(8)
    assert reference_f32(x32) is x32
    xb = torch.rand(8).bfloat16()
    assert torch.equal(reference_f32(xb), xb.float())


# ---- the oracle against the real reference, on inputs outside fp32 and [0, 1] ---------------------------------------
def _t0_torch(seed, den):
    d, omd = float(np.float32(den)), float(np.float32(1.0) - np.float32(den))
    cache = {}

    def fn(px, s, _d):
        if px.shape not in cache:
            cache[px.shape] = torch.from_numpy(orc.t0_noise(seed, tuple(px.shape)))
        return torch.clamp(px * omd + cache[px.shape] * d, 0.0, 1.0)
    return fn


def _run_reference(monkeypatch, img, fn, tile, pad, blur, uniform):
    node, fake_nodes = ref_loader.make_reference_node()
    fake_nodes.fn = fn
    monkeypatch.setitem(sys.modules, "nodes", fake_nodes.module)      # other tests swap their own stand-in in and out
    (res,) = node.process_single_gpu(torch.from_numpy(img), None, [[torch.zeros(1, 77, 8), {}]], [[torch.zeros(1, 77, 8), {}]],
                                     None, 5, 20, 8.0, "euler", "normal", 0.5, tile, tile, pad, blur, uniform, False)
    return res


def fp16_node_case():
    """An fp16 IMAGE holding fp16(k / 255) for every k: the multiply in fp16 gives k back, one in fp32 does not."""
    img = make_input("noise", 21, 1, 100, 140)
    k = np.round(img * 255).astype(np.int64)
    return (k / 255).astype(np.float16), dict(tile=64, pad=8, blur=4, uniform=True)


def wild_input_case():
    """An image with NaN, +-inf and values outside [0, 1], and the WildSampler."""
    img = make_input("smooth", 22, 1, 96, 120) * np.float32(1.25) - np.float32(0.1)
    img[0, 0, :3] = [np.nan, np.inf, -np.inf]
    img[0, 50, 60:63] = [1e10, 1.01, -0.01]
    return img.astype(np.float32), dict(tile=64, pad=8, blur=4, uniform=True)


def test_oracle_matches_reference_on_an_fp16_image(monkeypatch):
    img, g = fp16_node_case()
    ref = orc.process_single(img, orc.make_t0_denoiser(5, 0.5), g["tile"], g["tile"], g["pad"], g["blur"], g["uniform"])
    assert not np.array_equal(orc.quantize_u8(img), orc.quantize_u8(img.astype(np.float32)))     # the case tells them apart
    key = "u8_cast/process_single_gpu/fp16_image"
    assert digest(ref) == reference_digest(key, ref_loader.available(),
                                           lambda: _run_reference(monkeypatch, img, _t0_torch(5, 0.5), g["tile"], g["pad"], g["blur"], g["uniform"]))


def test_oracle_matches_reference_with_an_out_of_range_sampler(monkeypatch):
    img, g = wild_input_case()
    s = WildSampler()
    ref = orc.process_single(img, s.numpy(), g["tile"], g["tile"], g["pad"], g["blur"], g["uniform"])
    key = "u8_cast/process_single_gpu/wild_sampler"
    assert digest(ref) == reference_digest(key, ref_loader.available(),
                                           lambda: _run_reference(monkeypatch, img, lambda px, seed, den: s(px), g["tile"], g["pad"], g["blur"],
                                                                  g["uniform"]))
