"""Every float -> u8 cast of the CUDA path against the reference's rule, `(255 * arr).astype(np.uint8)` on x86
(tests/u8_model.py, pinned to numpy by tests/test_u8_cast_model.py), outside [0, 1] and fp32 as well as inside:

- pack_tiles_u8 and quantize_rows on all 2^32 fp32 bit patterns, and their scalar tails;
- Q1, the blend's staging of fp32 sampler output, in each kernel family on all 2^32 patterns;
- Q0 in the crop that reads the fp32 image itself (usdu_tile_crop_resize_f32) on all 2^32 patterns;
- whole jobs with NaN, +-inf and out-of-range values in the image and in the sampler output, on every kernel family
  and level schedule, against the oracle;
- fp16 / fp64 inputs to the node, the conditioning masks, the collector and the sampler output, against the oracle.

Expected bytes are computed on the GPU by model_u8 in chunks of at most 2^26 elements."""
import numpy as np
import pytest
import torch

import usdu_oracle as orc
from __graft_entry__ import load_package
from inputs import MASK_CROP_CASES, make_input, make_mask
from u8_model import WildSampler, model_u8_of, seeded_f32, special_f32

load_package()
from comfyui_distributed_b200 import _native as nat  # noqa: E402
from comfyui_distributed_b200 import conditioning as C  # noqa: E402
from comfyui_distributed_b200 import engine, planner  # noqa: E402
from comfyui_distributed_b200.nodes import UltimateSDUpscaleDistributed  # noqa: E402
from comfyui_distributed_b200.nodes.collector import _native_pack  # noqa: E402
from comfyui_distributed_b200.testing import T0Model  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ALL = 1 << 32


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _patterns(start: int, n: int) -> torch.Tensor:
    """fp32 tensor of the bit patterns start, start + 1, ... (mod 2^32) on the device."""
    b = torch.arange(start, start + n, dtype=torch.int64, device=DEV) & 0xFFFFFFFF
    return torch.where(b >= 1 << 31, b - (1 << 32), b).to(torch.int32).view(torch.float32)


def _assert_bytes(what: str, x: torch.Tensor, got: torch.Tensor, want: torch.Tensor):
    bad = torch.nonzero(got.reshape(-1) != want.reshape(-1)).flatten()
    if bad.numel():
        i = bad[:6]
        xs = x.reshape(-1)[i]
        rows = [(f"0x{b & 0xFFFFFFFF:08x}", v, g, w) for b, v, g, w in
                zip(xs.view(torch.int32).tolist(), xs.tolist(), got.reshape(-1)[i].tolist(), want.reshape(-1)[i].tolist())]
        pytest.fail(f"{what}: {bad.numel()} mismatches; first (bits, x, got, want): {rows}")


@pytest.fixture(params=["mma", "fast", "generic"])
def family(request):
    engine.FORCE_GENERIC = request.param == "generic"
    engine.FORCE_NO_MMA = request.param != "mma"
    yield request.param
    engine.FORCE_GENERIC = False
    engine.FORCE_NO_MMA = False


# ---- the streaming casts -------------------------------------------------------------------------------------------
def test_every_fp32_pattern_through_pack_and_quantize_rows():
    """Vector paths: n % 16 == 0 for pack_tiles_u8; W = 4096 (3W % 16 == 0) for quantize_rows."""
    W, H = 4096, 5461
    n = H * W * 3                                                   # just under 2^26
    q = torch.empty(n, dtype=torch.uint8, device=DEV)
    canvas = torch.empty((1, H, W * 3), dtype=torch.uint8, device=DEV)
    for start in range(0, ALL, n):
        x = _patterns(start, n)
        want = model_u8_of(x)
        nat.pack_tiles_u8(x.data_ptr(), q.data_ptr(), n, _stream())
        _assert_bytes("pack_tiles_u8", x, q, want)
        nat.quantize_rows(x.data_ptr(), canvas.data_ptr(), 1, H, W, W * 3, 0, H, _stream())
        _assert_bytes("quantize_rows", x, canvas, want)


def _mixed(n: int, seed: int) -> np.ndarray:
    """The special values first, then seeded bit patterns."""
    s = special_f32()
    return np.concatenate([s, seeded_f32(seed, max(n - s.size, 0))])[:n]


@pytest.mark.parametrize("r", range(1, 16))
def test_pack_scalar_tail(r):
    """n % 16 == r: the last r elements take the scalar loop; every special value passes through it."""
    s = special_f32()
    body = seeded_f32(r, 16 * 40)
    for k in range(0, s.size, r):
        tail = np.resize(s[k:k + r], r)
        x = torch.from_numpy(np.concatenate([body, tail])).to(DEV)
        q = torch.empty(x.numel(), dtype=torch.uint8, device=DEV)
        nat.pack_tiles_u8(x.data_ptr(), q.data_ptr(), x.numel(), _stream())
        _assert_bytes(f"pack_tiles_u8 n={x.numel()}", x, q, model_u8_of(x))


@pytest.mark.parametrize("B,H,W,y0,y1", [(2, 7, 13, 0, 7), (2, 7, 13, 2, 5), (1, 5, 333, 1, 4), (3, 9, 20, 4, 9),
                                         (1, 4, 1021, 0, 1), (2, 6, 4, 5, 6), (1, 3, 7, 0, 3)])
def test_quantize_rows_tails_and_row_ranges(B, H, W, y0, y1):
    """W % 4 != 0 (no vector path), 3W % 16 != 0 (vector rows with scalar ends), and partial row ranges: rows
    [y0, y1) of every frame are cast; nothing else of the canvas (other rows, pitch padding) is written."""
    pitch = (3 * W + 127) // 128 * 128
    x = torch.from_numpy(_mixed(B * H * W * 3, 10 * W + y0).reshape(B, H, W, 3)).to(DEV)
    canvas = torch.full((B, H, pitch), 0xA5, dtype=torch.uint8, device=DEV)
    nat.quantize_rows(x.data_ptr(), canvas.data_ptr(), B, H, W, pitch, y0, y1, _stream())
    want = torch.full_like(canvas, 0xA5)
    want[:, y0:y1, :3 * W] = model_u8_of(x[:, y0:y1]).reshape(B, y1 - y0, 3 * W)
    xs = torch.zeros((B, H, pitch), dtype=torch.float32, device=DEV)
    xs[:, :, :3 * W] = x.reshape(B, H, 3 * W)
    _assert_bytes(f"quantize_rows {B}x{H}x{W} rows [{y0}, {y1})", xs, canvas, want)


# ---- Q1 in the blend, Q0 in the crop from the fp32 image: an identity, fully opaque geometry --------------------------
# 4096 x 4096, 512-px tiles, no padding, no blur: 64 tiles in one wave, every tile's window is its own 512 x 512 square
# at full alpha, and nothing is resampled -- so the blended canvas is exactly the cast of the sampler output, and the
# crop's output exactly the dequantised cast of the image.
GEO = (4096, 4096, 512, 0, 0)


def _identity_plan():
    W, H, tile, pad, blur = GEO
    p = planner.Plan.build(W, H, tile, tile, pad, blur, True)
    ids = list(range(len(p.tiles)))
    assert len(ids) == 64 and len(p.waves(ids)) == 1
    assert all((t.pw, t.ph, t.ew, t.eh) == (tile, tile, tile, tile) for t in p.tiles)
    offs, total = p.slot_offsets(ids, 1)
    gather = torch.empty((H, W, 3), dtype=torch.int64, device=DEV)       # canvas pixel -> element of the packed tiles
    for i, t in enumerate(p.tiles):
        gather[t.y1:t.y2, t.x1:t.x2] = int(offs[i]) + torch.arange(tile * tile * 3, device=DEV).view(tile, tile, 3)
    return p, ids, offs, total, gather.view(-1)


def test_every_fp32_pattern_through_the_blend(family):
    p, ids, offs, total, gather = _identity_plan()
    canvas = engine.Canvas(engine.DevicePlan.get(p, torch.device(DEV)), 1)
    assert canvas.path_blend == {"mma": 2, "fast": 1, "generic": 0}[family]
    canvas.buf.zero_()
    got = canvas.result_u8()
    src = torch.zeros(total, dtype=torch.float32, device=DEV)
    for start in range(0, ALL, gather.numel()):
        x = _patterns(start, gather.numel())
        src[gather] = x
        canvas.blend(ids, src, offs)
        _assert_bytes(f"blend ({family})", x, got, model_u8_of(x))


def test_every_fp32_pattern_through_the_crop_from_the_image():
    """usdu_tile_crop_resize_f32 (tensor-core crop reading the fp32 IMAGE, Q0 on the fly): k / 255 of the cast."""
    p, ids, offs, total, gather = _identity_plan()
    W, H = GEO[0], GEO[1]
    canvas = engine.Canvas(engine.DevicePlan.get(p, torch.device(DEV)), 1)
    assert canvas.can_crop_image()
    codes = torch.from_numpy(orc.dequantize_u8(np.arange(256, dtype=np.uint8))).to(DEV)
    out = torch.empty(total, dtype=torch.float32, device=DEV)
    for start in range(0, ALL, gather.numel()):
        img = _patterns(start, gather.numel()).view(1, H, W, 3)
        canvas.crop(ids, out=out, image=img)
        want = codes[model_u8_of(img).long()].view(-1)
        got = out[gather]
        if not torch.equal(got, want):
            _assert_bytes("crop from the fp32 image (as k / 255 -> k)", img, torch.round(got * 255).to(torch.int64),
                          torch.round(want * 255).to(torch.int64))
            pytest.fail("crop output is not exactly k / 255")


# ---- whole jobs ----------------------------------------------------------------------------------------------------
JOB = dict(W=420, H=300, tile=128, pad=16, blur=8)


def _wild_image(B, H, W, seed):
    img = make_input("smooth", seed, B, H, W) * np.float32(1.25) - np.float32(0.1)
    s = special_f32()
    flat = img.reshape(-1)
    flat[::997][:s.size] = s[:flat[::997].size]
    flat[5:5 + s.size] = s
    return img.astype(np.float32)


def _job(img, denoiser):
    return engine.upscale_single(torch.from_numpy(img).to(DEV), denoiser, JOB["tile"], JOB["tile"], JOB["pad"], JOB["blur"], True)


def _oracle_job(img, fn):
    return orc.process_single(img, fn, JOB["tile"], JOB["tile"], JOB["pad"], JOB["blur"], True)


@pytest.mark.parametrize("schedule", ["split_crop", "waves"])
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.float16])
def test_job_with_an_out_of_range_sampler_and_image(family, schedule, out_dtype):
    """NaN, +-inf, +-1e10 and values just outside [0, 1] in the image (Q0) and in the sampler output (Q1), fp32 and
    fp16 sampler output; twice, so that the second call replays the captured wave graph."""
    img = _wild_image(1, JOB["H"], JOB["W"], 31)
    sampler = WildSampler(out_dtype)
    want = _oracle_job(img, sampler.numpy())
    saved = engine.SCHEDULE
    engine.SCHEDULE = schedule
    try:
        for _ in range(2):
            got = _job(img, sampler).cpu().numpy()
            assert np.array_equal(got, want), f"{int((got != want).sum())} pixels differ from the oracle"
    finally:
        engine.SCHEDULE = saved


def _node_run(x, seed=5, den=0.5):
    (out,) = UltimateSDUpscaleDistributed().run(x, T0Model(), None, None, None, seed, 20, 8.0, "euler", "normal", den,
                                                JOB["tile"], JOB["tile"], JOB["pad"], JOB["blur"], True, False)
    return out.cpu().numpy()


@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("dtype", ["fp32_out_of_range", "fp16", "fp64"])
def test_node_image_dtype_and_range(where, dtype):
    """The node's IMAGE cast (Q0) on the host route (banded upload) and the device route: fp32 with out-of-range values,
    and fp16 / fp64, which the reference multiplies by 255 in their own dtype."""
    if dtype == "fp32_out_of_range":
        img = _wild_image(1, JOB["H"], JOB["W"], 32)
    else:
        k = np.round(make_input("noise", 33, 1, JOB["H"], JOB["W"]) * 255)
        img = (k / 255).astype(np.float16 if dtype == "fp16" else np.float64)
        if dtype == "fp64":
            img += np.random.default_rng(3).uniform(-4e-9, 4e-9, img.shape)      # products a hair either side of k
    x = torch.from_numpy(img)
    want = _oracle_job(img, orc.make_t0_denoiser(5, 0.5))
    got = _node_run(x.to(DEV) if where == "device" else x)
    assert np.array_equal(got, want), f"{int((got != want).sum())} pixels differ from the oracle"


@pytest.mark.parametrize("where", ["cpu", "cuda"])
@pytest.mark.parametrize("kind", ["fp16", "out_of_range"])
def test_mask_crop_dtype_and_range(where, kind):
    name, mkind, seed, B, (Hm, Wm), region, canvas, tile = MASK_CROP_CASES[0]
    m = make_mask(mkind, seed, B, Hm, Wm)
    if kind == "fp16":
        m = m.astype(np.float16)
    else:
        m = m * np.float32(1.5) - np.float32(0.2)
        s = special_f32()
        m.reshape(-1)[7::101][:s.size] = s                               # spread over the mask, inside the cropped region
    out = C.MaskCropper(DEV).crop(torch.from_numpy(m).to(where), region, canvas, tile)
    got = np.round(out.cpu().numpy() * 255).astype(np.uint8)
    want = np.stack([orc.crop_mask_u8(orc.quantize_u8(m[b]), region, canvas, tile) for b in range(B)])
    assert np.array_equal(got, want)


@pytest.mark.parametrize("where", ["cpu", "cuda"])
@pytest.mark.parametrize("kind", ["fp16", "out_of_range"])
def test_collector_pack_dtype_and_range(where, kind):
    rng = np.random.default_rng(8)
    if kind == "fp16":
        imgs = (np.round(rng.random((2, 40, 56, 3)) * 255) / 255).astype(np.float16)
    else:
        imgs = rng.uniform(-1.5, 2.5, (2, 40, 56, 3)).astype(np.float32)
        imgs.reshape(-1)[3:3 + special_f32().size] = special_f32()
    q = _native_pack(torch.from_numpy(imgs).to(where))
    assert q.is_cuda and q.dtype == torch.uint8
    assert np.array_equal(q.cpu().numpy(), orc.quantize_u8(imgs))
