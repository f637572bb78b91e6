"""The tile path on batches past 2^31 elements, on u8 canvases past 2^32 bytes and at the 65,535-frame launch limit,
against the oracle.

A full oracle run is out of reach at these sizes, but every frame of a job is independent of the others given its own
input and its own sampler noise.  So every big batch here is periodic, frame b = base[b % k] for k distinct base frames:
the oracle computes the k base frames only, and the device compares all B frames with them through a [B // k, k, ...]
view.  Output buffers are filled with a sentinel (NaN, 0xA5) before each launch, so a write that lands in the wrong
place, or never happens, shows up as a mismatch.  The whole-job cases use PeriodicT0, the T0 sampler with the noise of
k frames, so frame b of a job sees the noise frame b % k of the k-frame job.

Each case states the device memory it needs and skips, naming that number, when less is free; it frees what it holds
before it returns, and prints its peak allocation and wall time (run pytest with -s to see them)."""
import gc
import hashlib
import json
import os
import time

import numpy as np
import pytest
import torch

import png_model
import usdu_oracle as orc
from __graft_entry__ import load_package
from inputs import make_input

load_package()
from comfyui_distributed_b200 import _native as nat  # noqa: E402
from comfyui_distributed_b200 import engine, planner  # noqa: E402
from comfyui_distributed_b200 import http_worker as hw  # noqa: E402
from comfyui_distributed_b200.denoise import T0Denoiser  # noqa: E402
from comfyui_distributed_b200.nodes import UltimateSDUpscaleDistributed, collector  # noqa: E402
from comfyui_distributed_b200.testing import T0Model  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GB = 1 << 30
H4K, W4K = 2160, 3840
CFG5 = (512, 32, 8)                         # tile, padding, mask blur of BASELINE.md cfg5
TINY = (48, 64, 64, 8, 8)                   # H, W, tile, padding, mask blur: one 72 x 72 processed tile per frame
FAMILY_PATH = {"mma": 2, "fast": 1, "generic": 0}
DIGESTS = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "bench_digests.json")))["digests"]


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _need(nbytes: int):
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip(f"needs {nbytes / GB:.1f} GiB of free device memory, {free / GB:.1f} GiB free")


@pytest.fixture(autouse=True)
def _measure(request):
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    held = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated() - held
    gc.collect()
    torch.cuda.empty_cache()
    print(f"\n[large batch] {request.node.name}: peak {peak / GB:.2f} GiB, {dt:.1f} s")
    assert torch.cuda.memory_allocated() - held < 64 << 20, "the case left device memory behind"


@pytest.fixture
def kernel_family(request):
    """Force one kernel family (engine.Canvas.path); the flags are restored afterwards."""
    saved = engine.FORCE_GENERIC, engine.FORCE_NO_MMA
    engine.FORCE_GENERIC = request.param == "generic"
    engine.FORCE_NO_MMA = request.param != "mma"
    yield request.param
    engine.FORCE_GENERIC, engine.FORCE_NO_MMA = saved


class PeriodicT0(T0Denoiser):
    """T0Denoiser for a batch whose frame b is base[b % k]: the noise of the k-frame T0 job.  The fused T0 pass reads
    the noise modulo its length (usdu_t0_denoise), so the k-frame noise stands for its B / k-fold repetition without
    the copy.  The period is part of graph_key, so GraphedWaves never confuses these graphs with the plain T0 ones."""

    def __init__(self, seed: int, denoise: float, k: int):
        super().__init__(seed, denoise)
        self.k = int(k)
        self.graph_key = self.graph_key + ("period", self.k)

    def noise(self, shape, device):
        assert shape[0] % self.k == 0, (shape, self.k)
        return super().noise((self.k,) + tuple(shape[1:]), device)


def _drop_graphs(graph_key):
    """Forget the captured graphs (and the canvases they hold) of one sampler configuration."""
    d = engine.GraphedWaves._cache._d
    for key in [key for key in d if key[2] == graph_key]:
        del d[key]


# ---------------------------------------------------------------------------------------------------------------------
# periodic batches
# ---------------------------------------------------------------------------------------------------------------------
def _periodic(base: torch.Tensor, B: int, out: torch.Tensor = None) -> torch.Tensor:
    """[B, ...] with frame b = base[b % k] (base [k, ...] on the device); into `out` when given."""
    k = base.shape[0]
    assert B % k == 0, (B, k)
    if out is None:
        out = torch.empty((B,) + tuple(base.shape[1:]), dtype=base.dtype, device=base.device)
    out.view((B // k,) + tuple(base.shape)).copy_(base.unsqueeze(0).expand((B // k,) + tuple(base.shape)))
    return out


def _assert_periodic(t: torch.Tensor, want: torch.Tensor, what):
    """t [B, ...] == want[b % k] for every frame b, compared on the device a few hundred MB at a time; NaN equals NaN
    (the sentinel of fp32 outputs that must stay untouched)."""
    k, B = want.shape[0], t.shape[0]
    assert B % k == 0 and tuple(t.shape[1:]) == tuple(want.shape[1:]), (what, tuple(t.shape), tuple(want.shape))
    v = t.reshape((B // k,) + tuple(want.shape))
    step = max(1, (256 << 20) // max(want.numel() * want.element_size(), 1))
    for i in range(0, B // k, step):
        blk = v[i:i + step]
        bad = blk != want
        if want.is_floating_point():
            bad &= ~(blk.isnan() & want.isnan())
        if bad.any():
            j, f = (int(x) for x in bad.flatten(2).any(2).nonzero()[0])
            pytest.fail(f"{what}: frame {(i + j) * k + f} of {B} differs from base frame {f}")


def _flat_periodic(flat: torch.Tensor, want: torch.Tensor, n: int, what):
    """flat[:n] == want (flat, period P) repeated, n not necessarily a multiple of P."""
    P = want.numel()
    full = n // P
    if full:
        _assert_periodic(flat[:full * P].view(full, P), want.view(1, P), what)
    rest = n - full * P
    assert torch.equal(flat[full * P: n], want[:rest]) if not want.is_floating_point() else \
        bool(((flat[full * P: n] == want[:rest]) | (flat[full * P: n].isnan() & want[:rest].isnan())).all()), what


def _base_image(seed: int, k: int, H: int, W: int) -> np.ndarray:
    """k fp32 frames: half on the k/255 grid, half anywhere in [-0.02, 1.02) (the cast's clamping and wrap-around)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(k, H, W, 3, generator=g)
    grid = torch.floor(x * 255) / 255
    anywhere = x * 1.04 - 0.02
    return torch.where(torch.rand(k, H, W, 3, generator=g) < 0.5, grid, anywhere).numpy()


def _pitched(u8: np.ndarray, pitch: int, fill: int = 0xA5) -> np.ndarray:
    """u8 frames [k, H, W, 3] -> the canvas rows [k, H, pitch], padding bytes = fill."""
    k, H, W, _ = u8.shape
    out = np.full((k, H, pitch), fill, np.uint8)
    out[:, :, :W * 3] = u8.reshape(k, H, W * 3)
    return out


def _canvas_buffer(B: int, H: int, W: int, fill: int = 0xA5):
    """A u8 canvas [B, H, pitch] with the kernels' 16 bytes of slack behind it, all set to `fill`."""
    pitch = engine.Canvas.pitch_of(W)
    n = B * H * pitch
    raw = torch.full((n + nat.CANVAS_SLACK,), fill, dtype=torch.uint8, device=DEV)
    return raw, raw[:n].view(B, H, pitch), pitch


def _dev(a: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


# ---------------------------------------------------------------------------------------------------------------------
# the canvas casts on an fp32 image of more than 2^31 elements (u8 canvas of more than 2^31 bytes)
# ---------------------------------------------------------------------------------------------------------------------
CAST_B, CAST_K = 102, 3                     # 102 x 2160 x 3840 x 3 = 2.54e9 elements (10.2 GB fp32)


@pytest.mark.parametrize("W", [W4K, W4K - 2], ids=["vector", "scalar"])
def test_casts_past_2_31_elements(W):
    """quantize_canvas / quantize_rows and dequantize_canvas / dequantize_rows on both paths (W % 4 != 0 is the scalar
    one), row bands that end in the last frame, and on the vector path the streamed pair behind a usdu_stream_args block
    at 1, 7 and all SMs' worth of CTAs."""
    B, k, H = CAST_B, CAST_K, H4K
    pitch = engine.Canvas.pitch_of(W)
    assert B * H * W * 3 > 1 << 31 and B * H * pitch > 1 << 31
    _need(B * H * W * 12 + B * H * pitch + 2 * GB)
    base = _base_image(1, k, H, W)
    q = orc.quantize_u8(base)
    want_c = _dev(_pitched(q, pitch))
    want_d = _dev(orc.dequantize_u8(q))
    img = _periodic(_dev(base), B)
    raw, cv, _ = _canvas_buffer(B, H, W)
    bands = [(0, 1000), (1000, H)]

    def fresh_canvas():
        raw.fill_(0xA5)

    def quantized(what):
        _assert_periodic(cv, want_c, what)
        assert bool((raw[-nat.CANVAS_SLACK:] == 0xA5).all()), (what, "slack")

    nat.quantize_canvas(img.data_ptr(), raw.data_ptr(), B, H, W, pitch, _stream())
    quantized("quantize_canvas")
    fresh_canvas()
    for y0, y1 in bands:
        nat.quantize_rows(img.data_ptr(), raw.data_ptr(), B, H, W, pitch, y0, y1, _stream())
    quantized("quantize_rows")
    fresh_canvas()
    nat.quantize_rows(img.data_ptr(), raw.data_ptr(), B, H, W, pitch, H - 8, H, _stream())
    part = want_c.clone()
    part[:, :H - 8] = 0xA5
    _assert_periodic(cv, part, "quantize_rows, last 8 rows")
    del part
    nat.quantize_canvas(img.data_ptr(), raw.data_ptr(), B, H, W, pitch, _stream())

    img.fill_(float("nan"))                  # the image buffer is now the result
    nat.dequantize_canvas(raw.data_ptr(), img.data_ptr(), B, H, W, pitch, _stream())
    _assert_periodic(img, want_d, "dequantize_canvas")
    img.fill_(float("nan"))
    for y0, y1 in bands:
        nat.dequantize_rows(raw.data_ptr(), img.data_ptr(), B, H, W, pitch, y0, y1, _stream())
    _assert_periodic(img, want_d, "dequantize_rows")
    img.fill_(float("nan"))
    nat.dequantize_rows(raw.data_ptr(), img.data_ptr(), B, H, W, pitch, H - 8, H, _stream())
    part = want_d.clone()
    part[:, :H - 8] = float("nan")
    _assert_periodic(img, part, "dequantize_rows, last 8 rows")
    del part

    if W % 4 == 0:
        args = torch.zeros(nat.STREAM_ARGS_BYTES, dtype=torch.uint8, device=DEV)
        for ctas in (1, 7, nat.sm_count()):
            _periodic(_dev(base), B, out=img)
            nat.stream_args_set(args.data_ptr(), img.data_ptr(), img.data_ptr(), _stream())
            fresh_canvas()
            for y0, y1 in bands:
                nat.quantize_rows_streamed(args.data_ptr(), raw.data_ptr(), B, H, W, pitch, y0, y1, ctas, _stream())
            quantized(f"quantize_rows_streamed, {ctas} CTAs")
            img.fill_(float("nan"))
            for y0, y1 in bands:
                nat.dequantize_rows_streamed(raw.data_ptr(), args.data_ptr(), B, H, W, pitch, y0, y1, ctas, _stream())
            _assert_periodic(img, want_d, f"dequantize_rows_streamed, {ctas} CTAs")
    del img, raw, cv, want_c, want_d


def test_pack_and_unpack_past_2_31_elements():
    """pack_tiles_u8 / unpack_tiles_f32 over n > 2^31 elements with a tail of 7 (not a multiple of 16), in the image
    buffer itself; the bytes and floats past n stay untouched."""
    B, k, H, W = CAST_B, CAST_K, H4K, W4K
    N = B * H * W * 3
    n = N - 9
    assert n > 1 << 31 and n % 16 == 7
    _need(N * 5 + 2 * GB)
    base = _base_image(2, k, H, W)
    q = orc.quantize_u8(base)
    want_q = _dev(q).view(-1)
    want_d = _dev(orc.dequantize_u8(q)).view(-1)
    img = _periodic(_dev(base), B)
    flat = img.view(-1)
    dst = torch.full((n + 32,), 0xA5, dtype=torch.uint8, device=DEV)
    nat.pack_tiles_u8(img.data_ptr(), dst.data_ptr(), n, _stream())
    _flat_periodic(dst, want_q, n, "pack_tiles_u8")
    assert bool((dst[n:] == 0xA5).all()), "pack_tiles_u8 wrote past n"
    flat.fill_(float("nan"))
    nat.unpack_tiles_f32(dst.data_ptr(), img.data_ptr(), n, _stream())
    _flat_periodic(flat, want_d, n, "unpack_tiles_f32")
    assert bool(flat[n:].isnan().all()), "unpack_tiles_f32 wrote past n"
    del img, flat, dst, want_q, want_d


# ---------------------------------------------------------------------------------------------------------------------
# crop and blend on a u8 canvas of more than 2^32 bytes, every kernel family
# ---------------------------------------------------------------------------------------------------------------------
TB_B, TB_K = 188, 4                          # 188 x 2160 x 11520 bytes = 4.68 GB


def _cfg5_plan():
    tile, pad, blur = CFG5
    return planner.get_plan(W4K, H4K, tile, tile, pad, blur, True)


def _tile_ids(p):
    return [0, len(p.tiles) // 2 + 1, len(p.tiles) - 1]         # among them the bottom-right tile


_ORACLE = {}


def _oracle_tiles(k, H, W, tile, pad, blur, ids, seed):
    """-> (u8 base canvas [k, H, W, 3], oracle crops per tile, processed tiles per tile [k, ph, pw, 3] fp32, oracle
    canvas after blending them in ascending order)."""
    key = (k, H, W, tile, pad, blur, tuple(ids), seed)
    if key not in _ORACLE:
        _ORACLE.clear()
        cu8 = orc.quantize_u8(make_input("noise", seed, k, H, W))
        mw, mh, oplan = orc.make_plan(W, H, tile, tile, pad, True)
        crops = [orc.extract_tile(cu8, oplan[t]) for t in ids]
        rng = np.random.default_rng(seed)
        proc = [rng.random((k, oplan[t].ph, oplan[t].pw, 3), dtype=np.float32) for t in ids]
        want = cu8.copy()
        for t, pr in zip(ids, proc):
            o = oplan[t]
            orc.blend_processed(want, pr, o, orc.tile_mask_window(W, H, o.x, o.y, mw, mh, blur, (o.x1, o.y1, o.x2, o.y2)))
        _ORACLE[key] = (cu8, crops, proc, want)
    return _ORACLE[key]


def _crop_and_blend(p, B, k, ids, seed, family):
    """One crop launch of `ids` == extract_tile of every base frame; one blend launch from fp32 and from u8 sampler
    output == blend_processed tile after tile, and nothing else on the canvas changes."""
    H, W = p.H, p.W
    cu8, crops, proc, want = _oracle_tiles(k, H, W, p.tile_width, p.padding, p.mask_blur, ids, seed)
    dp = engine.DevicePlan.get(p, torch.device(DEV))
    base_c = _dev(_pitched(cu8, engine.Canvas.pitch_of(W), 0))
    raw, cv, _ = _canvas_buffer(B, H, W)
    _periodic(base_c, B, out=cv)
    c = engine.Canvas(dp, B, buf=cv)
    assert c.path == FAMILY_PATH[family]
    offs, total = p.slot_offsets(ids, B)
    offs = [int(o) for o in offs]
    out = torch.full((total,), float("nan"), dtype=torch.float32, device=DEV)
    _, coffs = c.crop(ids, out=out)
    assert np.array_equal(coffs, offs)
    for i, t in enumerate(ids):
        ref = crops[i]
        _assert_periodic(out[offs[i]: offs[i] + B * ref[0].size].view((B,) + ref.shape[1:]), _dev(ref), ("crop", family, t))
    del out
    src = torch.empty(total, dtype=torch.float32, device=DEV)
    for i, t in enumerate(ids):
        _periodic(_dev(proc[i]), B, out=src[offs[i]: offs[i] + B * proc[i][0].size].view((B,) + proc[i].shape[1:]))
    q = torch.full((total + 16,), 0xA5, dtype=torch.uint8, device=DEV)[:total]
    nat.pack_tiles_u8(src.data_ptr(), q.data_ptr(), total, _stream())
    want_c = _dev(_pitched(want, engine.Canvas.pitch_of(W), 0))
    for s in (src, q):
        _periodic(base_c, B, out=cv)
        c.blend(ids, s, offs)
        _assert_periodic(cv, want_c, ("blend", family, str(s.dtype)))
        assert bool((raw[-nat.CANVAS_SLACK:] == 0xA5).all()), "blend wrote into the canvas slack"
    del raw, cv, c, src, q, base_c, want_c


@pytest.mark.parametrize("kernel_family", ["mma", "fast", "generic"], indirect=True)
def test_crop_and_blend_on_a_canvas_past_2_32_bytes(kernel_family):
    p = _cfg5_plan()
    B, k = TB_B, TB_K
    assert B * H4K * engine.Canvas.pitch_of(W4K) > 1 << 32
    ids = _tile_ids(p)
    slots = p.slot_offsets(ids, B)[1]
    _need(B * H4K * engine.Canvas.pitch_of(W4K) + slots * 9 + 2 * GB)
    _crop_and_blend(p, B, k, ids, 11, kernel_family)


def test_crop_from_an_fp32_image_past_2_31_elements():
    """usdu_tile_crop_resize_f32 (crop_mma<2, *>): the crops straight from the fp32 image == extract_tile of the
    quantised base frames."""
    p = _cfg5_plan()
    B, k, H, W = CAST_B, CAST_K, H4K, W4K
    ids = _tile_ids(p)
    offs, total = p.slot_offsets(ids, B)
    offs = [int(o) for o in offs]
    _need(B * H * W * 12 + B * H * engine.Canvas.pitch_of(W) + total * 4 + 2 * GB)
    base = _base_image(3, k, H, W)
    cu8 = orc.quantize_u8(base)
    tile, pad, _ = CFG5
    oplan = orc.make_plan(W, H, tile, tile, pad, True)[2]
    img = _periodic(_dev(base), B)
    c = engine.Canvas(engine.DevicePlan.get(p, torch.device(DEV)), B)
    assert c.can_crop_image()
    out = torch.full((total,), float("nan"), dtype=torch.float32, device=DEV)
    c.crop(ids, out=out, image=img)
    for i, t in enumerate(ids):
        ref = orc.extract_tile(cu8, oplan[t])
        _assert_periodic(out[offs[i]: offs[i] + B * ref[0].size].view((B,) + ref.shape[1:]), _dev(ref), ("crop f32", t))
    del img, c, out


# ---------------------------------------------------------------------------------------------------------------------
# the gathers of a multi-GPU job over canvases of more than 2^31 bytes
# ---------------------------------------------------------------------------------------------------------------------
def test_gathers_from_slabs_past_2_31_bytes():
    """gather_canvas and gather_dequantize over three slabs, each a distinct canvas of 2.19 GB with its own content:
    rows [y_q, y_q+1) of every frame come from slab q."""
    B, k, H, W = 88, 2, H4K, W4K
    pitch = engine.Canvas.pitch_of(W)
    rows = [0, 700, 1500, H]
    assert B * H * pitch > 1 << 31 and B * H * W * 3 > 1 << 31
    _need(3 * B * H * pitch + B * H * W * 12 + 2 * GB)
    bases = [orc.quantize_u8(make_input("noise", 20 + q, k, H, W)) for q in range(3)]
    slabs = [_periodic(_dev(_pitched(b, pitch, 0)), B) for b in bases]
    want = np.zeros((k, H, W, 3), np.uint8)
    for q in range(3):
        want[:, rows[q]:rows[q + 1]] = bases[q][:, rows[q]:rows[q + 1]]
    ptrs = [s.data_ptr() for s in slabs]
    raw, cv, _ = _canvas_buffer(B, H, W)
    nat.gather_canvas(ptrs, rows, raw.data_ptr(), B, H, W, pitch, _stream())
    _assert_periodic(cv, _dev(_pitched(want, pitch, 0)), "gather_canvas")
    del raw, cv
    img = torch.full((B, H, W, 3), float("nan"), dtype=torch.float32, device=DEV)
    nat.gather_dequantize(ptrs, rows, img.data_ptr(), B, H, W, pitch, _stream())
    _assert_periodic(img, _dev(orc.dequantize_u8(want)), "gather_dequantize")
    del img, slabs


def test_gather_unpack_past_2_31_elements():
    """gather_unpack_f32 into a destination of 2.17e9 floats that starts 4 bytes past a 16-byte boundary, the frame
    pointers cycling over three source frames."""
    n, k, H, W = 87, 3, H4K, W4K
    fe = H * W * 3
    assert n * fe > 1 << 31
    _need(n * fe * 4 + 2 * GB)
    src = _dev(orc.quantize_u8(_base_image(4, k, H, W)))
    ptrs = torch.tensor([src[f % k].data_ptr() for f in range(n)], dtype=torch.int64, device=DEV)
    dst = torch.full((n * fe + 8,), float("nan"), dtype=torch.float32, device=DEV)
    nat.gather_unpack_f32(ptrs.data_ptr(), n, fe, dst.data_ptr() + 4, _stream())
    assert bool(dst[0].isnan()) and bool(dst[1 + n * fe:].isnan().all()), "gather_unpack_f32 wrote outside its frames"
    _assert_periodic(dst[1:1 + n * fe].view(n, fe), _dev(orc.dequantize_u8(src.cpu().numpy())).view(k, fe),
                     "gather_unpack_f32")
    del src, ptrs, dst


# ---------------------------------------------------------------------------------------------------------------------
# 65,535 frames: every batched entry point at the grid limit, and one frame more refused before any launch
# ---------------------------------------------------------------------------------------------------------------------
LIMIT = 65535


def _tiny_plan():
    H, W, tile, pad, blur = TINY
    return planner.get_plan(W, H, tile, tile, pad, blur, True)


@pytest.mark.parametrize("kernel_family", ["mma", "fast", "generic"], indirect=True)
def test_crop_and_blend_at_65535_frames(kernel_family):
    p = _tiny_plan()
    assert p.mma and len(p.tiles) == 1
    total = p.slot_offsets([0], LIMIT)[1]
    _need(LIMIT * p.H * engine.Canvas.pitch_of(p.W) + total * 9 + GB)
    _crop_and_blend(p, LIMIT, 5, [0], 12, kernel_family)


def _refused(fn, untouched):
    """fn raises NativeError before it launches anything: the sentinel-filled output is as it was (`untouched()`)."""
    with pytest.raises(nat.NativeError, match="65535|grid.y"):
        fn()
    torch.cuda.synchronize()
    assert untouched()


@pytest.mark.parametrize("kernel_family", ["mma", "fast", "generic"], indirect=True)
def test_crop_and_blend_refuse_65536_frames(kernel_family):
    p = _tiny_plan()
    B = LIMIT + 1
    ids = [0]
    total = p.slot_offsets(ids, B)[1]
    _need(B * p.H * engine.Canvas.pitch_of(p.W) + total * 5 + GB)
    raw, cv, _ = _canvas_buffer(B, p.H, p.W)
    c = engine.Canvas(engine.DevicePlan.get(p, torch.device(DEV)), B, buf=cv)
    out = torch.full((total,), float("nan"), dtype=torch.float32, device=DEV)
    _refused(lambda: c.crop(ids, out=out), lambda: bool(out.isnan().all()))
    src = torch.zeros(total, dtype=torch.uint8, device=DEV)
    _refused(lambda: c.blend(ids, src, np.zeros(1, np.int64)), lambda: bool((raw == 0xA5).all()))
    if kernel_family == "mma":
        img = torch.zeros((B, p.H, p.W, 3), dtype=torch.float32, device=DEV)
        _refused(lambda: c.crop(ids, out=out, image=img), lambda: bool(out.isnan().all()))
        del img
    del raw, cv, c, out, src


@pytest.mark.parametrize("B", [LIMIT, LIMIT + 1])
def test_casts_at_the_grid_limit(B):
    """The casts stride over rows and frames: at and past 65,535 frames they equal the reference per frame."""
    H, W = TINY[:2]
    k = 5 if B == LIMIT else 8
    pitch = engine.Canvas.pitch_of(W)
    _need(B * H * W * 12 + B * H * pitch + GB)
    base = _base_image(5, k, H, W)
    q = orc.quantize_u8(base)
    img = _periodic(_dev(base), B)
    raw, cv, _ = _canvas_buffer(B, H, W)
    nat.quantize_canvas(img.data_ptr(), raw.data_ptr(), B, H, W, pitch, _stream())
    _assert_periodic(cv, _dev(_pitched(q, pitch)), "quantize_canvas")
    img.fill_(float("nan"))
    nat.dequantize_canvas(raw.data_ptr(), img.data_ptr(), B, H, W, pitch, _stream())
    _assert_periodic(img, _dev(orc.dequantize_u8(q)), "dequantize_canvas")
    del img, raw, cv


PNG_H, PNG_W = 8, 8


def test_png_base64_at_65535_frames_and_refused_past():
    k = 5
    frames = orc.quantize_u8(_base_image(6, k, PNG_H, PNG_W))
    png, text_len, staging_len = nat.png_sizes(PNG_H, PNG_W, 3)
    _need((LIMIT + 1) * (text_len + staging_len + PNG_H * PNG_W * 3) + GB)
    src = _periodic(_dev(frames), LIMIT + 5)[:LIMIT + 1]
    staging = torch.empty((LIMIT + 1) * staging_len, dtype=torch.uint8, device=DEV)
    text = torch.full(((LIMIT + 1) * text_len,), 0xA5, dtype=torch.uint8, device=DEV)
    _refused(lambda: nat.png_base64_u8(src.data_ptr(), LIMIT + 1, PNG_H, PNG_W, 3, staging.data_ptr(), text.data_ptr(),
                                       _stream()), lambda: bool((text == 0xA5).all()))
    nat.png_base64_u8(src.data_ptr(), LIMIT, PNG_H, PNG_W, 3, staging.data_ptr(), text.data_ptr(), _stream())
    want = _dev(np.stack([np.frombuffer(png_model.png_stored_b64(f), np.uint8) for f in frames]))
    _assert_periodic(text[:LIMIT * text_len].view(LIMIT, text_len), want, "png_base64_u8")
    assert bool((text[LIMIT * text_len:] == 0xA5).all())
    del src, staging, text, want


def test_png_encode_at_65535_frames_and_refused_past():
    k = 5
    frames = orc.quantize_u8(_base_image(7, k, PNG_H, PNG_W))
    layout = hw.png_layout(PNG_H, PNG_W)
    assert layout is not None
    n = layout.png_len
    _need((LIMIT + 1) * (n + nat.png_encode_scratch_bytes(1, PNG_H, PNG_W) + PNG_H * PNG_W * 3) + GB)
    src = _periodic(_dev(frames), LIMIT + 5)[:LIMIT + 1]
    out = torch.full(((LIMIT + 1) * n,), 0xA5, dtype=torch.uint8, device=DEV)
    scratch = torch.empty(nat.png_encode_scratch_bytes(LIMIT + 1, PNG_H, PNG_W), dtype=torch.uint8, device=DEV)
    tmpl, runs, chunks = layout.device_tables(src.device)

    def encode(B):
        nat.png_encode_u8(src.data_ptr(), B, PNG_H, PNG_W, 3, tmpl.data_ptr(), n, runs.data_ptr(), len(layout.runs),
                          chunks.data_ptr(), len(layout.chunks), layout.adler_at, scratch.data_ptr(), out.data_ptr(),
                          _stream())

    _refused(lambda: encode(LIMIT + 1), lambda: bool((out == 0xA5).all()))
    encode(LIMIT)
    want = _dev(np.stack([np.frombuffer(hw.encode_png(f), np.uint8) for f in frames]))
    _assert_periodic(out[:LIMIT * n].view(LIMIT, n), want, "png_encode_u8")
    assert bool((out[LIMIT * n:] == 0xA5).all())
    del src, out, scratch


def test_collector_sends_70000_frames_in_groups_of_at_most_65535(monkeypatch):
    """send_to_master's encode of 70,000 8 x 8 frames: one usdu_png_base64_u8 launch of 65,535 frames and one of the
    rest, and frame by frame the texts of the layout model (tests/png_model.py)."""
    B, k = 70000, 7
    base = _base_image(8, k, PNG_H, PNG_W)
    _, text_len, staging_len = nat.png_sizes(PNG_H, PNG_W, 3)
    _need(B * (PNG_H * PNG_W * 3 * 5 + text_len + staging_len) + GB)
    x = _periodic(_dev(base), B)
    calls = []
    real = nat.png_base64_u8

    def counted(src_ptr, n, *rest):
        calls.append(n)
        return real(src_ptr, n, *rest)

    monkeypatch.setattr(nat, "png_base64_u8", counted)
    node = collector.DistributedCollectorNode
    texts = [bytes(t) for t in node.encode(node.pack(x))]
    assert calls == [65535, B - 65535]
    want = [png_model.png_stored_b64(orc.quantize_u8(f)) for f in base]
    assert len(texts) == B
    bad = [b for b in range(B) if texts[b] != want[b % k]]
    assert not bad, f"{len(bad)} frames differ, the first is {bad[0]}"
    del x


# ---------------------------------------------------------------------------------------------------------------------
# whole jobs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("no_mma", [False, True], ids=["default", "no_mma"])
def test_102_frame_cfg5_job_matches_the_reference_digest(no_mma, monkeypatch):
    """bench.py's 17-frame cfg5 input repeated 6 times (2.54e9 elements) through engine.upscale_single with the 17-frame
    T0 noise: every 17-frame block of the result is the real reference's result for the 17-frame job."""
    from test_gpu_fullsize import _canvas
    B, k, H, W = 102, 17, H4K, W4K
    tile, pad, blur = CFG5
    want = DIGESTS["cfg5_video_17f_4k/n1/reference"]["sha256"]
    _need(2 * B * H * W * 12 + B * H * engine.Canvas.pitch_of(W) + 8 * GB)
    monkeypatch.setattr(engine, "FORCE_NO_MMA", no_mma)
    img = _periodic(_canvas(k, H, W).to(DEV), B)
    den = PeriodicT0(123, 0.5, k)
    try:
        out = engine.upscale_single(img, den, tile, tile, pad, blur, True)
        del img
        for i in range(B // k):
            q = torch.round(out[i * k:(i + 1) * k] * 255).to(torch.uint8).cpu().contiguous()
            assert hashlib.sha256(q.numpy().tobytes()).hexdigest() == want, f"frames {i * k}..{(i + 1) * k - 1}"
        del out, q
    finally:
        _drop_graphs(den.graph_key)


def test_65533_frame_job_and_the_node_accept_the_largest_4n1_batch():
    """B = 65,533 (4n+1) tiny frames, periodic over 13 base frames, through engine.upscale_single: every frame equals the
    oracle's process_single of its base frame under the 13-frame T0 noise.  The node takes the same batch (its output,
    with T0 noise drawn for all 65,533 frames, is not compared: the oracle would need gigabytes of host noise)."""
    B, k = 65533, 13
    H, W, tile, pad, blur = TINY
    assert B % 4 == 1 and B % k == 0
    p = _tiny_plan()
    slot = p.slot_offsets([0], B)[1]
    _need(2 * B * H * W * 12 + B * H * engine.Canvas.pitch_of(W) + 3 * slot * 4 + GB)
    base = make_input("noise", 31, k, H, W)
    ref = orc.process_single(base, orc.make_t0_denoiser(123, 0.5), tile, tile, pad, blur, True)
    img = _periodic(_dev(base), B)
    den = PeriodicT0(123, 0.5, k)
    try:
        out = engine.upscale_single(img, den, tile, tile, pad, blur, True)
        _assert_periodic(out, _dev(ref), "upscale_single")
        del out
    finally:
        _drop_graphs(den.graph_key)
    node_den = T0Model().as_usdu_denoiser(seed=123, denoise=0.5)
    try:
        (out,) = UltimateSDUpscaleDistributed().run(img, T0Model(), None, None, None, 123, 20, 8.0, "euler", "normal", 0.5,
                                                    tile, tile, pad, blur, True, False)
        assert out.is_cuda and tuple(out.shape) == (B, H, W, 3) and bool(out.isfinite().all())
        del out
    finally:
        _drop_graphs(node_den.graph_key)
    del img
