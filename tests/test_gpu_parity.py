"""GPU parity tests: the sm_90a kernels (through the C ABI / ctypes) against the oracle
and the committed golden fixtures.  Bit-exact (integer / byte work)."""
import json
import os

import numpy as np
import pytest
import torch

import usdu_oracle as orc
from __graft_entry__ import load_package
from inputs import make_input

load_package()
from comfyui_distributed_b200 import _native as nat  # noqa: E402
from comfyui_distributed_b200 import engine, planner  # noqa: E402
from comfyui_distributed_b200.denoise import T0Denoiser  # noqa: E402
from comfyui_distributed_b200.nodes import UltimateSDUpscaleDistributed  # noqa: E402
from comfyui_distributed_b200.testing import T0Model  # noqa: E402

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
SINGLE = json.load(open(os.path.join(G, "single_index.json")))["cases"]
DEV = "cuda:0"


def _stream():
    return torch.cuda.current_stream().cuda_stream


@pytest.fixture(params=["mma", "fast", "generic"], autouse=True)
def kernel_path(request):
    """Every test runs three times: with the tensor-core kernels (when the plan allows them), with the integer-pipe
    fast kernels, and with the generic any-scale kernels forced."""
    engine.FORCE_GENERIC = request.param == "generic"
    engine.FORCE_NO_MMA = request.param != "mma"
    yield request.param
    engine.FORCE_GENERIC = False
    engine.FORCE_NO_MMA = False


@pytest.mark.parametrize("B,H,W", [(1, 64, 64), (2, 33, 50), (1, 7, 1021), (1, 540, 960)])
def test_quantize_dequantize(B, H, W):
    rng = np.random.default_rng(0)
    img = rng.random((B, H, W, 3), dtype=np.float32)
    img[0, 0, 0] = [0.0, 1.0, 0.999999]
    x = torch.from_numpy(img).to(DEV)
    pitch = (W * 3 + 127) // 128 * 128
    canvas = torch.zeros((B, H, pitch), dtype=torch.uint8, device=DEV)
    nat.quantize_canvas(x.data_ptr(), canvas.data_ptr(), B, H, W, pitch, _stream())
    got = canvas[:, :, :W * 3].reshape(B, H, W, 3).cpu().numpy()
    assert np.array_equal(got, orc.quantize_u8(img))
    back = torch.empty_like(x)
    nat.dequantize_canvas(canvas.data_ptr(), back.data_ptr(), B, H, W, pitch, _stream())
    assert np.array_equal(back.cpu().numpy(), orc.dequantize_u8(got))


def test_dequantize_every_code_is_ieee_division():
    u = np.arange(256, dtype=np.uint8).repeat(48).reshape(1, 16, 256, 3)          # W3 = 768: vector path
    canvas = torch.from_numpy(u.reshape(1, 16, 768)).to(DEV).contiguous()
    out = torch.empty((1, 16, 256, 3), dtype=torch.float32, device=DEV)
    nat.dequantize_canvas(canvas.data_ptr(), out.data_ptr(), 1, 16, 256, 768, _stream())
    assert np.array_equal(out.cpu().numpy(), u.astype(np.float32) / np.float32(255.0))


@pytest.mark.parametrize("n", [0, 1, 15, 16, 4099, 544 * 544 * 3])
def test_pack_unpack(n):
    rng = np.random.default_rng(n)
    v = rng.random(n, dtype=np.float32)
    x = torch.from_numpy(v).to(DEV)
    q = torch.empty(n, dtype=torch.uint8, device=DEV)
    nat.pack_tiles_u8(x.data_ptr(), q.data_ptr(), n, _stream())
    assert np.array_equal(q.cpu().numpy(), orc.quantize_u8(v))
    f = torch.empty(n, dtype=torch.float32, device=DEV)
    nat.unpack_tiles_f32(q.data_ptr(), f.data_ptr(), n, _stream())
    assert np.array_equal(f.cpu().numpy(), orc.dequantize_u8(orc.quantize_u8(v)))


@pytest.mark.parametrize("W,H,tile,pad,blur,uniform", [
    (700, 500, 256, 32, 8, True), (700, 500, 256, 32, 16, True), (300, 260, 128, 16, 32, True),
    (300, 260, 128, 16, 0, True), (200, 168, 64, 8, 64, False), (1300, 1100, 512, 32, 8, True),
    (640, 400, 128, 64, 255, True)])
def test_feather_templates(W, H, tile, pad, blur, uniform):
    p = planner.Plan.build(W, H, tile, tile, pad, blur, uniform)
    dp = engine.DevicePlan(p, torch.device(DEV))
    pool = dp.mask_pool.cpu().numpy()
    for t in p.tiles:
        off, pitch = p._mask_off[t.idx], p._mask_pitch[t.idx]
        got = pool[off: off + pitch * t.eh].reshape(t.eh, pitch)[:, :t.ew]
        ref = orc.tile_mask_window(W, H, t.x, t.y, p.tw, p.th, blur, t.region)
        assert np.array_equal(got, ref), (t.idx, blur)


def _crop_all(img_np, p, B):
    dp = engine.DevicePlan.get(p, torch.device(DEV))
    canvas = engine.Canvas(dp, B).load(torch.from_numpy(img_np).to(DEV))
    ids = list(range(len(p.tiles)))
    buf, offs = canvas.crop(ids)
    return canvas, ids, buf, offs


@pytest.mark.parametrize("kind,B,H,W,tile,pad,uniform", [
    ("noise", 1, 512, 512, 256, 32, True), ("checker", 1, 300, 420, 128, 16, True), ("noise", 2, 260, 300, 128, 16, True),
    ("smooth", 1, 168, 200, 64, 8, False), ("noise", 1, 90, 100, 128, 32, True), ("noise", 1, 1100, 1300, 512, 32, True),
    ("noise", 1, 333, 777, 64, 128, True)])
def test_crop_resize_matches_oracle(kind, B, H, W, tile, pad, uniform):
    img = make_input(kind, 3, B, H, W)
    p = planner.Plan.build(W, H, tile, tile, pad, 8, uniform)
    canvas, ids, buf, offs = _crop_all(img, p, B)
    cu8 = orc.quantize_u8(img)
    oplan = orc.make_plan(W, H, tile, tile, pad, uniform)[2]
    host = buf.cpu().numpy()
    for i, t in enumerate(oplan):
        ref = orc.extract_tile(cu8, t)
        got = host[offs[i]: offs[i] + ref.size].reshape(ref.shape)
        assert np.array_equal(got, ref), t.idx


@pytest.mark.parametrize("src_u8", [False, True])
@pytest.mark.parametrize("kind,B,H,W,tile,pad,blur,uniform", [
    ("noise", 1, 512, 512, 256, 32, 8, True), ("checker", 1, 300, 420, 128, 16, 16, True),
    ("noise", 2, 260, 300, 128, 16, 4, True), ("smooth", 1, 168, 200, 64, 8, 8, False),
    ("noise", 1, 90, 100, 128, 32, 8, True), ("noise", 1, 333, 777, 64, 128, 8, True)])
def test_blend_all_tiles_in_order_matches_oracle(kind, B, H, W, tile, pad, blur, uniform, src_u8):
    """One launch, overlapping tiles, ascending order == sequential blend_tile calls."""
    img = make_input(kind, 5, B, H, W)
    p = planner.Plan.build(W, H, tile, tile, pad, blur, uniform)
    dp = engine.DevicePlan.get(p, torch.device(DEV))
    canvas = engine.Canvas(dp, B).load(torch.from_numpy(img).to(DEV))
    ids = list(range(len(p.tiles)))
    offs, total = p.slot_offsets(ids, B)
    rng = np.random.default_rng(11)
    proc = rng.random(total, dtype=np.float32)
    if kind == "checker":
        proc = (rng.integers(0, 2, total) * 1.0).astype(np.float32)
    src = torch.from_numpy(proc).to(DEV)
    if src_u8:
        q = torch.empty(total, dtype=torch.uint8, device=DEV)
        nat.pack_tiles_u8(src.data_ptr(), q.data_ptr(), total, _stream())
        src = q
    canvas.blend(ids, src, offs)
    ref = orc.quantize_u8(img)
    tw, th, oplan = orc.make_plan(W, H, tile, tile, pad, uniform)
    for i, t in enumerate(oplan):
        m = orc.tile_mask_window(W, H, t.x, t.y, tw, th, blur, (t.x1, t.y1, t.x2, t.y2))
        tile_f = proc[offs[i]: offs[i] + B * t.ph * t.pw * 3].reshape(B, t.ph, t.pw, 3)
        orc.blend_processed(ref, tile_f, t, m)
    assert np.array_equal(canvas.result_u8().cpu().numpy(), ref)


@pytest.mark.parametrize("case", SINGLE, ids=lambda c: c["name"])
def test_single_gpu_job_matches_reference_golden(case):
    """Whole path through the node API == fixtures produced by the REAL reference."""
    img = make_input(case["kind"], case["seed"], case["B"], case["H"], case["W"])
    if case["B"] == 1 or case["B"] % 4 == 1:
        node = UltimateSDUpscaleDistributed()
        (out,) = node.run(torch.from_numpy(img).to(DEV), T0Model(), None, None, None, case["denoise_seed"], 20, 8.0,
                          "euler", "normal", case["denoise"], case["tile_w"], case["tile_h"], case["padding"],
                          case["mask_blur"], case["uniform"], False)
    else:   # the fixture came from process_single_gpu directly (run() enforces the 4n+1 rule)
        out = engine.upscale_single(torch.from_numpy(img).to(DEV), T0Denoiser(case["denoise_seed"], case["denoise"]),
                                    case["tile_w"], case["tile_h"], case["padding"], case["mask_blur"], case["uniform"])
    assert out.is_cuda and out.dtype == torch.float32
    got = out.cpu().numpy()
    ref = np.load(os.path.join(G, f"single_{case['name']}.npz"))["out"]
    assert np.array_equal(got, orc.dequantize_u8(ref))
    assert np.abs(got.astype(np.float16).astype(np.float32) - ref / 255.0).max() <= 1e-3   # north_star tolerance


def test_node_accepts_host_tensor_and_returns_host_tensor():
    case = SINGLE[0]
    img = make_input(case["kind"], case["seed"], case["B"], case["H"], case["W"])
    node = UltimateSDUpscaleDistributed()
    x = torch.from_numpy(img)
    keep = x.clone()
    (out,) = node.run(x, T0Model(), None, None, None, case["denoise_seed"], 20, 8.0, "euler", "normal",
                      case["denoise"], case["tile_w"], case["tile_h"], case["padding"], case["mask_blur"],
                      case["uniform"], False)
    assert not out.is_cuda
    assert torch.equal(x, keep)                                     # inputs are not mutated
    ref = np.load(os.path.join(G, f"single_{case['name']}.npz"))["out"]
    assert np.array_equal(out.numpy(), orc.dequantize_u8(ref))
    assert node.last_stats["gpu_launches"] > 0


def test_alternating_geometries_keep_their_graphs_and_evict_one_at_a_time(kernel_path):
    """Two jobs of different geometry called in turn replay their captured graphs (no recapture), and filling the graph
    cache with other geometries evicts the least recently used entry only; results stay those of the reference."""
    if kernel_path != "mma":
        pytest.skip("host-side caching is the same for every kernel family")
    cases = [c for c in SINGLE if c["B"] == 1][:2]
    assert len(cases) == 2

    def run(c):
        img = torch.from_numpy(make_input(c["kind"], c["seed"], c["B"], c["H"], c["W"])).to(DEV)
        out = engine.upscale_single(img, T0Denoiser(c["denoise_seed"], c["denoise"]), c["tile_w"], c["tile_h"], c["padding"],
                                    c["mask_blur"], c["uniform"])
        ref = np.load(os.path.join(G, f"single_{c['name']}.npz"))["out"]
        assert np.array_equal(out.cpu().numpy(), orc.dequantize_u8(ref))

    cache = engine.GraphedWaves._cache
    cache.clear()
    run(cases[0]), run(cases[1])
    held = list(cache.values())
    assert len(held) == 2
    for _ in range(3):
        run(cases[0]), run(cases[1])
    assert list(cache.values()) == held or list(cache.values()) == held[::-1]        # same objects: nothing was recaptured
    first = held[0]
    for i in range(cache.capacity - 1):                                              # fill the cache with other geometries
        x = torch.rand(1, 96 + 8 * i, 128, 3, device=DEV)
        engine.upscale_single(x, T0Denoiser(1, 0.5), 64, 64, 8, 4, True)
        run(cases[1])                                                                # keeps this one recent
    assert held[1] in cache.values() and first not in cache.values() and len(cache) == cache.capacity
    run(cases[0])                                                                    # recaptured, still exact


def test_node_rejects_bad_batch():
    node = UltimateSDUpscaleDistributed()
    with pytest.raises(ValueError, match="4n\\+1"):
        node.run(torch.zeros(2, 64, 64, 3), T0Model(), None, None, None, 0, 20, 8.0, "euler", "normal", 0.5,
                 64, 64, 8, 8, True, False)


def test_static_replay_semantics_single_process():
    """A 3-participant static-mode job replayed on ONE GPU (per-participant canvases,
    u8 transport, ordered final blend) == oracle.replay_static."""
    B, H, W, tile, pad, blur = 1, 300, 420, 128, 16, 8
    img = make_input("noise", 8, B, H, W)
    p = planner.Plan.build(W, H, tile, tile, pad, blur, True)
    asg = [[1, 4, 7, 8, 11], [2, 6, 9], [0, 3, 5, 10]]
    den = T0Denoiser(77, 0.5)
    dp = engine.DevicePlan.get(p, torch.device(DEV))
    x = torch.from_numpy(img).to(DEV)
    master = None
    shipped = {}
    for r, tiles in enumerate(asg):
        c = engine.Canvas(dp, B).load(x)
        s = engine.run_progressive(c, tiles, den, keep_processed=True)
        if r == 0:
            master = c
        else:
            shipped.update(s)
    order = sorted(shipped)
    offs, cur = [], 0
    for t in order:
        offs.append(cur)
        cur += shipped[t].numel()
    src = torch.cat([shipped[t].reshape(-1) for t in order])
    master.blend(order, src, np.array(offs, dtype=np.int64))
    ref = orc.replay_static(img, orc.make_t0_denoiser(77, 0.5), tile, tile, pad, blur, True, asg)
    assert np.array_equal(master.result().cpu().numpy(), ref)


STATIC_REF = json.load(open(os.path.join(G, "static_ref_index.json")))["cases"]


@pytest.mark.parametrize("case", STATIC_REF, ids=lambda c: c["name"])
def test_static_jobs_of_the_real_reference_replayed_on_one_gpu(case):
    """The multi-worker jobs the REAL reference ran over HTTP (oracle/ref_static_run.py; recorded pull
    order, uniform and non-uniform tiles, B = 1 and 5) replayed participant by participant on one GPU:
    per-participant progressive canvases in the recorded order, u8 transport, ascending final blend."""
    import hashlib
    B, H, W, tile = case["B"], case["H"], case["W"], case["tile"]
    img = make_input(case["kind"], case["seed"], B, H, W)
    p = planner.Plan.build(W, H, tile, tile, case["padding"], case["mask_blur"], case["uniform"])
    den = T0Denoiser(case["denoise_seed"], case["denoise"])
    dp = engine.DevicePlan.get(p, torch.device(DEV))
    x = torch.from_numpy(img).to(DEV)
    master, shipped = None, {}
    for r, tiles in enumerate(case["assignment"]):
        c = engine.Canvas(dp, B).load(x)
        s = engine.run_progressive(c, tiles, den, keep_processed=True)
        if r == 0:
            master = c
        else:
            shipped.update(s)
    order = sorted(shipped)
    offs, cur = [], 0
    for t in order:
        offs.append(cur)
        cur += (shipped[t].numel() + 15) // 16 * 16
    src = torch.zeros(max(cur, 16), dtype=torch.uint8, device=DEV)
    for t, o in zip(order, offs):
        src[o:o + shipped[t].numel()] = shipped[t].reshape(-1)
    master.blend(order, src, np.array(offs, dtype=np.int64))
    out = master.result_u8().cpu().numpy()
    assert hashlib.sha256(np.ascontiguousarray(out).tobytes()).hexdigest() == case["sha256"]


def test_full_size_properties_cfg2():
    """4K->8K canvas, 512-px tiles (BASELINE.json configs[1]) through size-independent
    properties: (i) denoise=0 with an identity sampler leaves every pixel whose crop was
    not resampled... in general LANCZOS down/up is lossy, so use the exact invariants:
    constant canvases are fixed points; (ii) result == oracle on a sampled set of windows
    of the final canvas is covered by the golden cases; here (iii) idempotence of the
    blend for alpha in {0,255} and determinism across two runs."""
    B, H, W = 1, 4320, 7680
    const = torch.full((B, H, W, 3), 200 / 255.0, dtype=torch.float32, device=DEV)
    ident = lambda tiles, rows: tiles
    out = engine.upscale_single(const, ident, 512, 512, 32, 8, True)
    assert torch.equal(out, const)                                  # LANCZOS of a constant is the constant
    g = torch.Generator(device=DEV).manual_seed(0)
    img = torch.floor(torch.rand((B, H, W, 3), device=DEV, generator=g) * 255) / 255
    den = T0Denoiser(123, 0.5)
    st = {}
    a = engine.upscale_single(img, den, 512, 512, 32, 8, True, stats=st)
    b = engine.upscale_single(img, den, 512, 512, 32, 8, True)
    assert torch.equal(a, b)
    assert st["tiles"] == 135 and st["waves"] == 31
    assert planner.get_plan(W, H, 512, 512, 32, 8, True).fast
    part = a[:, 1000:1400].cpu().numpy()                            # output values are k/255 (IEEE division)
    assert np.array_equal(orc.dequantize_u8(np.round(part * 255).astype(np.uint8)), part)
    # spot-check three windows of the big canvas against the oracle run on a sub-canvas is not
    # valid (progressive dependencies), so check the FIRST tile's window, which depends on nothing
    p = planner.get_plan(W, H, 512, 512, 32, 8, True)
    t0 = p.tiles[0]
    ot = orc.make_plan(W, H, 512, 512, 32, True)[2][0]
    cu8 = orc.quantize_u8(img[:, :ot.y2, :ot.x2].cpu().numpy())
    tin = orc.extract_tile(cu8, ot)
    tout = orc.make_t0_denoiser(123, 0.5)(tin, ot)
    m = orc.tile_mask_window(W, H, ot.x, ot.y, 512, 512, 8, (ot.x1, ot.y1, ot.x2, ot.y2))
    orc.blend_processed(cu8, tout, ot, m)
    # only the part of tile 0's window not touched by later tiles: its interior minus the overlap bands
    safe = (slice(None), slice(0, 512 - 64), slice(0, 512 - 64))
    assert np.array_equal((a[safe].cpu().numpy() * 255).round().astype(np.uint8), cu8[safe])


@pytest.mark.parametrize("n_bands", [1, 2, 4, 9, None])
@pytest.mark.parametrize("kind,B,H,W,tile,pad,blur", [("noise", 1, 600, 420, 128, 16, 8), ("smooth", 5, 300, 260, 64, 32, 40),
                                                      ("noise", 1, 333, 777, 64, 128, 8)])
def test_host_pipeline_matches_oracle(kind, B, H, W, tile, pad, blur, n_bands):
    """Band-pipelined host path (overlapped upload / kernels / download, a different topological
    order of the same DAG) == the sequential reference semantics; pageable inputs (staged band by
    band through a pinned buffer) and pinned inputs (uploaded in place)."""
    img = make_input(kind, 13, B, H, W)
    ref = orc.process_single(img, orc.make_t0_denoiser(5, 0.4), tile, tile, pad, blur, True)
    for pinned in (False, True, False):                  # later calls replay the captured band graphs
        x = torch.from_numpy(img.copy())
        x = x.pin_memory() if pinned else x
        out = engine.upscale_host(x, T0Denoiser(5, 0.4), tile, tile, pad, blur, True, n_bands=n_bands)
        assert not out.is_cuda and out.is_pinned() and np.array_equal(out.numpy(), ref)
        assert np.array_equal(x.numpy(), img)            # the caller's tensor is never written
