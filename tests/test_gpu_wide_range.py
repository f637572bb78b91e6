"""The tile kernels across the node's whole parameter range -- tile_width / tile_height 64..2048, padding 0..256,
mask_blur 0..256 (tests/golden/node_signatures.json) -- against the oracle bit for bit, and whole jobs against the real
reference's digests (tests/golden/wide_ref_digests.json, made by oracle/gen_golden.py gen_wide_digests).

Large padding and tiles are where the crop kernel leaves its common build: a tensor-core crop patch taller than the TMA
boxes is staged with plain loads, a crop down-scale above ~1.3 needs two k-steps, and a canvas far smaller than a tile
makes the generic kernels' back-resize read a patch too large for shared memory.  The case list (tests/inputs.py
WIDE_CASES) is pinned to those builds: the CPU tests below derive, from the planner's work lists, which build of each
kernel every case launches, and fail when the list no longer reaches one of them."""
import functools
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import usdu_oracle as orc
from __graft_entry__ import load_package
from inputs import WIDE_CASES, make_input, wide_sampler

load_package()
from comfyui_distributed_b200 import _native as nat  # noqa: E402
from comfyui_distributed_b200 import engine, planner  # noqa: E402
from comfyui_distributed_b200.denoise import T0Denoiser  # noqa: E402

DEV = "cuda:0"
DIGESTS = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "wide_ref_digests.json")))["digests"]
SMEM_LIMIT = 227 * 1024                 # dynamic shared memory one CTA may opt in to on sm_90 (usdu_kernels.cu kMaxSmem)
BOX_ROWS, BOX_BYTES = 48, 512           # the tensor-core crop's two TMA boxes (usdu_mma.cu: kBoxR rows, 2 * kBoxB bytes)
FAMILY_PATH = {"mma": 2, "fast": 1, "generic": 0}


def _cid(c):
    i, B, H, W, tw, th, pad, blur, uni, _ = c
    return f"{i}-b{B}-{W}x{H}-t{tw}x{th}-p{pad}-m{blur}-{'u' if uni else 'n'}"


def _geometry(c):
    """-> (B, H, W, tile_w, tile_h, padding, mask_blur, uniform)"""
    return c[1:9]


# ---------------------------------------------------------------------------------------------------------------------
# which kernel builds a case launches (mirrors the launchers' choices)
# ---------------------------------------------------------------------------------------------------------------------
def generic_smem(wl: planner.WorkList, blend: bool):
    """Shared memory of a generic crop / blend launch (usdu_tile_crop_resize / usdu_tile_blend) -> (bytes, direct).
    Crop: the staged input patch + the intermediate (64-px pitch).  Blend: the canvas block + the intermediate (block-width
    pitch) + the staged patch of the processed tile, or, when that does not fit, no patch -- the horizontal pass then
    reads the tile in global memory (direct)."""
    patch = wl.patch_h * ((wl.patch_w * 3 + 15) // 16 * 16)
    if not blend:
        return patch + wl.patch_h * nat.BLOCK_W * 3, False
    held = nat.BLOCK_H * nat.BLOCK_W * 3 + wl.patch_h * wl.block_cols * 3
    return (held + patch, False) if held + patch <= SMEM_LIMIT else (held, True)


def launched_variants(B, H, W, tw, th, pad, blur, uniform):
    """Kernel builds that one crop and one ordered blend of ALL tiles launch, per family the plan supports:
    crop_mma<SRC,KS> with SRC 1 = canvas through TMA, 0 = canvas through LDG (the patch exceeds the boxes), 2 = the fp32
    image, KS = k-steps (usdu_mma.cu launch_crop); blend_mma<rows,KS>; for the generic kernels the block and whether the
    input patch is staged or read in place.  -> (set of labels, {label: shared-memory bytes} of the generic launches)"""
    p = planner.Plan.build(W, H, tw, th, pad, blur, uniform)
    ids = list(range(len(p.tiles)))
    seen, smem = set(), {}
    if p.mma:
        cr, offs, _ = p.crop_worklist(ids, B, 2)
        bl = p.blend_worklist(ids, offs, 4, 2, B)
        assert cr.path == bl.path == 2
        ks = 2 if cr.ks2 else 1
        tma = (cr.patch_h & 0xFFFF) <= BOX_ROWS and 12 + 3 * cr.patch_w <= BOX_BYTES
        seen.add(f"crop_mma<{1 if tma else 0},{ks}>")
        if W % 4 == 0:                                      # engine.Canvas.can_crop_image
            seen.add(f"crop_mma<2,{ks}>")
        seen.add(f"blend_mma<{bl.block_rows},{2 if bl.ks2 else 1}>")
    cr, offs, _ = p.crop_worklist(ids, B, 0)
    bl = p.blend_worklist(ids, offs, 4, 0, B)
    assert cr.path == bl.path == 0
    seen.add(f"generic_block<{bl.block_cols}x{bl.block_rows}>")
    for name, wl, is_blend in (("generic_crop", cr, False), ("generic_blend", bl, True)):
        n, direct = generic_smem(wl, is_blend)
        label = f"{name}<{'direct' if direct else 'staged'}>"
        seen.add(label)
        smem[label] = max(smem.get(label, 0), n)
    return seen, smem


def families(c):
    """Kernel families the plan of case c supports (the generic kernels take any geometry)."""
    B, H, W, tw, th, pad, blur, uniform = _geometry(c)
    p = planner.get_plan(W, H, tw, th, pad, blur, uniform)
    return [f for f, ok in (("mma", p.mma), ("fast", p.fast), ("generic", True)) if ok]


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the case list reaches every build, and no legal geometry is refused
# ---------------------------------------------------------------------------------------------------------------------
REQUIRED = {
    "crop_mma<1,1>",                 # TMA staging, one k-step (the common build)
    "crop_mma<0,1>",                 # LDG staging: crop patch > 48 plane rows or 12 + 3 * patch_w > 512
    "crop_mma<0,2>",                 # LDG staging and two k-steps (crop down-scale above ~1.3)
    "crop_mma<2,2>",                 # from the fp32 image, two k-steps
    "blend_mma<16,1>", "blend_mma<32,1>", "blend_mma<16,2>", "blend_mma<32,2>",
    "generic_block<64x32>", "generic_block<4x4>",
    "generic_crop<staged>", "generic_blend<staged>",
    "generic_blend<direct>",         # back-resize of a 2304-px tile onto a 64-px canvas: the patch is read in place
}


def test_wide_cases_reach_every_kernel_build():
    seen, smem = set(), {}
    for c in WIDE_CASES:
        s, m = launched_variants(*_geometry(c))
        seen |= s
        for k, v in m.items():
            smem[k] = max(smem.get(k, 0), v)
    assert REQUIRED <= seen, sorted(REQUIRED - seen)
    assert max(smem.values()) <= SMEM_LIMIT, smem


def test_wide_cases_span_the_node_range():
    tiles = {(c[4], c[8]) for c in WIDE_CASES} | {(c[5], c[8]) for c in WIDE_CASES}
    for t in (768, 1024, 2048):
        assert any(tt == t for tt, _ in tiles), t
    for t in (1024, 2048):
        assert (t, True) in tiles and (t, False) in tiles, t          # uniform and non-uniform tiles
    assert {48, 96, 192, 256} <= {c[6] for c in WIDE_CASES}
    assert {64, 128, 256} <= {c[7] for c in WIDE_CASES}
    assert any(c[7] > min(c[4], c[5]) for c in WIDE_CASES)             # feather ramp wider than the tile
    assert {1, 2, 5} <= {c[1] for c in WIDE_CASES}
    assert any(c[3] % 4 for c in WIDE_CASES)
    assert any(c[4] != c[5] for c in WIDE_CASES)
    small = {(c[3], c[2], c[4], c[6]) for c in WIDE_CASES}
    assert {(64, 64, 2048, 256), (48, 80, 2048, 256), (1024, 24, 2048, 256), (32, 32, 1024, 256)} <= small
    assert sum(c[9] for c in WIDE_CASES) >= 6 and set(DIGESTS) == {str(c[0]) for c in WIDE_CASES if c[9]}


@pytest.mark.parametrize("tile", [1024, 1536, 2048])
def test_generic_kernels_fit_shared_memory_on_small_canvases(tile):
    """A canvas far smaller than a tile makes the generic blend read the whole processed tile for a 4x4 block
    (2304 -> 64 px: a 324 x 324 patch).  Every such geometry must still launch: the generic crop and blend need at most
    227 KB of shared memory (the staged patch, or the intermediate alone when the patch is read in place)."""
    worst = 0
    for pad in (64, 128, 192, 256):
        for s in (8, 16, 24, 32, 40, 48, 64, 76, 84, 96, 128, 200):
            for W, H in ((s, s), (s, 1024), (1024, s), (s, 3 * s)):
                p = planner.Plan.build(W, H, tile, tile, pad, 8, True)
                ids = list(range(len(p.tiles)))
                cr, offs, _ = p.crop_worklist(ids, 1, False)
                bl = p.blend_worklist(ids, offs, 4, False, 1)
                for wl, is_blend in ((cr, False), (bl, True)):
                    n, _ = generic_smem(wl, is_blend)
                    assert n <= SMEM_LIMIT, (W, H, tile, pad, is_blend, n)
                    worst = max(worst, n)
    assert worst > 0


# ---------------------------------------------------------------------------------------------------------------------
# GPU: every kernel family on every case against the oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", autouse=True)
def _memo_masks():
    """The oracle's feather windows are pure functions of the geometry and cost seconds at blur 256 on a 2k canvas:
    compute each once for the whole module (read-only, so no caller can change a shared copy)."""
    raw = orc.tile_mask_window

    @functools.lru_cache(maxsize=None)
    def memo(*args):
        m = raw(*args)
        m.setflags(write=False)
        return m

    mp = pytest.MonkeyPatch()
    mp.setattr(orc, "tile_mask_window", lambda W, H, x, y, tw, th, blur, window: memo(W, H, x, y, tw, th, blur, tuple(window)))
    yield
    mp.undo()


@pytest.fixture
def kernel_family(request):
    """Force one kernel family (engine.Canvas.path); the flags are restored afterwards."""
    saved = engine.FORCE_GENERIC, engine.FORCE_NO_MMA
    engine.FORCE_GENERIC = request.param == "generic"
    engine.FORCE_NO_MMA = request.param != "mma"
    yield request.param
    engine.FORCE_GENERIC, engine.FORCE_NO_MMA = saved


def pixel_checker(B, H, W):
    """1-px checker of 0 and 1 in opposite phase per channel: every LANCZOS output is pushed past 0 or 255 by the
    negative lobes, so the clipping of both passes is exercised on every pixel."""
    yy, xx = np.mgrid[0:H, 0:W]
    c = ((xx + yy) % 2).astype(np.float32)
    return np.stack([c, 1 - c, c], -1)[None].repeat(B, 0)


@functools.lru_cache(maxsize=1)
def _oracle_tiles(c, kind):
    """-> (input, oracle crops, processed tiles (flat fp32, the planner's slot offsets), oracle canvas after blending all
    of them in ascending order)."""
    B, H, W, tw, th, pad, blur, uniform = _geometry(c)
    img = make_input("noise", c[0], B, H, W) if kind == "noise" else pixel_checker(B, H, W)
    cu8 = orc.quantize_u8(img)
    mw, mh, oplan = orc.make_plan(W, H, tw, th, pad, uniform)
    crops = [orc.extract_tile(cu8, t) for t in oplan]
    offs, total = planner.get_plan(W, H, tw, th, pad, blur, uniform).slot_offsets(range(len(oplan)), B)
    rng = np.random.default_rng(c[0])
    proc = rng.random(total, dtype=np.float32) if kind == "noise" else rng.integers(0, 2, total).astype(np.float32)
    want = cu8.copy()
    for t, o in zip(oplan, offs):
        m = orc.tile_mask_window(W, H, t.x, t.y, mw, mh, blur, (t.x1, t.y1, t.x2, t.y2))
        orc.blend_processed(want, proc[o:o + B * t.ph * t.pw * 3].reshape(B, t.ph, t.pw, 3), t, m)
    return img, crops, proc, want


KERNEL_CASES = [pytest.param(c, kind, f, id=f"{_cid(c)}-{kind}-{f}")
                for c in WIDE_CASES for kind in ("noise", "checker") for f in families(c)]


@pytest.mark.gpu
@pytest.mark.parametrize("case,kind,kernel_family", KERNEL_CASES, indirect=["kernel_family"])
def test_crop_and_ordered_blend_match_oracle(case, kind, kernel_family):
    """One crop launch of every tile == extract_tile; one blend launch of every tile in ascending order ==
    blend_processed tile after tile, from fp32 and from u8 sampler output; the tensor-core crop straight from the fp32
    image == the canvas crop."""
    B, H, W, tw, th, pad, blur, uniform = _geometry(case)
    img, crops, proc, want = _oracle_tiles(case, kind)
    p = planner.get_plan(W, H, tw, th, pad, blur, uniform)
    dp = engine.DevicePlan.get(p, torch.device(DEV))
    x = torch.from_numpy(img).to(DEV)
    canvas = engine.Canvas(dp, B).load(x)
    assert canvas.path == FAMILY_PATH[kernel_family]
    ids = list(range(len(p.tiles)))
    buf, offs = canvas.crop(ids)
    host = buf.cpu().numpy()
    for i, ref in enumerate(crops):
        assert np.array_equal(host[offs[i]: offs[i] + ref.size].reshape(ref.shape), ref), ("crop", i)
    if canvas.can_crop_image():
        fbuf, foffs = canvas.crop(ids, image=x)
        assert np.array_equal(foffs, offs) and torch.equal(fbuf, buf)
    boffs, total = p.slot_offsets(ids, B)
    src = torch.from_numpy(proc).to(DEV)
    q = torch.empty(total, dtype=torch.uint8, device=DEV)
    nat.pack_tiles_u8(src.data_ptr(), q.data_ptr(), total, torch.cuda.current_stream().cuda_stream)
    for s in (src, q):
        c = engine.Canvas(dp, B).load(x)
        c.blend(ids, s, boffs)
        assert np.array_equal(c.result_u8().cpu().numpy(), want), ("blend", s.dtype)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: whole jobs == oracle.process_single == the real reference
# ---------------------------------------------------------------------------------------------------------------------
JOBS = [c for c in WIDE_CASES if c[9]]


@functools.lru_cache(maxsize=1)
def _oracle_job(c):
    B, H, W, tw, th, pad, blur, uniform = _geometry(c)
    img = make_input("noise", c[0], B, H, W)
    seed, den = wide_sampler(c[0])
    return img, orc.process_single(img, orc.make_t0_denoiser(seed, den), tw, th, pad, blur, uniform)


def _run_job(c):
    B, H, W, tw, th, pad, blur, uniform = _geometry(c)
    img, ref = _oracle_job(c)
    seed, den = wide_sampler(c[0])
    out = engine.upscale_single(torch.from_numpy(img).to(DEV), T0Denoiser(seed, den), tw, th, pad, blur, uniform).cpu().numpy()
    assert np.array_equal(out, ref), _cid(c)
    q = np.round(out * 255).astype(np.uint8)
    assert hashlib.sha256(q.tobytes()).hexdigest() == DIGESTS[str(c[0])]          # what the reference itself produced


@pytest.mark.gpu
@pytest.mark.parametrize("case,kernel_family", [pytest.param(c, f, id=f"{_cid(c)}-{f}") for c in JOBS for f in ("mma", "fast")],
                         indirect=["kernel_family"])
def test_whole_job_matches_oracle_and_reference(case, kernel_family):
    """Default kernel choice (tensor-core where the plan allows, else integer-pipe, else generic) and the same job with
    the tensor-core kernels switched off."""
    _run_job(case)


def _ldg_or_two_ksteps(c):
    return bool({"crop_mma<0,1>", "crop_mma<0,2>", "crop_mma<1,2>"} & launched_variants(*_geometry(c))[0])


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in JOBS if _ldg_or_two_ksteps(c)], ids=_cid)
def test_ldg_and_two_kstep_jobs_under_every_schedule(case, monkeypatch):
    """Jobs whose tensor-core crops are staged with LDG or need two k-steps, under the level-wave schedule and the
    split-crop schedule (default); a replay of the captured graph gives the same result."""
    for schedule in ("waves", "split_crop"):
        monkeypatch.setattr(engine, "SCHEDULE", schedule)
        _run_job(case)
    held = list(engine.GraphedWaves._cache.values())
    _run_job(case)                                                                   # replays the captured graph
    assert list(engine.GraphedWaves._cache.values()) == held


# ---------------------------------------------------------------------------------------------------------------------
# GPU: feather templates at large blur
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("blur", [1, 2, 3, 31, 63, 64, 65, 127, 128, 255, 256])
@pytest.mark.parametrize("W,H,tw,th,pad,uniform", [(520, 400, 256, 192, 96, False), (100, 90, 64, 64, 16, True)])
def test_feather_templates_at_large_blur(W, H, tw, th, pad, uniform, blur):
    """DevicePlan.mask_pool == tile_mask_window for every tile; on the 100 x 90 canvas with 64-px tiles the ramp of the
    larger blurs is wider than the tile and than the canvas."""
    p = planner.Plan.build(W, H, tw, th, pad, blur, uniform)
    pool = engine.DevicePlan(p, torch.device(DEV)).mask_pool.cpu().numpy()
    for t in p.tiles:
        off, pitch = p._mask_off[t.idx], p._mask_pitch[t.idx]
        got = pool[off: off + pitch * t.eh].reshape(t.eh, pitch)[:, :t.ew]
        assert np.array_equal(got, orc.tile_mask_window(W, H, t.x, t.y, p.tw, p.th, blur, t.region)), (t.idx, blur)
