"""The planner's fast-path job records, interpreted by a numpy model of the kernels (tests/kernel_model.py),
reproduce the oracle: crop + LANCZOS of every tile, and the ordered seam blend (single launch with
overlapping tiles, per-wave launches, partitioned launches).  Checks on a machine WITHOUT a GPU what the
device tests check with one: staging windows, table rows, clip boxes, mask offsets, chain order, addresses."""
import numpy as np
import pytest

import kernel_model as km
import usdu_oracle as orc
from __graft_entry__ import load_package
from inputs import make_input

load_package()
from comfyui_distributed_b200 import _native as nat  # noqa: E402
from comfyui_distributed_b200 import planner  # noqa: E402

CASES = [("noise", 1, 300, 420, 128, 16, 8, True), ("smooth", 2, 260, 300, 128, 32, 16, True),
         ("noise", 1, 200, 232, 96, 16, 8, False), ("checker", 1, 150, 530, 64, 8, 4, True),
         ("noise", 1, 333, 257, 128, 0, 8, True), ("noise", 1, 96, 100, 128, 32, 8, True)]


def _ids(c):
    return f"{c[0]}-b{c[1]}-{c[3]}x{c[2]}-t{c[4]}-p{c[5]}-m{c[6]}-{'u' if c[7] else 'n'}"


MMA_CASES = CASES + [("noise", 1, 320, 480, 256, 32, 8, True), ("noise", 1, 1200, 1600, 512, 32, 8, True),
                     # tensor-core crops staged with LDG (patch > the TMA boxes), one and two k-steps; two-k-step blend
                     ("noise", 1, 500, 700, 128, 48, 8, True), ("noise", 1, 500, 700, 128, 96, 8, True),
                     ("noise", 2, 400, 520, 128, 96, 8, True)]


@pytest.mark.parametrize("path", [1, 2], ids=["fast", "mma"])
@pytest.mark.parametrize("case", MMA_CASES, ids=_ids)
def test_crop_records_reproduce_extract_tile(case, path):
    kind, B, H, W, tile, pad, blur, uniform = case
    p = planner.Plan.build(W, H, tile, tile, pad, blur, uniform)
    if not p.fast or (path == 2 and not p.mma):
        pytest.skip("this geometry runs on the generic kernels" if not p.fast else "no tensor-core path for this geometry")
    canvas = orc.quantize_u8(make_input(kind, 3, B, H, W))
    _, _, oplan = orc.make_plan(W, H, tile, tile, pad, uniform)
    ids = list(range(len(p.tiles)))
    wl, offs, total = p.crop_worklist(ids, B, path)
    assert wl.path == path
    out = np.full(total, -1.0, dtype=np.float32)
    (km.run_crop_mma if path == 2 else km.run_crop)(p, canvas, wl, out)
    for t, o in zip(oplan, offs):
        want = orc.extract_tile(canvas, t)
        got = out[o:o + want.size].reshape(want.shape)
        assert np.array_equal(got, want), t.idx
    assert not (out < 0).any()                       # every element of every tile slot was written exactly by some block


@pytest.mark.parametrize("path", [1, 2], ids=["fast", "mma"])
@pytest.mark.parametrize("src_u8", [False, True])
@pytest.mark.parametrize("case", MMA_CASES, ids=_ids)
def test_blend_records_reproduce_ordered_blend(case, src_u8, path):
    kind, B, H, W, tile, pad, blur, uniform = case
    p = planner.Plan.build(W, H, tile, tile, pad, blur, uniform)
    if not p.fast or (path == 2 and not p.mma):
        pytest.skip("this geometry runs on the generic kernels" if not p.fast else "no tensor-core path for this geometry")
    run_blend = km.run_blend_mma if path == 2 else km.run_blend
    tw, th, oplan = orc.make_plan(W, H, tile, tile, pad, uniform)
    base = orc.quantize_u8(make_input(kind, 4, B, H, W))
    rng = np.random.default_rng(1)
    ids = list(range(len(p.tiles)))
    offs, total = p.slot_offsets(ids, B)
    src = rng.random(total, dtype=np.float32)
    pool = km.mask_pool(p)
    want = base.copy()
    for t, o in zip(oplan, offs):
        proc = src[o:o + B * t.ph * t.pw * 3].reshape(B, t.ph, t.pw, 3)
        m = orc.tile_mask_window(W, H, t.x, t.y, tw, th, blur, (t.x1, t.y1, t.x2, t.y2))
        orc.blend_processed(want, proc, t, m)
    feed = orc.quantize_u8(src) if src_u8 else src
    # (a) ONE launch with every tile in ascending order (the static-mode final blend)
    got = base.copy()
    run_blend(p, got, p.blend_worklist(ids, offs, 1 if src_u8 else 4, path, B), feed, pool)
    assert np.array_equal(got, want)
    # (b) the same launch shared out over 3 participants (dist.upscale_static)
    got = base.copy()
    for i in (2, 0, 1):                               # any order: the shares own disjoint blocks
        run_blend(p, got, p.blend_worklist(ids, offs, 1 if src_u8 else 4, path, B, part=(i, 3)), feed, pool)
    assert np.array_equal(got, want)
    # (c) wave by wave (the progressive driver blends each wave with its own launch)
    got = base.copy()
    pos = {t: i for i, t in enumerate(ids)}
    for wave in p.waves():
        run_blend(p, got, p.blend_worklist(wave, np.array([offs[pos[t]] for t in wave]), 1 if src_u8 else 4, path, B), feed, pool)
    assert np.array_equal(got, want)


def _random_geometry(seed):
    rng = np.random.default_rng(1000 + seed)
    tw = int(rng.choice([64, 96, 128, 192, 256]))
    th = tw if rng.random() < 0.7 else int(rng.choice([64, 96, 128, 192, 256]))
    return (int(rng.integers(40, 700)), int(rng.integers(40, 500)), tw, th, int(rng.choice([0, 8, 16, 32, 48])),
            int(rng.choice([0, 1, 4, 8, 16, 32])), bool(rng.random() < 0.7), int(rng.choice([1, 1, 2])))


@pytest.mark.parametrize("seed", range(13))
def test_random_geometries_records_reproduce_the_oracle(seed):
    """Seeded random canvases / tile sizes / paddings / blurs / uniform or not / 1-2 frames (rectangular tiles, canvases
    smaller than a tile, ramps wider than the padding ...): the records of every kernel family the plan selects, run by
    the numpy model, give the oracle's crops and the oracle's canvas after the ordered blend."""
    W, H, tw, th, pad, blur, uniform, B = _random_geometry(seed)
    p = planner.Plan.build(W, H, tw, th, pad, blur, uniform)
    if not p.fast:
        pytest.skip("generic kernels: covered by the structural test below and on the GPU")
    canvas = orc.quantize_u8(make_input("noise", seed, B, H, W))
    mw, mh, oplan = orc.make_plan(W, H, tw, th, pad, uniform)
    ids = list(range(len(p.tiles)))
    boffs, btotal = p.slot_offsets(ids, B)
    src = np.random.default_rng(seed).random(btotal, dtype=np.float32)
    pool = km.mask_pool(p)
    want = canvas.copy()
    for t, o in zip(oplan, boffs):
        proc = src[o:o + B * t.ph * t.pw * 3].reshape(B, t.ph, t.pw, 3)
        orc.blend_processed(want, proc, t, orc.tile_mask_window(W, H, t.x, t.y, mw, mh, blur, (t.x1, t.y1, t.x2, t.y2)))
    for path in ([1, 2] if p.mma else [1]):
        wl, offs, total = p.crop_worklist(ids, B, path)
        out = np.full(total, -1.0, dtype=np.float32)
        (km.run_crop_mma if path == 2 else km.run_crop)(p, canvas, wl, out)
        for t, o in zip(oplan, offs):
            crop = orc.extract_tile(canvas, t)
            assert np.array_equal(out[o:o + crop.size].reshape(crop.shape), crop), (path, t.idx)
        for src_u8 in (False, True):
            got = canvas.copy()
            (km.run_blend_mma if path == 2 else km.run_blend)(
                p, got, p.blend_worklist(ids, boffs, 1 if src_u8 else 4, path, B), orc.quantize_u8(src) if src_u8 else src, pool)
            assert np.array_equal(got, want), (path, src_u8)


GENERIC = [(48, 64, 512, 32, 8, True), (1021, 37, 64, 8, 8, True), (33, 515, 128, 16, 255, True), (300, 260, 128, 16, 16, False),
           (2304, 96, 1152, 0, 4, True)]


@pytest.mark.parametrize("W,H,tile,pad,blur,uniform", GENERIC)
def test_generic_work_items_cover_every_output_once_and_fit_the_declared_patch(W, H, tile, pad, blur, uniform):
    """The any-scale kernels compute their input windows from the tables themselves; the planner's part is
    the item lists and the shared-memory capacity it declares (patch_w x patch_h).  Crop: the blocks tile
    every output pixel of every tile exactly once and no block needs more input than declared.  Blend: every
    canvas block appears once, lists exactly the tiles whose feather support touches it, in blend order,
    and no (block, tile) pair needs more of the processed tile than declared."""
    p = planner.Plan.build(W, H, tile, tile, pad, blur, uniform)
    ids = list(range(len(p.tiles)))
    H_ = nat.TAB_HEADER

    def span(n_in, n_out, o0, cnt):
        if n_in == n_out:
            return o0, o0 + cnt
        off = p._tab_off[(n_in, n_out)]
        b = p.tabs[off + H_: off + H_ + 2 * n_out].reshape(n_out, 2)
        return int(b[o0, 0]), int(b[o0 + cnt - 1, 0] + b[o0 + cnt - 1, 1])

    wl, offs, total = p.crop_worklist(ids, 1, False)
    bw, bh = wl.block_cols, wl.block_rows
    hit = {t: np.zeros((p.tiles[t].ph, p.tiles[t].pw), dtype=np.int32) for t in ids}
    for tid, ox0, oy0, off_lo, off_hi, rows in wl.items.reshape(-1, nat.CROP_ITEM_WORDS).tolist():
        t = p.tiles[tid]
        ow, oh = min(bw, t.pw - ox0), min(rows, t.ph - oy0)
        assert ow > 0 and oh > 0 and rows <= bh
        hit[tid][oy0:oy0 + oh, ox0:ox0 + ow] += 1
        lo, hi = span(t.ew, t.pw, ox0, ow)
        assert hi - lo <= wl.patch_w, ("crop", tid, hi - lo, wl.patch_w)
        lo, hi = span(t.eh, t.ph, oy0, oh)
        assert hi - lo <= wl.patch_h
        assert (off_lo & 0xFFFFFFFF) | (off_hi << 32) == offs[ids.index(tid)]
    assert all((h == 1).all() for h in hit.values())

    boffs, _ = p.slot_offsets(ids, 1)
    wl = p.blend_worklist(ids, boffs, 4, False, 1)
    bw, bh = wl.block_cols, wl.block_rows
    items, cover = wl.items.reshape(-1, nat.BLEND_ITEM_WORDS), wl.cover.reshape(-1, nat.COVER_WORDS)
    seen = set()
    for bx, by, first, count in items.tolist():
        assert (bx, by) not in seen and bx % bw == 0 and by % bh == 0
        seen.add((bx, by))
        listed = [int(cover[j, 0]) for j in range(first, first + count)]
        assert listed == sorted(listed)                                   # blend order of this launch = ascending id
        want = []
        for t in p.tiles:
            sx0, sy0, sx1, sy1 = p.support(t)
            X0, Y0, X1, Y1 = t.x1 + sx0, t.y1 + sy0, t.x1 + sx1, t.y1 + sy1
            if X1 > X0 and Y1 > Y0 and X0 < bx + bw and X1 > bx and Y0 < by + bh and Y1 > by:
                want.append(t.idx)
                cx0, cx1 = max(bx, X0) - t.x1, min(bx + bw, X1) - t.x1    # outputs of the back-resize this block needs
                lo, hi = span(t.pw, t.ew, cx0, cx1 - cx0)
                assert hi - lo <= wl.patch_w, ("blend", t.idx, hi - lo, wl.patch_w)
                cy0, cy1 = max(by, Y0) - t.y1, min(by + bh, Y1) - t.y1
                lo, hi = span(t.ph, t.eh, cy0, cy1 - cy0)
                assert hi - lo <= wl.patch_h
        assert listed == want, (bx, by)
        for j in range(first, first + count):
            assert (int(cover[j, 1]) & 0xFFFFFFFF) | (int(cover[j, 2]) << 32) == boffs[int(cover[j, 0])]


@pytest.mark.parametrize("W,H,tile,pad,blur,B,extreme,path", [
    (1100, 900, 256, 32, 16, 1, "early_first", 2), (700, 560, 128, 16, 8, 2, "early_first", 2),
    (700, 560, 128, 16, 8, 2, "early_last", 2), (640, 512, 128, 16, 8, 1, "early_first", 1)])
#   (2300 x 1500 / 512, both orders: checked once, 3 min)
def test_split_levels_give_the_sequential_result_in_every_legal_order(W, H, tile, pad, blur, B, extreme, path):
    """engine.run_split launches, per dependency wave, crop_early / crop_late and one blend (planner.split_level) on two
    streams.  The numpy model executes the same lists SEQUENTIALLY in the two extreme placements the stream dependencies
    allow the early crops of wave k+1 -- before ANY blend of wave k, or right before the sampler of wave k+1 needs them --
    and must reproduce the oracle's process_single (tile after tile) bit for bit: the split only reorders work that does
    not interact."""
    p = planner.Plan.build(W, H, tile, tile, pad, blur, True)
    if not (p.mma if path == 2 else p.fast):
        pytest.skip("no job-record path")
    run_crop, run_blend = (km.run_crop_mma, km.run_blend_mma) if path == 2 else (km.run_crop, km.run_blend)
    img = make_input("noise", 3, B, H, W)
    den = orc.make_t0_denoiser(5, 0.5)
    want = orc.process_single(img, den, tile, tile, pad, blur, True)
    _, _, oplan = orc.make_plan(W, H, tile, tile, pad, True)
    canvas = orc.quantize_u8(img)
    pool = km.mask_pool(p)
    waves = [sorted(w, key=lambda i: (p.tiles[i].ph, p.tiles[i].pw, i)) for w in p.waves()]
    assert len(waves) > 2
    L = []
    for k, w in enumerate(waves):
        offs, _ = p.slot_offsets(w, B)
        cr, coffs, ctotal, late, blend = p.split_level(w, offs, waves[k - 1] if k else None, B, path)
        assert np.array_equal(coffs, offs)
        early = lt = None
        if late is not None and late.any() and not late.all():
            early, lt = p.sub_worklist(cr, ~late), p.sub_worklist(cr, late)
        L.append(dict(crop=cr, early=early, late=lt, total=ctotal, offs=offs, blend=blend))
    assert any(e["early"] is not None for e in L)

    def sample(k, buf):
        out = np.empty_like(buf)
        for tid, o in zip(waves[k], L[k]["offs"]):
            t = oplan[tid]
            n = B * t.ph * t.pw * 3
            out[o:o + n] = den(buf[o:o + n].reshape(B, t.ph, t.pw, 3), t).ravel()
        return out

    bufs = {0: np.full(L[0]["total"], -1.0, np.float32)}
    early_pending = {}
    for k in range(len(waves)):
        e = L[k]
        if e["late"] is not None:
            if k in early_pending:                                # "early last": right before the sampler needs it
                run_crop(p, canvas, early_pending.pop(k), bufs[k])
            run_crop(p, canvas, e["late"], bufs[k])
        else:
            run_crop(p, canvas, e["crop"], bufs[k])
        assert not (bufs[k] < 0).any()
        out = sample(k, bufs[k])
        if k + 1 < len(waves):
            bufs[k + 1] = np.full(L[k + 1]["total"], -1.0, np.float32)
            if L[k + 1]["early"] is not None:
                if extreme == "early_first":                      # before any blend of wave k
                    run_crop(p, canvas, L[k + 1]["early"], bufs[k + 1])
                else:
                    early_pending[k + 1] = L[k + 1]["early"]
        run_blend(p, canvas, e["blend"], out, pool)
        del bufs[k]
    assert np.array_equal(orc.dequantize_u8(canvas), want)
