"""CPU tests of the host side: planner geometry against the reference fixtures, the
C-ABI library (loads, exports every declared symbol, host-side table builders equal the
oracle), schedules and work lists.  No compute calls on a device."""
import json
import os
import re

import numpy as np
import torch
import pytest

import usdu_oracle as orc
from __graft_entry__ import ROOT, load_package

load_package()
from comfyui_distributed_b200 import _native as nat  # noqa: E402
from comfyui_distributed_b200 import planner  # noqa: E402

G = os.path.join(os.path.dirname(__file__), "golden")
GEO = json.load(open(os.path.join(G, "geometry.json")))["cases"]
HEADER = open(os.path.join(ROOT, "include", "usdu_b200.h")).read()


def test_library_exports_every_declared_symbol():
    declared = set(re.findall(r"^\s*(?:int|int64_t|const char\*)\s+(usdu_\w+)\s*\(", HEADER, re.M))
    assert declared, "no declarations parsed from include/usdu_b200.h"
    assert declared == set(nat.EXPORTS)
    lib = nat.lib()
    for name in declared:
        assert hasattr(lib, name)
    assert lib.usdu_abi_version() == int(re.search(r"#define USDU_ABI_VERSION (\d+)", HEADER).group(1))


def test_binding_constants_match_header():
    for cname, val in [("USDU_TILE_WORDS", nat.TILE_WORDS), ("USDU_TAB_HEADER", nat.TAB_HEADER),
                       ("USDU_CROP_ITEM_WORDS", nat.CROP_ITEM_WORDS), ("USDU_BLEND_ITEM_WORDS", nat.BLEND_ITEM_WORDS),
                       ("USDU_COVER_WORDS", nat.COVER_WORDS), ("USDU_MASK_WORDS", nat.MASK_WORDS),
                       ("USDU_BLOCK_W", nat.BLOCK_W), ("USDU_BLOCK_H", nat.BLOCK_H),
                       ("USDU_T_TAB_BLEND_V", nat.T_TAB_BLEND_V), ("USDU_T_SUP_Y1", nat.T_SUP_Y1),
                       ("USDU_T_MASK_PITCH", nat.T_MASK_PITCH)]:
        assert int(re.search(rf"#define {cname} (\d+)", HEADER).group(1)) == val, cname


def test_error_reporting_without_device_or_with_bad_args():
    lib = nat.lib()
    assert lib.usdu_resample_ksize(0, 5) < 0
    assert b"positive" in lib.usdu_last_error()
    with pytest.raises(nat.NativeError):
        nat.quantize_canvas(0, 0, 1, 1, 1, 16, 0)      # null pointers are rejected before any CUDA call
    with pytest.raises(nat.NativeError):
        nat.tile_blend(1, 1, 8, 8, 17, 1, 1, 1, 1, 1, 1, 8, 8, 0, 0, 0, 0)


@pytest.mark.parametrize("n_in,n_out", [(576, 544), (544, 576), (320, 288), (288, 544), (100, 160), (1, 8), (2304, 1152), (37, 64), (544, 64), (160, 100)])
def test_resample_table_equals_oracle(n_in, n_out):
    tab = nat.build_resample_table(n_in, n_out)
    bounds, kk = orc.lanczos_coeffs(n_in, n_out)
    ks = kk.shape[1]
    H = nat.TAB_HEADER
    assert tab[0] == n_in and tab[1] == n_out and tab[2] == ks
    assert np.array_equal(tab[H:H + 2 * n_out].reshape(n_out, 2), bounds)
    assert np.array_equal(tab[H + 2 * n_out:H + 2 * n_out + n_out * ks].reshape(n_out, ks), kk)
    assert tab[3] == bounds[:, 1].max()
    assert tab[4] % 4 == 0 and tab.shape[0] % 4 == 0     # 128-bit loads of packed rows stay aligned in the pool
    if tab[4]:                                           # packed rows: {first, k0..k(stride-2)}, zero padded
        st = int(tab[6])
        assert st == (8 if tab[3] <= 7 else 16) and tab[3] <= 15
        rows = tab[tab[4]:tab[4] + st * n_out].reshape(n_out, st)
        assert np.array_equal(rows[:, 0], bounds[:, 0])
        kpad = kk[:, :st - 1] if ks >= st - 1 else np.pad(kk, ((0, 0), (0, st - 1 - ks)))
        assert np.array_equal(rows[:, 1:], kpad)
        assert not kk[:, st - 1:].any()                  # nothing was cut off
    else:
        assert tab[3] > 15


@pytest.mark.parametrize("filt,name", [(0, "lanczos"), (1, "bicubic")])
@pytest.mark.parametrize("n_in,n_out", [(64, 300), (300, 64), (135, 1080), (576, 544), (7, 63), (960, 7680)])
def test_filter_table_equals_oracle(filt, name, n_in, n_out):
    tab = nat.build_filter_table(filt, n_in, n_out)
    bounds, kk = orc.resample_coeffs(n_in, n_out, name)
    H, ks = nat.TAB_HEADER, kk.shape[1]
    assert (tab[0], tab[1], tab[2]) == (n_in, n_out, ks)
    assert np.array_equal(tab[H:H + 2 * n_out].reshape(n_out, 2), bounds)
    assert np.array_equal(tab[H + 2 * n_out:].reshape(n_out, ks), kk)
    lo, n = nat.table_input_span(tab, n_out // 3, max(1, n_out // 2))
    b = bounds[n_out // 3:n_out // 3 + max(1, n_out // 2)]
    assert lo == b[:, 0].min() and lo + n == (b[:, 0] + b[:, 1]).max()


def test_filter_table_rejects_unknown_filter_and_span_outside_table():
    with pytest.raises(nat.NativeError):
        nat.build_filter_table(7, 10, 20)
    with pytest.raises(nat.NativeError):
        nat.table_input_span(nat.build_filter_table(1, 10, 20), 15, 10)


@pytest.mark.parametrize("n_in,n_out", [(5, 17), (542, 576), (30, 7), (100, 100), (3, 1000), (1, 4)])
def test_nearest_index_equals_oracle(n_in, n_out):
    assert np.array_equal(nat.nearest_index(n_in, n_out), orc.nearest_index(n_in, n_out))


def test_mask_fit_geometry_equals_oracle():
    from comfyui_distributed_b200.conditioning import mask_fit_geometry
    rng = np.random.default_rng(0)
    for _ in range(500):
        cw, ch, pw, ph = (int(v) for v in rng.integers(8, 700, 4))
        assert mask_fit_geometry(cw, ch, pw, ph) == orc.mask_fit_geometry(cw, ch, pw, ph)


def test_identity_table():
    tab = nat.build_identity_table(5)
    assert tab[4] % 4 == 0 and tab.shape[0] % 4 == 0
    rows = tab[tab[4]:].reshape(5, 8)
    assert list(rows[:, 0]) == [0, 1, 2, 3, 4] and (rows[:, 1] == 1 << 22).all() and not rows[:, 2:].any()


def test_box_blur_params_equal_oracle_for_every_radius():
    for r in range(1, 257):
        assert nat.box_blur_params(r) == orc.box_blur_params(r), r


@pytest.mark.parametrize("case", GEO, ids=lambda c: f"{c['W']}x{c['H']}_t{c['tile_w']}x{c['tile_h']}_p{c['padding']}_{'u' if c['uniform'] else 'n'}")
def test_planner_geometry_matches_reference(case):
    p = planner.Plan.build(case["W"], case["H"], case["tile_w"], case["tile_h"], case["padding"], 8, case["uniform"])
    assert (p.tw, p.th) == (case["tw"], case["th"])
    rows = [[t.x, t.y, t.x1, t.y1, t.ew, t.eh, t.pw, t.ph] for t in p.tiles]
    assert rows == case["rows"]


def _windows_overlap(a, b):
    return a.x1 < b.x2 and b.x1 < a.x2 and a.y1 < b.y2 and b.y1 < a.y2


@pytest.mark.parametrize("W,H,tile,pad", [(7680, 4320, 512, 32), (1600, 1200, 512, 32), (1000, 900, 256, 64), (777, 333, 64, 128)])
def test_neighbors_and_waves(W, H, tile, pad):
    p = planner.Plan.build(W, H, tile, tile, pad, 8, True)
    T = len(p.tiles)
    for i in range(T):                                    # neighbour lists == brute force
        brute = sorted(j for j in range(T) if j != i and _windows_overlap(p.tiles[i], p.tiles[j]))
        assert sorted(p.neighbors[i]) == brute
    waves = p.waves()
    assert sorted(t for w in waves for t in w) == list(range(T))
    level = {t: k for k, w in enumerate(waves) for t in w}
    for w in waves:                                       # tiles of a wave are independent
        for a in w:
            assert not any(b in p.neighbors[a] for b in w)
    for i in range(T):                                    # every dependency points to an earlier wave
        for j in p.neighbors[i]:
            if j < i:
                assert level[j] < level[i]
    if (W, H, tile) == (7680, 4320, 512):
        assert len(waves) == 31 and max(len(w) for w in waves) == 8     # SURVEY.md 8e


def test_partitions():
    p = planner.get_plan(7680, 4320, 512, 512, 32, 8, True)
    for world in (1, 2, 4, 8):
        asg = p.partition(world)
        assert sorted(t for a in asg for t in a) == list(range(135))
        assert len(asg) == world
        if world >= 4:
            assert p.conflict_free(asg)
            assert max(map(len, asg)) - min(map(len, asg)) <= 5
    assert not p.conflict_free(p.partition(2))            # two ranks always own neighbours


def test_mask_classes_and_worklists():
    p = planner.get_plan(7680, 4320, 512, 512, 32, 8, True)
    assert p.mask_specs.shape == (9, nat.MASK_WORDS)       # 3 x-classes x 3 y-classes
    # equal class => equal template (checked with the oracle on one representative pair)
    by_class = {}
    for t in p.tiles:
        by_class.setdefault(p.mask_class[t.idx], []).append(t)
    for c, ts in by_class.items():
        a, b = ts[0], ts[-1]
        ma = orc.tile_mask_window(p.W, p.H, a.x, a.y, p.tw, p.th, 8, a.region)
        mb = orc.tile_mask_window(p.W, p.H, b.x, b.y, p.tw, p.th, 8, b.region)
        assert np.array_equal(ma, mb)
        sx0, sy0, sx1, sy1 = p.support(a)                 # alpha is exactly 0 outside the support box
        z = ma.copy()
        z[sy0:sy1, sx0:sx1] = 0
        assert not z.any()
        fx0, fy0, fx1, fy1 = p.opaque_core(a)             # ... and exactly 255 inside the opaque core
        assert fx1 > fx0 and (ma[fy0:fy1, fx0:fx1] == 255).all()
    ids = list(range(135))
    wl, offs, total = p.crop_worklist(ids, 1)
    assert total == 135 * 544 * 544 * 3
    assert p.fast and wl.items.shape == (135 * 5 * 17, nat.JOB_WORDS)              # 128 x 32 fast blocks, job records
    wg, _, _ = p.crop_worklist(ids, 1, use_fast=False)
    assert wg.items.shape == (135 * 9 * 17, nat.CROP_ITEM_WORDS)                    # 64 x 32 generic blocks
    bl = p.blend_worklist(ids, offs, use_fast=False)
    cov = bl.cover.reshape(-1, nat.COVER_WORDS)
    for it in bl.items[::997]:                            # cover lists are ascending in tile id
        c = cov[it[2]: it[2] + it[3], 0]
        assert list(c) == sorted(c)
    # fast job records: heads first, chains cover every (block, tile) pair once, in ascending tile order
    fj = p.blend_worklist(ids, offs)
    J = fj.items
    assert fj.cover is None and fj.n_launch == len({(int(a), int(b)) for a, b in zip(J[:, nat.J_DST_X], J[:, nat.J_DST_Y])})
    seen = np.zeros(J.shape[0], bool)
    for h in range(fj.n_launch):
        i, last = h, -1
        while i >= 0:
            assert not seen[i] and (J[i, nat.J_DST_X], J[i, nat.J_DST_Y]) == (J[h, nat.J_DST_X], J[h, nat.J_DST_Y])
            seen[i] = True
            i = int(J[i, nat.J_NEXT])
    assert seen.all()
    assert (J[:, nat.J_ROWS] <= fj.patch_h).all() and (J[:, nat.J_COLS] <= fj.patch_w).all()
    # every (tile, block) pair with intersecting support is present exactly once
    assert bl.cover.shape[0] == sum(
        ((t.x1 + p.support(t)[2] - 1) // 64 - (t.x1 + p.support(t)[0]) // 64 + 1) *
        ((t.y1 + p.support(t)[3] - 1) // 32 - (t.y1 + p.support(t)[1]) // 32 + 1) for t in p.tiles)


def test_image_batch_divider_matches_reference_chunking():
    import torch
    from comfyui_distributed_b200.nodes import NODE_CLASS_MAPPINGS
    from comfyui_distributed_b200.nodes.utilities import chunk_bounds
    node = NODE_CLASS_MAPPINGS["ImageBatchDivider"]()
    assert chunk_bounds(10, 3) == [(0, 4), (4, 7), (7, 10)] and chunk_bounds(2, 4) == [(0, 1), (1, 2), (2, 2), (2, 2)]
    x = torch.arange(7 * 2 * 2 * 3, dtype=torch.float32).reshape(7, 2, 2, 3)
    outs = node.divide_batch(x, 3)
    assert len(outs) == 10 and [o.shape[0] for o in outs] == [3, 2, 2] + [0] * 7
    assert torch.equal(torch.cat(outs[:3]), x) and outs[0].data_ptr() == x.data_ptr()      # zero-copy views
    assert [o.shape[0] for o in node.divide_batch(x, 99)] == [1, 1, 1, 1, 1, 1, 1, 0, 0, 0]


@pytest.mark.parametrize("use_fast", [True, False])
def test_blend_worklist_shares_cover_the_launch_disjointly(use_fast):
    """part=(i, n): n participants given the same tile list own disjoint sets of canvas blocks whose
    union is the whole launch, with every block's tile list intact (dist.upscale_static shares the
    final blend out like this)."""
    p = planner.Plan.build(2048, 1536, 512, 512, 32, 8, True)
    assert p.fast
    tiles = [t for t in range(len(p.tiles)) if t % 3]
    offs = np.arange(len(tiles), dtype=np.int64) * (1 << 20)
    full = p.blend_worklist(tiles, offs, 1, use_fast)

    def blocks(wl):
        """{(block x, block y): [(tile-specific word, ...) per record in order]}"""
        out = {}
        if use_fast:
            J = wl.items.reshape(-1, nat.JOB_WORDS)
            n_heads = wl.n_launch
            for h in range(n_heads):
                key, chain, i = (int(J[h, nat.J_DST_X]), int(J[h, nat.J_DST_Y])), [], h
                while i >= 0:
                    chain.append((int(J[i, nat.J_SRC_A]), int(J[i, nat.J_SRC_B]), int(J[i, nat.J_OFF_LO])))
                    i = int(J[i, nat.J_NEXT])
                assert key not in out
                out[key] = chain
        else:
            it, cv = wl.items.reshape(-1, nat.BLEND_ITEM_WORDS), wl.cover.reshape(-1, nat.COVER_WORDS)
            for x, y, first, cnt in it:
                out[(int(x), int(y))] = [tuple(int(v) for v in cv[j, :3]) for j in range(first, first + cnt)]
        return out

    want = blocks(full)
    for n in (2, 3, 8):
        got, y_next = {}, 0
        for i in range(n):
            wl = p.blend_worklist(tiles, offs, 1, use_fast, part=(i, n))
            part = blocks(wl)
            assert not (set(part) & set(got))
            got.update(part)
            y0, y1 = wl.rows                                   # the shares are horizontal slabs of whole block rows
            assert y0 == y_next and y1 >= y0 and (y1 % wl.block_rows == 0 or y1 == p.H)
            assert all(y0 <= by < y1 for (_, by) in part)
            y_next = y1
        assert y_next == p.H
        assert got == want
    empty = p.blend_worklist(tiles[:1], offs[:1], 1, use_fast, part=(63, 64))
    assert empty.items.shape[0] in (0, empty.items.shape[0])          # tiny launches may leave a share empty


def test_pinned_pool_never_recycles_a_buffer_somebody_still_sees():
    """engine._PinnedPool hands a result buffer out again only when neither the tensor, nor a view, nor
    a numpy array made from it is alive (page-locked memory is replaced by ordinary memory here)."""
    from comfyui_distributed_b200 import engine

    class Pool(engine._PinnedPool):
        def get(self, shape, dtype=torch.float32):
            import unittest.mock as um
            real_empty = torch.empty
            with um.patch.object(torch, "empty", lambda *a, **k: real_empty(*a, **{x: y for x, y in k.items() if x != "pin_memory"})):
                return super().get(shape, dtype)

    pool = Pool(keep=3)
    a = pool.get((4, 8))
    pa = a.data_ptr()
    assert pool.get((4, 8)).data_ptr() != pa          # `a` is alive
    del a
    b = pool.get((4, 8))
    assert b.data_ptr() == pa                          # dropped -> recycled
    v = b[1]
    del b
    assert pool.get((4, 8)).data_ptr() != pa          # a view is alive
    del v
    c = pool.get((4, 8))
    n = c.numpy()
    pc = c.data_ptr()
    del c
    assert pool.get((4, 8)).data_ptr() != pc          # a numpy array is alive
    del n
    assert pool.get((4, 8)).data_ptr() in (pa, pc)
    for i in range(10):                                 # many shapes: only the most recently used ones keep buffers
        pool.get((3, 5 + i))
    assert len(pool.bufs) == pool.bufs.capacity and ((4, 8), torch.float32) not in pool.bufs


@pytest.mark.parametrize("W,H,tile,pad,blur,uniform", [(7680, 4320, 512, 32, 8, True), (1300, 1100, 256, 32, 16, True),
                                                        (700, 520, 256, 32, 8, False), (333, 777, 64, 128, 40, True),
                                                        (3840, 2160, 512, 32, 8, True), (100, 90, 128, 32, 8, True)])
def test_host_pipeline_bands_are_a_safe_schedule(W, H, tile, pad, blur, uniform):
    """engine.host_bands: the band-by-band order is a topological order of the progressive DAG, a band
    never crops rows that have not been uploaded yet, and rows declared final are never written again."""
    from comfyui_distributed_b200.engine import host_bands
    p = planner.Plan.build(W, H, tile, tile, pad, blur, uniform)
    n_rows = len({t.y for t in p.tiles})
    for n_bands in sorted({1, 2, 3, n_rows, n_rows + 5}):
        bands = host_bands(p, n_bands)
        assert 1 <= len(bands) <= min(n_bands, n_rows)
        order = [t for b in bands for w in p.waves(b["tiles"]) for t in w]
        assert sorted(order) == list(range(len(p.tiles)))
        pos = {t: i for i, t in enumerate(order)}
        for t in range(len(p.tiles)):                  # every earlier overlapping tile of the row-major order comes first
            assert all(pos[n] < pos[t] for n in p.neighbors[t] if n < t), (n_bands, t)
        in_end = fin_end = 0
        for k, b in enumerate(bands):
            assert b["in"][0] == in_end and b["in"][1] >= b["in"][0]
            in_end = b["in"][1]
            assert max(p.tiles[t].y2 for t in b["tiles"]) <= in_end          # crops read uploaded rows only
            assert b["fin"][0] == fin_end and b["fin"][1] >= b["fin"][0]
            fin_end = b["fin"][1]
            later = [t for bb in bands[k + 1:] for t in bb["tiles"]]
            for t in later:                                                     # nobody writes below fin_end any more
                assert p.tiles[t].y1 + p.support(p.tiles[t])[1] >= fin_end
            assert fin_end <= in_end
        assert in_end == H and fin_end == H


def test_table_builders_fuzz_against_oracle():
    """300 random (filter, in, out) axes: the C builders' bounds / coefficients / input spans and the
    NEAREST index arithmetic equal the oracle's restatement of Pillow bit for bit."""
    rng = np.random.default_rng(7)
    for _ in range(300):
        filt = int(rng.integers(0, 2))
        n_in, n_out = int(rng.integers(1, 900)), int(rng.integers(1, 900))
        if n_in / n_out > 40:                 # keep ksize (and the test) small
            continue
        tab = nat.build_filter_table(filt, n_in, n_out)
        bounds, kk = orc.resample_coeffs(n_in, n_out, ("lanczos", "bicubic")[filt])
        H = nat.TAB_HEADER
        assert tab[2] == kk.shape[1]
        assert np.array_equal(tab[H:H + 2 * n_out].reshape(n_out, 2), bounds)
        assert np.array_equal(tab[H + 2 * n_out:].reshape(n_out, kk.shape[1]), kk)
        a = int(rng.integers(0, n_out))
        n = int(rng.integers(1, n_out - a + 1))
        lo, cnt = nat.table_input_span(tab, a, n)
        assert lo == bounds[a:a + n, 0].min() and lo + cnt == (bounds[a:a + n, 0] + bounds[a:a + n, 1]).max()
        assert np.array_equal(nat.nearest_index(n_in, n_out), orc.nearest_index(n_in, n_out))


def test_caches_evict_the_least_recently_used_entry_only():
    """Alternating geometries keep their plans (and, on the device, tables and graphs) warm: the host caches are LRU,
    they never drop everything at once."""
    from comfyui_distributed_b200.lru import LruCache
    c = LruCache(3)
    built = []

    def make(k):
        return c.get_or_build(k, lambda: built.append(k) or ("v", k))

    for k in (1, 2, 3, 1, 4):                      # 4 evicts 2 (1 was touched after it)
        make(k)
    assert built == [1, 2, 3, 4] and list(c.keys()) == [3, 1, 4]
    make(1), make(3)
    assert built == [1, 2, 3, 4]
    make(2)                                        # evicts 4, the least recently used
    assert list(c.keys()) == [1, 3, 2] and len(c) == 3
    # an id()-keyed entry whose object was replaced is rebuilt in place
    assert c.get_or_build(2, lambda: "fresh", valid=lambda v: False) == "fresh" and len(c) == 3
    # the plan cache: two alternating geometries never rebuild
    a = planner.get_plan(640, 480, 128, 128, 16, 8, True)
    for i in range(40):
        planner.get_plan(300 + i, 200, 64, 64, 8, 4, True)
        assert planner.get_plan(640, 480, 128, 128, 16, 8, True) is a
