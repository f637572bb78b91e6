"""Batches past 2^31 elements and at the 65,535-frame grid limit, on the host: the planner in libusdu_b200.so against
tests/planner_model.py for B = 102 (the smallest multiple of 17 whose 4K fp32 image passes 2^31 elements), 187 (a 4K u8
canvas past 2^32 bytes) and 65,535 (one frame per grid.y index), and the batch refusals of the node and the engine.
These pin down, without a device, the addresses tests/test_gpu_large_batch.py relies on."""
import numpy as np
import pytest
import torch

import planner_model as pm
from __graft_entry__ import load_package

load_package()
from comfyui_distributed_b200 import _native as nat  # noqa: E402
from comfyui_distributed_b200 import engine, planner  # noqa: E402
from comfyui_distributed_b200.nodes import UltimateSDUpscaleDistributed  # noqa: E402
from comfyui_distributed_b200.testing import T0Model  # noqa: E402

GEOMETRIES = {  # name: (W, H, tile, padding, blur)
    "cfg5": (3840, 2160, 512, 32, 8),
    "tiny": (64, 48, 64, 8, 8),
    "tiny2": (128, 48, 64, 8, 8),
}
BATCHES = (102, 187, 65535)
WL_FIELDS = ("patch_w", "patch_h", "algo_bytes", "n_launch", "block_rows", "block_cols", "rows", "path", "ks2")


@pytest.fixture
def launch_model(monkeypatch):
    """Both planners get the same block-height model inputs (as in test_native_planner.py)."""
    monkeypatch.setattr(pm.Plan, "resident_slots", classmethod(lambda cls: 132 * pm.Plan.CTAS_PER_SM))
    monkeypatch.setattr(planner.Plan, "_launch_model", staticmethod(lambda: (132, 0)))
    monkeypatch.delenv("USDU_MMA_BH", raising=False)


def _same_worklist(got, want, what):
    assert got.items.dtype == want.items.dtype == np.int32, what
    assert got.items.shape == want.items.shape and np.array_equal(got.items, want.items), what
    assert (got.cover is None) == (want.cover is None), what
    if want.cover is not None:
        assert np.array_equal(got.cover, want.cover), what
    assert {f: getattr(got, f) for f in WL_FIELDS} == {f: getattr(want, f) for f in WL_FIELDS}, what


def _i64(items, lo):
    return items[:, lo].astype(np.int64) & 0xFFFFFFFF | items[:, lo + 1].astype(np.int64) << 32


def _check_crop_jobs(wl, p, ids, offs, B, total):
    """Job records (fast and tensor-core crop): J_OFF is the tile's slot, J_FRAME one frame of it, and the last frame's
    last row ends inside the slot."""
    if wl.path == 0:
        it = wl.items.astype(np.int64)
        off = it[:, 3] & 0xFFFFFFFF | it[:, 4] << 32
        slots = dict(zip(ids, (int(o) for o in offs)))
        assert all(int(o) == slots[int(t)] for t, o in zip(it[:, 0], off))
        return
    off, frame = _i64(wl.items, nat.J_OFF_LO), _i64(wl.items, nat.J_FRAME_LO)
    sizes = {int(o): 3 * p.tiles[t].pw * p.tiles[t].ph for t, o in zip(ids, offs)}
    assert all(int(o) in sizes and sizes[int(o)] == int(f) for o, f in zip(off, frame))
    it = wl.items.astype(np.int64)
    end = (off + (B - 1) * frame + (it[:, nat.J_DST_Y] + it[:, nat.J_ROWS_OUT] - 1) * it[:, nat.J_PITCH]
           + 3 * (it[:, nat.J_DST_X] + it[:, nat.J_COLS_OUT] // 3))
    assert (end <= total).all() and (end > total - frame.max()).any()


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("geo", list(GEOMETRIES))
def test_large_batch_lists_equal_the_numpy_model(geo, B, launch_model):
    W, H, tile, pad, blur = GEOMETRIES[geo]
    p, m = planner.Plan.build(W, H, tile, tile, pad, blur, True), pm.Plan.build(W, H, tile, tile, pad, blur, True)
    T = len(p.tiles)
    waves = [sorted(w, key=lambda t: (m.tiles[t].ph, m.tiles[t].pw, t)) for w in m.waves()]
    lists = [list(range(T)), sorted({0, T - 1})] + waves[:3]
    big_offsets = want_big = 0
    for k, ids in enumerate(lists):
        offs, total = p.slot_offsets(ids, B)
        moffs, mtotal = m.slot_offsets(ids, B)
        assert np.array_equal(offs, moffs) and total == mtotal
        assert total == B * sum(3 * p.tiles[t].pw * p.tiles[t].ph for t in ids)
        for path in (0, 1, 2):
            got, goffs, gtotal = p.crop_worklist(ids, B, path)
            want, woffs, wtotal = m.crop_worklist(ids, B, path)
            _same_worklist(got, want, (geo, B, "crop", path, k))
            assert np.array_equal(goffs, offs) and np.array_equal(woffs, offs) and gtotal == wtotal == total
            _check_crop_jobs(got, p, ids, offs, B, total)
            if got.path:
                big_offsets += int((_i64(got.items, nat.J_OFF_LO) >= 1 << 32).sum())
                want_big += int(path > 0 and (offs >= 1 << 32).any())
            # blend sources: the crop's own slots, then the same slots behind 2^32 + 2^31 elements of other data
            for base in (0, (3 << 31) + 16):
                for src_bytes in (4, 1):
                    _same_worklist(p.blend_worklist(ids, offs + base, src_bytes, path, B),
                                   m.blend_worklist(ids, offs + base, src_bytes, path, B), (geo, B, "blend", path, k, base))
                if got.path and base:
                    bl = p.blend_worklist(ids, offs + base, 4, path, B)
                    src = _i64(bl.items, nat.J_SRC_A)
                    assert (src >= base).all() and (src + (B - 1) * _i64(bl.items, nat.J_FRAME_LO) < base + total).all()
        if k >= 2:
            prev = lists[k - 1] if k > 2 else None
            for path in (1, 2):
                got, want = p.split_level(ids, offs, prev, B, path), m.split_level(ids, offs, prev, B, path)
                _same_worklist(got[0], want[0], (geo, B, "split crop", k))
                assert np.array_equal(got[1], want[1]) and got[2] == want[2]
                assert (got[3] is None) == (want[3] is None) and (got[3] is None or np.array_equal(got[3], want[3]))
                _same_worklist(got[4], want[4], (geo, B, "split blend", k))
    assert (big_offsets > 0) == (want_big > 0)               # J_OFF words above 2^32 wherever a slot starts there
    if geo == "cfg5" and B >= 187:
        assert want_big > 0


@pytest.mark.parametrize("B", BATCHES + (188,))
@pytest.mark.parametrize("H,W", [(2160, 3840), (2160, 3838), (48, 64)])
def test_canvas_bytes_at_large_batches(B, H, W):
    pitch = (3 * W + 127) // 128 * 128
    assert nat.canvas_bytes(B, H, W) == B * H * pitch + nat.CANVAS_SLACK
    assert engine.Canvas.pitch_of(W) == pitch
    if (B, H, W) == (188, 2160, 3840):
        assert nat.canvas_bytes(B, H, W) > 1 << 32


# ---------------------------------------------------------------------------------------------------------------------
# more than 65,535 frames is refused before any device work
# ---------------------------------------------------------------------------------------------------------------------
def _node_args(img, **hidden):
    return (img, T0Model(), None, None, None, 123, 20, 8.0, "euler", "normal", 0.5, 64, 64, 8, 8, True, False), hidden


@pytest.mark.parametrize("B", [65537, 65541, 100001])
def test_node_refuses_more_than_65535_frames_as_master(B):
    args, hidden = _node_args(torch.zeros(B, 1, 1, 3))
    with pytest.raises(ValueError, match="65535"):
        UltimateSDUpscaleDistributed().run(*args, **hidden)


@pytest.mark.parametrize("B", [65536, 65537, 70000])
def test_node_refuses_more_than_65535_frames_as_worker(B):
    args, hidden = _node_args(torch.zeros(B, 1, 1, 3), multi_job_id="job", is_worker=True,
                              master_url="http://127.0.0.1:9", worker_id="w1")
    with pytest.raises(ValueError, match="65535"):
        UltimateSDUpscaleDistributed().run(*args, **hidden)


def test_node_still_refuses_other_batch_sizes_first():
    args, hidden = _node_args(torch.zeros(65536, 1, 1, 3))
    with pytest.raises(ValueError, match="4n\\+1"):
        UltimateSDUpscaleDistributed().run(*args, **hidden)


def test_engine_refuses_more_than_65535_frames():
    from comfyui_distributed_b200.denoise import T0Denoiser
    img = torch.zeros(65536, 1, 1, 3)
    with pytest.raises(ValueError, match="65535"):
        engine.upscale_single(img, T0Denoiser(1, 0.5), 64, 64, 8, 8, True)      # a host tensor: refused before the CUDA check
    with pytest.raises(ValueError, match="65535"):
        engine.upscale_host(img, T0Denoiser(1, 0.5), 64, 64, 8, 8, True)
    engine.check_batch(engine.MAX_BATCH)
    assert engine.MAX_BATCH == 65535
