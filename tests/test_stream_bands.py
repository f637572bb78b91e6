"""Plan.stream_bands: the row bands of the canvas quantise / dequantise passes that run beside the level waves
(engine.CastBands).  Checked on the CPU against the plan's geometry and the kernels' job records, for the sweep cases,
the bench workloads and seeded random geometries: every canvas row a wave's crop or blend bulk-tensor boxes can load
is quantised before that wave starts, no dequantise band starts before the last blend that writes its rows, and the
bands cover every row exactly once."""
import numpy as np
import pytest

from __graft_entry__ import load_package
from inputs import sweep_cases

load_package()
from comfyui_distributed_b200 import _native as nat  # noqa: E402
from comfyui_distributed_b200 import planner  # noqa: E402

# (W, H, tile_w, tile_h, padding, mask_blur, uniform, B): cfg1, cfg2, cfg4, cfg4 alt (8192² / 256), cfg5
BENCH = [(512, 512, 256, 256, 32, 8, True, 1), (7680, 4320, 512, 512, 32, 8, True, 1), (15360, 8640, 256, 256, 32, 8, True, 1),
         (8192, 8192, 256, 256, 32, 8, True, 1), (3840, 2160, 512, 512, 32, 8, True, 17)]
SWEEP = [(W, H, tw, th, pad, blur, uni, B) for (_, _, B, H, W, tw, th, pad, blur, uni) in sweep_cases()]


def _random(seed):
    rng = np.random.default_rng(5000 + seed)
    tw = int(rng.choice([64, 96, 128, 256, 512]))
    return (int(rng.integers(64, 2400)) // 4 * 4, int(rng.integers(64, 1800)), tw, tw, int(rng.choice([0, 8, 16, 32, 64])),
            int(rng.choice([0, 4, 8, 16, 40])), bool(rng.random() < 0.7), int(rng.choice([1, 2])))


CASES = BENCH + SWEEP + [_random(s) for s in range(12)]


def _loads_and_stores(p, wave, B, path):
    """Rows wave `wave` can load (crop boxes, blend blocks) and store (blend blocks), straight from the kernels' records:
    a crop box is usdu_mma.cu's / usdu_fast.cu's 48 / 40 rows from the first staged row (the integer-pipe staging may
    over-read 16 bytes into the next row); a blend block is block_rows rows from its canvas row, loaded and stored whole."""
    cr, offs, _ = p.crop_worklist(wave, B, path)
    bl = p.blend_worklist(wave, offs, 4, path, B)
    load, store = np.zeros(p.H, bool), np.zeros(p.H, bool)
    box = 48 if cr.path == 2 else 40
    for J in cr.items.reshape(-1, nat.JOB_WORDS):
        y0 = int(J[nat.J_SRC_B])
        load[y0:y0 + max(box, int(J[nat.J_ROWS])) + (cr.path == 1)] = True
    for J in bl.items.reshape(-1, nat.JOB_WORDS):
        y0 = int(J[nat.J_DST_Y])
        store[y0:y0 + bl.block_rows] = True
    for t in wave:                                   # the crop window and the mask support, from the tile geometry alone
        tile = p.tiles[t]
        load[tile.y1:tile.y2] = True
        sy0, sy1 = p.support(tile)[1::2]
        assert store[tile.y1 + sy0:tile.y1 + sy1].all() or sy1 <= sy0
    return load | store, store


@pytest.mark.parametrize("path", [1, 2], ids=["fast", "mma"])
@pytest.mark.parametrize("n_bands", [2, 5, 16, 32])
@pytest.mark.parametrize("case", CASES, ids=lambda c: "x".join(map(str, c[:6])) + ("u" if c[6] else "n") + f"b{c[7]}")
def test_bands_gate_every_wave_and_cover_every_row_once(case, n_bands, path):
    W, H, tw, th, pad, blur, uniform, B = case
    p = planner.Plan.build(W, H, tw, th, pad, blur, uniform)
    if p.kernel_path(path == 1 or None) != path:
        pytest.skip("this geometry does not run on these kernels; the cast bands need job-record work lists")
    waves = p.waves()
    q, d = p.stream_bands(None, B, n_bands, path, path)
    for bands in (q, d):
        assert bands[0][0] == 0 and bands[-1][1] == H
        assert all(a[1] == b[0] for a, b in zip(bands, bands[1:])) and all(y0 < y1 for y0, y1, _ in bands)
        assert len(bands) <= n_bands and all(0 <= k < len(waves) for _, _, k in bands)
    q_gate, d_fork = np.empty(H, int), np.empty(H, int)
    for y0, y1, k in q:
        q_gate[y0:y1] = k
    for y0, y1, k in d:
        d_fork[y0:y1] = k
    rows = [_loads_and_stores(p, w, B, path) for w in waves]
    for k, (touch, store) in enumerate(rows):
        assert (q_gate[touch] <= k).all(), f"wave {k} reads a row quantised after it starts"
        assert (d_fork[store] >= k).all(), f"wave {k} writes a row dequantised before its blend"
    touch0 = rows[0][0]
    assert q[0][:2] == (0, int(np.nonzero(touch0)[0].max()) + 1)        # the critical first band: only what wave 0 needs
    assert d[-1][:2] == (int(np.nonzero(rows[-1][1])[0].min()), H)      # ... and the last one: only what the last wave writes
