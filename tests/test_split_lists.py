"""Plan.split_lists (usdu_plan_split_worklists): the work lists engine.run_split launches per dependency wave, each sized
for its role -- late crop jobs on the chain in short blocks, early crop jobs beside the previous wave in tall blocks, the
blend at the block height of the residency model.  CPU only: every output of a wave is cropped exactly once, no early
job reads a pixel the previous wave's blend changes, the library equals a numpy restatement built from
tests/planner_model.py, the cast bands gate the rows of the launched lists, and the kernel model runs the lists in both
extreme interleavings the streams allow to the sequential result."""
import numpy as np
import pytest

import kernel_model as km
import planner_model as pm
import usdu_oracle as orc
from __graft_entry__ import load_package
from inputs import make_input

load_package()
from comfyui_distributed_b200 import _native as nat  # noqa: E402
from comfyui_distributed_b200 import planner  # noqa: E402

# (W, H, tile, padding, blur, B): cfg1, cfg2, cfg5, then smaller geometries with two k-steps, odd supports and batches
CASES = [(512, 512, 256, 32, 8, 1), (7680, 4320, 512, 32, 8, 1), (3840, 2160, 512, 32, 8, 17), (1100, 900, 256, 32, 16, 1),
         (700, 560, 128, 16, 8, 2), (700, 500, 1024, 32, 8, 1), (1500, 900, 256, 256, 255, 5), (640, 480, 128, 0, 0, 1)]
SMS = 132


def _ids(c):
    return "x".join(map(str, c))


def _waves(p):
    return [sorted(w, key=lambda t: (p.tiles[t].ph, p.tiles[t].pw, t)) for w in p.waves()]


def _slot(J):
    return (J[:, nat.J_OFF_LO].astype(np.int64) & 0xFFFFFFFF) | (J[:, nat.J_OFF_HI].astype(np.int64) << 32)


@pytest.fixture
def sms(monkeypatch):
    monkeypatch.setattr(planner.Plan, "_launch_model", staticmethod(lambda: (SMS, 0)))
    monkeypatch.setattr(pm.Plan, "resident_slots", classmethod(lambda cls: SMS * pm.Plan.CTAS_PER_SM))
    monkeypatch.delenv("USDU_MMA_BH", raising=False)


@pytest.mark.parametrize("path", [1, 2], ids=["fast", "mma"])
@pytest.mark.parametrize("case", CASES, ids=_ids)
def test_every_output_is_cropped_once_and_early_jobs_read_nothing_the_previous_wave_changes(case, path, sms):
    W, H, tile, pad, blur, B = case
    p = planner.Plan.build(W, H, tile, tile, pad, blur, True)
    if p.kernel_path(path == 1 or None) != path:
        pytest.skip("no job records on this path")
    waves = _waves(p)
    for k, w in enumerate(waves):
        offs, total = p.slot_offsets(w, B)
        chain, side, coffs, ctotal, _ = p.split_lists(w, offs, waves[k - 1] if k else None, B, path)
        assert np.array_equal(coffs, offs) and ctotal == total
        hits = np.zeros(total // (3 * B), np.int32)            # per output pixel of the wave's packed tiles
        for wl in [chain] + ([side] if side is not None else []):
            assert wl.path == path and wl.items.shape[1] == nat.JOB_WORDS
            J = wl.items.astype(np.int64)
            for s, ox, oy, pw, rows, cols in zip((_slot(J) // (3 * B)).tolist(), J[:, nat.J_DST_X].tolist(),
                                                 J[:, nat.J_DST_Y].tolist(), J[:, nat.J_N_OUT_H].tolist(),
                                                 J[:, nat.J_ROWS_OUT].tolist(), J[:, nat.J_COLS_OUT].tolist()):
                for y in range(oy, oy + rows):
                    hits[s + y * pw + ox:s + y * pw + ox + cols] += 1
        assert (hits == 1).all(), (k, np.unique(hits))
        if k == 0:
            assert side is None
        if side is not None:
            assert not p.crop_split(side, waves[k - 1]).any()
            if path == 2:                                      # the chain runs short blocks only
                assert (chain.items[:, nat.J_CY1] == 16).all()


def _model_split(m, wave, offs, prev, B, path, monkeypatch):
    """The numpy restatement of usdu_plan_split_worklists on tests/planner_model.py's work lists."""
    def crop(bh):
        monkeypatch.setenv("USDU_MMA_BH", str(bh)) if bh else monkeypatch.delenv("USDU_MMA_BH", raising=False)
        return m.crop_worklist(wave, B, path)

    short, _, _ = crop(16 if path == 2 else 0)
    tall = crop(32)[0] if path == 2 else short
    JS, JT = short.items.reshape(-1, nat.JOB_WORDS), tall.items.reshape(-1, nat.JOB_WORDS)
    outs = lambda J: J[:, nat.J_ROWS_OUT].astype(np.int64) * J[:, nat.J_COLS_OUT]
    all_out = int(outs(JS).sum())
    late, early = [], []
    if not prev:
        late = [(short, j) for j in range(len(JS))]
    else:
        ls, lt = m.crop_split(short, prev), m.crop_split(tall, prev)
        key = {(s, x, y): j for j, (s, x, y) in enumerate(zip(_slot(JS).tolist(), JS[:, nat.J_OX_BASE].tolist(),
                                                                JS[:, nat.J_OY_BASE].tolist()))}
        for j, (s, x, y, n) in enumerate(zip(_slot(JT).tolist(), JT[:, nat.J_OX_BASE].tolist(), JT[:, nat.J_OY_BASE].tolist(),
                                             JT[:, nat.J_ROWS_OUT].tolist())):
            if not lt[j]:
                early.append((tall, j))
                continue
            for q in sorted(i for (s2, x2, y2), i in key.items() if s2 == s and x2 == x and y <= y2 < y + n):
                (late if ls[q] else early).append((short, q))

    def take(pick, shape):
        J = np.array([wl.items.reshape(-1, nat.JOB_WORDS)[j] for wl, j in pick], np.int32).reshape(-1, nat.JOB_WORDS)
        pw, ph = shape.patch_w, shape.patch_h
        for wl in {id(wl): wl for wl, _ in pick}.values():
            pw = max(pw, wl.patch_w)
            if path == 2:
                ph = max(ph & 0xFFFF, wl.patch_h & 0xFFFF) | max(ph >> 16, wl.patch_h >> 16) << 16
            else:
                ph = max(ph, wl.patch_h)
        ks2 = path == 2 and bool(((J[:, nat.J_TAPS_H] > 1) | (J[:, nat.J_TAPS_V] > 1)).any())
        return J, pw, ph, int(shape.algo_bytes * int(outs(J).sum()) / max(all_out, 1)), ks2

    if path != 2:
        monkeypatch.delenv("USDU_MMA_BH", raising=False)
        blend = m.blend_worklist(wave, offs, 4, path, B)
    else:
        best = None
        for bh in (32, 16):
            monkeypatch.setenv("USDU_MMA_BH", str(bh))
            bl = m.blend_worklist(wave, offs, 4, path, B)
            if bl.n_launch <= 0:
                best = (0, bl)
                break
            per_sm = nat.resident_ctas(nat.KERNEL_BLEND, bl.ks2, bl.patch_w, bl.patch_h, bh, False)
            cost = -(-bl.n_launch * B // (SMS * max(per_sm, 1))) * ((bl.patch_h & 0xFFFF) + bh)
            if best is None or cost < best[0]:
                best = (cost, bl)
        blend = best[1]
    monkeypatch.delenv("USDU_MMA_BH", raising=False)
    return take(late, short), take(early, tall), blend


@pytest.mark.parametrize("path", [1, 2], ids=["fast", "mma"])
@pytest.mark.parametrize("case", [c for c in CASES if c[0] * c[1] <= 4_000_000], ids=_ids)
def test_library_split_lists_equal_the_numpy_model(case, path, sms, monkeypatch):
    W, H, tile, pad, blur, B = case
    p, m = planner.Plan.build(W, H, tile, tile, pad, blur, True), pm.Plan.build(W, H, tile, tile, pad, blur, True)
    if p.kernel_path(path == 1 or None) != path:
        pytest.skip("no job records on this path")
    waves = _waves(p)
    for k, w in enumerate(waves[:6]):
        offs, _ = m.slot_offsets(w, B)
        prev = waves[k - 1] if k else None
        late, early, blend = p._native.split_worklists(w, offs, prev or [], B, path, SMS)
        want_late, want_early, want_blend = _model_split(m, w, offs, prev, B, path, monkeypatch)
        for got, want in ((late, want_late), (early, want_early)):
            info = got["info"]
            assert np.array_equal(got["items"].reshape(-1, nat.JOB_WORDS), want[0]), k
            assert (info[nat.WL_PATCH_W], info[nat.WL_PATCH_H], info[nat.WL_ALGO_BYTES], bool(info[nat.WL_KS2])) == want[1:], k
        bl = p._worklist(blend, True)
        assert np.array_equal(bl.items, want_blend.items) and bl.block_rows == want_blend.block_rows, k
        assert (bl.patch_w, bl.patch_h, bl.n_launch, bl.ks2) == (want_blend.patch_w, want_blend.patch_h, want_blend.n_launch,
                                                                 want_blend.ks2), k


def test_the_residency_table_follows_the_launch_bounds():
    """Without a device: 3 CTAs per SM for the 80-register builds, 4 for the large crop, fewer when shared memory binds."""
    assert nat.resident_ctas(nat.KERNEL_BLEND, False, 140, 40 | 40 << 16, 32, False) == 3
    assert nat.resident_ctas(nat.KERNEL_CROP_TMA, False, 148, 48 | 48 << 16, 0, False) == 3
    assert nat.resident_ctas(nat.KERNEL_CROP_TMA | nat.KERNEL_LARGE, False, 148, 48 | 48 << 16, 0, False) == 4
    assert nat.resident_ctas(nat.KERNEL_CROP_TMA | nat.KERNEL_LARGE, True, 148, 48 | 48 << 16, 0, False) == 3
    assert nat.resident_ctas(nat.KERNEL_CROP_LDG, False, 600, 200 | 200 << 16, 0, False) in (0, 1)
    with pytest.raises(nat.NativeError):
        nat.resident_ctas(7, False, 148, 48 | 48 << 16, 0, False)


@pytest.mark.parametrize("case", CASES[1:4], ids=_ids)
def test_cast_bands_gate_the_rows_of_the_launched_lists(case, sms):
    """engine.CastBands passes the lists run_split launches: every row a launched crop box (tall early boxes included)
    or blend block loads is quantised before its wave starts, and no row is dequantised before its last blend."""
    W, H, tile, pad, blur, B = case
    p = planner.Plan.build(W, H, tile, tile, pad, blur, True)
    waves = _waves(p)
    levels = []
    for k, w in enumerate(waves):
        offs, _ = p.slot_offsets(w, B)
        chain, side, _, _, bl = p.split_lists(w, offs, waves[k - 1] if k else None, B, 2)
        levels.append(([chain] + ([side] if side is not None else []), bl))
    q, d = p.stream_bands(None, B, 16, levels=levels)
    q_gate, d_fork = np.empty(H, int), np.empty(H, int)
    for y0, y1, k in q:
        q_gate[y0:y1] = k
    for y0, y1, k in d:
        d_fork[y0:y1] = k
    for k, (crops, bl) in enumerate(levels):
        load, store = np.zeros(H, bool), np.zeros(H, bool)
        for cr in crops:
            for J in cr.items:
                load[J[nat.J_SRC_B]:J[nat.J_SRC_B] + max(48, int(J[nat.J_ROWS]))] = True
        for J in bl.items.reshape(-1, nat.JOB_WORDS):
            store[J[nat.J_DST_Y]:J[nat.J_DST_Y] + bl.block_rows] = True
        assert (q_gate[load | store] <= k).all(), f"wave {k} reads a row quantised after it starts"
        assert (d_fork[store] >= k).all(), f"wave {k} writes a row dequantised before its blend"


@pytest.mark.parametrize("W,H,tile,pad,blur,B,extreme,path", [
    (1100, 900, 256, 32, 16, 1, "early_first", 2), (700, 560, 128, 16, 8, 2, "early_last", 2),
    (640, 512, 128, 16, 8, 1, "early_first", 1)])
def test_split_lists_give_the_sequential_result_in_every_legal_order(W, H, tile, pad, blur, B, extreme, path, sms):
    """The kernel model runs each wave's lists sequentially with the early crops of wave k+1 placed at either end of
    what the streams allow -- before any blend of wave k, or right before the sampler of wave k+1 -- and must give the
    oracle's tile-after-tile result bit for bit."""
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
    waves = _waves(p)
    L = []
    for k, w in enumerate(waves):
        offs, total = p.slot_offsets(w, B)
        chain, side, _, _, bl = p.split_lists(w, offs, waves[k - 1] if k else None, B, path)
        L.append(dict(chain=chain, side=side, total=total, offs=offs, blend=bl))
    assert any(e["side"] is not None for e in L)

    def sample(k, buf):
        out = np.empty_like(buf)
        for tid, o in zip(waves[k], L[k]["offs"]):
            t = oplan[tid]
            n = B * t.ph * t.pw * 3
            out[o:o + n] = den(buf[o:o + n].reshape(B, t.ph, t.pw, 3), t).ravel()
        return out

    bufs = {0: np.full(L[0]["total"], -1.0, np.float32)}
    pending = {}
    for k in range(len(waves)):
        if k in pending:                                          # "early last": right before the sampler needs it
            run_crop(p, canvas, pending.pop(k), bufs[k])
        run_crop(p, canvas, L[k]["chain"], bufs[k])
        assert not (bufs[k] < 0).any()
        out = sample(k, bufs[k])
        if k + 1 < len(waves):
            bufs[k + 1] = np.full(L[k + 1]["total"], -1.0, np.float32)
            if L[k + 1]["side"] is not None:
                if extreme == "early_first":                      # before any blend of wave k
                    run_crop(p, canvas, L[k + 1]["side"], bufs[k + 1])
                else:
                    pending[k + 1] = L[k + 1]["side"]
        run_blend(p, canvas, L[k]["blend"], out, pool)
        del bufs[k]
    assert np.array_equal(orc.dequantize_u8(canvas), want)
