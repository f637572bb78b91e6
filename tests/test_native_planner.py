"""The planner in libusdu_b200.so (usdu_plan_* / usdu_worklist_*) against tests/planner_model.py, the numpy planner it
replaced: tile geometry, descriptors, the table pool with its fragment sections, mask specs, overlap lists, waves and
every field of the crop and blend work lists of all three kernel families, byte for byte.  CPU only: the block-height
model gets its SM count from the caller, so plans are the same with or without a device."""
import ctypes
import dataclasses
import json
import os

import numpy as np
import pytest

import planner_model as pm
from __graft_entry__ import load_package
from inputs import STATIC_REF_CASES, sweep_cases

load_package()
from comfyui_distributed_b200 import _native as nat  # noqa: E402
from comfyui_distributed_b200 import planner  # noqa: E402

G = os.path.join(os.path.dirname(__file__), "golden")
BENCH = {  # name: (B, H, W, tile, padding, blur) -- bench.py's workloads and the 8192^2 alternative
    "cfg1": (1, 512, 512, 256, 32, 8), "cfg2": (1, 4320, 7680, 512, 32, 8), "cfg4": (1, 8640, 15360, 256, 32, 8),
    "cfg4alt": (1, 8192, 8192, 256, 32, 8), "cfg5": (17, 2160, 3840, 512, 32, 8)}
WL_FIELDS = ("patch_w", "patch_h", "algo_bytes", "n_launch", "block_rows", "block_cols", "rows", "path", "ks2")


def _random_cases():
    """Seeded geometries, then the corners the kernels care about spelled out."""
    rng = np.random.default_rng(20261016)
    out = []
    for i in range(24):
        tw = int(rng.choice([64, 72, 96, 128, 200, 256, 512, 1024, 2048]))
        th = tw if rng.random() < 0.6 else int(rng.choice([64, 80, 128, 256, 384, 2048]))
        out.append((f"rnd{i}", int(rng.integers(16, 2600)), int(rng.integers(16, 1800)), tw, th,
                    int(rng.choice([0, 8, 16, 32, 64, 256])), int(rng.choice([0, 1, 4, 8, 16, 97, 255])), bool(rng.random() < 0.6),
                    int(rng.choice([1, 2, 5, 17]))))
    out += [
        ("nonuniform_odd_w", 1021, 700, 256, 200, 24, 8, False, 1),
        ("w_not_mult4", 1003, 517, 128, 128, 16, 8, True, 5),
        ("canvas_lt_tile_15taps", 48, 64, 512, 512, 32, 8, True, 1),       # 544 -> 48: far more than 15 taps
        ("canvas_lt_tile_flat", 1021, 37, 64, 64, 8, 8, True, 17),
        ("two_ksteps", 700, 500, 1024, 1024, 32, 8, True, 1),              # down-scales by ~1.5: two k-steps
        ("two_ksteps_nonuniform", 900, 300, 2048, 2048, 0, 4, False, 1),
        ("blur0_pad0", 640, 480, 128, 128, 0, 0, True, 1),
        ("blur255_pad256", 1500, 900, 256, 256, 256, 255, True, 5),
        ("tile2048", 4100, 2300, 2048, 2048, 64, 16, True, 1),
        ("banker_rounding", 640, 640, 500, 508, 24, 8, True, 1),
        ("tiny", 17, 9, 64, 64, 8, 8, True, 1),
    ]
    return out


def _cases():
    out = [(f"sweep{c[0]}", c[4], c[3], c[5], c[6], c[7], c[8], c[9], c[2]) for c in sweep_cases()]
    for c in json.load(open(os.path.join(G, "geometry.json")))["cases"]:
        out.append((f"geo_{c['W']}x{c['H']}_t{c['tile_w']}x{c['tile_h']}_p{c['padding']}_{'u' if c['uniform'] else 'n'}",
                    c["W"], c["H"], c["tile_w"], c["tile_h"], c["padding"], 8, c["uniform"], 1))
    for c in STATIC_REF_CASES:
        out.append((f"static_{c[0]}", c[5], c[4], c[6], c[6], c[7], c[8], c[9], c[3]))
    for name, (B, H, W, tile, pad, blur) in BENCH.items():
        out.append((name, W, H, tile, tile, pad, blur, True, B))
    return out + _random_cases()


CASES = _cases()


@pytest.fixture
def launch_model(monkeypatch):
    """Give both planners the same block-height model inputs: an SM count and an optional forced tensor-core block
    height (the library takes them as arguments, the model reads the device and USDU_MMA_BH)."""
    def set_model(sms, forced=0):
        monkeypatch.setattr(pm.Plan, "resident_slots", classmethod(lambda cls: sms * pm.Plan.CTAS_PER_SM))
        monkeypatch.setattr(planner.Plan, "_launch_model", staticmethod(lambda: (sms, forced)))
        if forced:
            monkeypatch.setenv("USDU_MMA_BH", str(forced))
        else:
            monkeypatch.delenv("USDU_MMA_BH", raising=False)
    return set_model


def _same_worklist(got, want, what):
    assert got.items.dtype == want.items.dtype == np.int32, what
    assert got.items.shape == want.items.shape and np.array_equal(got.items, want.items), what
    assert (got.cover is None) == (want.cover is None), what
    if want.cover is not None:
        assert got.cover.shape == want.cover.shape and np.array_equal(got.cover, want.cover), what
    assert {f: getattr(got, f) for f in WL_FIELDS} == {f: getattr(want, f) for f in WL_FIELDS}, what


def _same_plan(p, m):
    assert (p.tw, p.th, p.fast, p.mma) == (m.tw, m.th, m.fast, m.mma)
    assert [dataclasses.astuple(t) for t in p.tiles] == [dataclasses.astuple(t) for t in m.tiles]
    for name in ("tile_desc", "tabs", "mask_specs"):
        a, b = getattr(p, name), getattr(m, name)
        assert a.dtype == b.dtype == np.int32 and a.shape == b.shape and np.array_equal(a, b), name
    assert p.mask_pool_bytes == m.mask_pool_bytes and p.mask_class == m.mask_class
    assert p._mask_off == m._mask_off and p._mask_pitch == m._mask_pitch
    assert p.neighbors == m.neighbors
    for name in ("_tab_off", "_tab_packed", "_tab_frag", "_tab_ks", "_tab_taps", "_tab_job_taps"):
        assert getattr(p, name) == getattr(m, name), name
    for t in p.tiles:
        assert p.support(t) == m.support(m.tiles[t.idx]) and p.opaque_core(t) == m.opaque_core(m.tiles[t.idx])


@pytest.mark.parametrize("case", CASES, ids=lambda c: c[0])
def test_library_plan_equals_the_numpy_model(case, launch_model):
    name, W, H, tw, th, pad, blur, uniform, B = case
    i = CASES.index(case)
    sms, forced = [(132, 0), (114, 0), (132, 16), (78, 0)][i % 4]
    launch_model(sms, forced)
    p, m = planner.Plan.build(W, H, tw, th, pad, blur, uniform), pm.Plan.build(W, H, tw, th, pad, blur, uniform)
    _same_plan(p, m)
    T = len(p.tiles)
    rng = np.random.default_rng(i)
    shuffled = rng.permutation(T).tolist()
    assert p.waves() == m.waves() and p.waves(shuffled) == m.waves(shuffled)
    waves = m.waves()
    big = T > 1000                                   # cfg4-size grids: whole-canvas lists and the first waves only
    for path in (0, 1, 2):
        lists = [list(range(T))] + [sorted(w, key=lambda t: (m.tiles[t].ph, m.tiles[t].pw, t)) for w in waves[:2 if big else 4]]
        for k, ids in enumerate(lists):
            got, goffs, gtotal = p.crop_worklist(ids, B, path)
            want, woffs, wtotal = m.crop_worklist(ids, B, path)
            _same_worklist(got, want, (name, "crop", path, k))
            assert np.array_equal(goffs, woffs) and gtotal == wtotal
            offs = woffs + (0 if k % 2 else (5 << 32) + 48)            # source offsets beyond 2^32
            for src_bytes in (4, 1):
                _same_worklist(p.blend_worklist(ids, offs, src_bytes, path, B),
                               m.blend_worklist(ids, offs, src_bytes, path, B), (name, "blend", path, k, src_bytes))
            if k == 0 or not big:
                n = 2 + (i + k) % 3
                for part_i in range(n):
                    _same_worklist(p.blend_worklist(ids, offs, 4, path, B, (part_i, n)),
                                   m.blend_worklist(ids, offs, 4, path, B, (part_i, n)), (name, "blend part", path, k, part_i, n))


@pytest.mark.parametrize("case", [c for c in CASES if c[0] in ("cfg1", "cfg2", "blur255_pad256", "w_not_mult4", "nonuniform_odd_w")],
                         ids=lambda c: c[0])
def test_split_level_lists_equal_the_numpy_model(case, launch_model):
    """The split schedule, which stays in Python, consumes the library's records: per wave the crop list, the mask of its
    late jobs and the blend list."""
    name, W, H, tw, th, pad, blur, uniform, B = case
    launch_model(132)
    p, m = planner.Plan.build(W, H, tw, th, pad, blur, uniform), pm.Plan.build(W, H, tw, th, pad, blur, uniform)
    waves = [sorted(w, key=lambda t: (m.tiles[t].ph, m.tiles[t].pw, t)) for w in m.waves()][:4]
    for path in (1, 2):
        for k, w in enumerate(waves):
            offs, _ = m.slot_offsets(w, B)
            prev = waves[k - 1] if k else None
            got, want = p.split_level(w, offs, prev, B, path), m.split_level(w, offs, prev, B, path)
            _same_worklist(got[0], want[0], (name, "split crop", k))
            assert np.array_equal(got[1], want[1]) and got[2] == want[2]
            assert (got[3] is None) == (want[3] is None) and (got[3] is None or np.array_equal(got[3], want[3]))
            _same_worklist(got[4], want[4], (name, "split blend", k))


def test_empty_lists_and_the_default_launch_model(monkeypatch):
    monkeypatch.delenv("USDU_MMA_BH", raising=False)
    p, m = planner.Plan.build(640, 480, 128, 128, 16, 8, True), pm.Plan.build(640, 480, 128, 128, 16, 8, True)
    for path in (0, 1, 2):
        got, goffs, gtotal = p.crop_worklist([], 1, path)
        want, woffs, wtotal = m.crop_worklist([], 1, path)
        _same_worklist(got, want, ("empty crop", path))
        assert goffs.shape == woffs.shape == (0,) and gtotal == wtotal == 0
        _same_worklist(p.blend_worklist([], [], 4, path, 1), m.blend_worklist([], [], 4, path, 1), ("empty blend", path))
    # sm_count = 0: the library asks the device itself (132 SMs where there is none), like the model
    ids = list(range(len(p.tiles)))
    _same_worklist(p.crop_worklist(ids, 3)[0], m.crop_worklist(ids, 3)[0], "default model")


def _lib():
    return nat.lib()


@pytest.mark.parametrize("args,msg", [((640, 480, 3, 128, 16, 8, 1), b"rounds to zero"), ((640, 480, 128, -4, 16, 8, 1), b"rounds to zero"),
                                      ((46400, 46400, 46400, 46400, 0, 8, 1), b"2 GiB"), ((0, 480, 128, 128, 16, 8, 1), b"1x1")])
def test_invalid_plans_are_rejected(args, msg):
    h = ctypes.c_void_p(1)
    assert _lib().usdu_plan_create(*args, ctypes.byref(h)) == nat.ERR_INVALID
    assert h.value is None and msg in _lib().usdu_last_error()
    with pytest.raises(ValueError):
        planner.Plan.build(*args)
    if args[0] > 0:
        with pytest.raises(ValueError):
            pm.Plan.build(*args)                     # the numpy planner rejected the same inputs


def test_bad_worklist_arguments_are_rejected():
    p = planner.Plan.build(640, 480, 128, 128, 16, 8, True)
    with pytest.raises(nat.NativeError, match="out of range"):
        p.crop_worklist([0, len(p.tiles)], 1)
    with pytest.raises(nat.NativeError, match="bad arguments"):
        p.blend_worklist([0], [0], 2)                # source elements are fp32 or u8
    with pytest.raises(nat.NativeError, match="bad arguments"):
        p.blend_worklist([0], [0], 4, None, 1, (3, 3))
    with pytest.raises(ValueError, match="twice"):
        p.waves([0, 1, 0])


def test_canvas_size_includes_the_kernels_slack():
    assert nat.canvas_bytes(2, 5, 7) == 2 * 5 * 128 + nat.CANVAS_SLACK
    assert nat.canvas_bytes(1, 4320, 7680) == 4320 * (7680 * 3) + 16
    assert _lib().usdu_canvas_bytes(0, 1, 1) == nat.ERR_INVALID


def test_the_cases_reach_every_kind_of_plan():
    """The geometries above cover the corners the records have: generic-only plans (an axis with more than 15 taps),
    integer-pipe-only plans (windows off 4-pixel columns), tensor-core plans with two-k-step axes, non-uniform plans
    on the tensor cores, and frame batches of 1, 5 and 17."""
    seen = set()
    for name, W, H, tw, th, pad, blur, uniform, B in CASES:
        p = planner.Plan.build(W, H, tw, th, pad, blur, uniform)
        seen.add(("path", p.kernel_path(None)))
        seen.add(("B", B))
        if p.mma:
            seen.add(("ks2", bool(max(p._tab_ks.values()) > 1)))
            seen.add(("mma nonuniform", not uniform))
        if not p.fast:
            seen.add(("taps > 15", max(int(p.tabs[o + 3]) for o in p._tab_off.values()) > 15))
    assert {("path", 0), ("path", 1), ("path", 2), ("B", 1), ("B", 5), ("B", 17), ("ks2", True), ("mma nonuniform", True),
            ("taps > 15", True)} <= seen, seen


C_JOB = os.path.join(os.path.dirname(nat.LIB_PATH), "usdu_c_job")


def test_c_host_needs_no_python():
    """usdu_c_job (csrc/tools/usdu_c_job.c) is built with the library and links neither libpython nor torch; it plans
    on the host before it touches the device, so argument and plan errors come back without one."""
    import shutil
    import subprocess
    assert os.access(C_JOB, os.X_OK)
    if shutil.which("ldd"):
        libs = subprocess.run(["ldd", C_JOB], capture_output=True, text=True, check=True).stdout
        assert "libusdu_b200.so" in libs and "python" not in libs and "torch" not in libs
    r = subprocess.run([C_JOB], capture_output=True, text=True)
    assert r.returncode == 2 and "usage" in r.stderr
    r = subprocess.run([C_JOB, "640", "480", "1", "3", "3", "16", "8", "1", "0.5", "a", "b", "c"], capture_output=True, text=True)
    assert r.returncode == 1 and "rounds to zero" in r.stderr
