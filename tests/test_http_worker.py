"""The static-mode HTTP worker (http_worker.HttpStaticWorker, engine.WorkerJob, the node's worker role) against the
reference's real master: its aiohttp routes on 127.0.0.1 and its static-mode driver (oracle/ref_static_run._Env, loaded
from the bundle oracle/make_ref.py stages).  Workers pull tile ids from a queue, so who processes which tile differs from
run to run; each test records the assignment that happened and checks the master's result against
`usdu_oracle.replay_static` of that assignment, bit for bit."""
import json
import sys
import threading
import time

import numpy as np
import pytest
import torch

import ref_static_run
import usdu_oracle as orc
from __graft_entry__ import load_package
from inputs import make_input

load_package()
from comfyui_distributed_b200.http_worker import HttpStaticWorker  # noqa: E402

pytestmark = pytest.mark.skipif(not ref_static_run.available(), reason="reference bundle (oracle/_ref) not present")
SEED, DENOISE = 5, 0.5
JOB = "job1"


def _run_job(img, tile, pad, blur, uniform, workers, master_delay=0.5, master_log=None, before_master_tile=None,
             timeout=300):
    """The reference's master (T0 sampler, `master_delay` s before each of its tiles so that the workers get a share)
    plus `workers`: {name: fn(env, name, url) -> anything}, each in its own thread, started in this order.
    before_master_tile(k) runs before the master's k-th tile (k = 0, 1, ...).
    -> (master's fp32 result, master's tile ids in order, {name: what fn returned or raised})."""
    env = ref_static_run._Env()
    try:
        env.sampler = ref_static_run.torch_t0
        B, H, W, _ = img.shape
        _, _, plan = orc.make_plan(W, H, tile, tile, pad, uniform)
        by_origin = {(t.x, t.y): t.idx for t in plan}
        mlog = [] if master_log is None else master_log
        node = env.node_cls()
        extract = node.extract_batch_tile_with_padding      # called once per tile the master processes

        def spy(image, tx, ty, *rest):
            if before_master_tile is not None:
                before_master_tile(len(mlog))
            time.sleep(master_delay)
            mlog.append(by_origin[(int(tx), int(ty))])
            return extract(image, tx, ty, *rest)

        node.extract_batch_tile_with_padding = spy
        cond = [[torch.zeros(1, 77, 8), {}]]
        args = (None, cond, cond, None, SEED, 20, 8.0, "euler", "normal", DENOISE, tile, tile, pad, blur, uniform, False)
        url = f"http://127.0.0.1:{env.port}"
        out = {}

        def call(name, fn):
            try:
                out[name] = fn()
            except BaseException as e:      # noqa: BLE001 -- handed to the test
                out[name] = e

        def master():
            return node.run(torch.from_numpy(img), *args, multi_job_id=JOB, is_worker=False,
                            enabled_worker_ids=json.dumps(list(workers)))[0].numpy()

        threads = [threading.Thread(target=call, args=("master", master), name="master", daemon=True)]
        threads += [threading.Thread(target=call, args=(n, lambda n=n: workers[n](env, n, url)), name=n, daemon=True)
                    for n in workers]
        for t in threads:
            t.start()
        for t in threads:
            t.join(timeout)
        assert not any(t.is_alive() for t in threads), "job did not finish"
        res = out.pop("master")
        if isinstance(res, BaseException):
            raise res
        return res, mlog, out
    finally:
        env.close()


def _replay(img, tile, pad, blur, uniform, assignment):
    return orc.replay_static(img, orc.make_t0_denoiser(SEED, DENOISE), tile, tile, pad, blur, uniform, assignment)


def _n_tiles(img, tile, pad, uniform):
    return len(orc.make_plan(img.shape[2], img.shape[1], tile, tile, pad, uniform)[2])


def _first_tile_of(started: threading.Event):
    """before_master_tile: the master holds its first tile until a worker has one (`started`), so that the worker gets
    a share however long it takes to start."""
    def gate(k):
        if k == 0:
            assert started.wait(120), "the worker never started a tile"
    return gate


def _oracle_worker(img, tile, pad, blur, uniform, before_step=None, started=None):
    """HttpStaticWorker whose tile step is the oracle on this worker's own numpy canvas (static.py:242-280); it sets
    `started` when it reaches its first tile."""
    B, H, W, _ = img.shape
    tw, th, plan = orc.make_plan(W, H, tile, tile, pad, uniform)
    t0 = orc.make_t0_denoiser(SEED, DENOISE)

    def fn(env, name, url):
        canvas = orc.quantize_u8(img)
        w = HttpStaticWorker(url, JOB, name, pad, [(t.x1, t.y1, t.ew, t.eh) for t in plan], B)

        def step(tid):
            if started is not None:
                started.set()
            if before_step is not None:
                before_step(w, tid)
            t = plan[tid]
            res = t0(orc.extract_tile(canvas, t), t)
            orc.blend_processed(canvas, res, t, orc.tile_mask_window(W, H, t.x, t.y, tw, th, blur, (t.x1, t.y1, t.x2, t.y2)))
            return orc.quantize_u8(res)

        try:
            w.run(step)
        except BaseException as e:          # keep the worker's record next to its error
            e.worker = w
            raise
        return w

    return fn


@pytest.mark.timeout(600)
@pytest.mark.parametrize("kind,seed,B,H,W,tile,pad,blur,uniform", [
    ("noise", 17, 1, 520, 700, 256, 32, 8, True),
    ("smooth", 18, 5, 200, 260, 128, 16, 4, True),          # 5 frames per tile: the 20-entry flush falls mid-job
    ("noise", 19, 1, 640, 900, 256, 16, 16, False),        # force_uniform_tiles=False: processing size = window size
])
def test_transport_against_reference_master(kind, seed, B, H, W, tile, pad, blur, uniform):
    img = make_input(kind, seed, B, H, W)
    started = threading.Event()
    res, mlog, out = _run_job(img, tile, pad, blur, uniform,
                              {"w1": _oracle_worker(img, tile, pad, blur, uniform, started=started)},
                              before_master_tile=_first_tile_of(started))
    w = out["w1"]
    assert not isinstance(w, BaseException), w
    assert w.pulled, "the worker got no tile: nothing was checked"
    assert sorted(mlog + w.pulled) == list(range(_n_tiles(img, tile, pad, uniform)))
    assert np.array_equal(res, _replay(img, tile, pad, blur, uniform, [mlog, w.pulled])), (mlog, w.pulled)
    assert w.chunks == -(-len(w.pulled) * B // w.max_batch)     # an upload per COMFYUI_MAX_BATCH entries, the rest at the end


@pytest.mark.timeout(600)
def test_flush_splits_into_chunks(monkeypatch):
    img = make_input("noise", 20, 1, 520, 700)
    # 256 px tiles + 2 * 32 padding: ~300 KB level-0 PNGs; the 1 MB headroom + 700 KB leaves room for two per chunk
    monkeypatch.setenv("COMFYUI_MAX_PAYLOAD_SIZE", str((1 << 20) + 700_000))
    started = threading.Event()
    res, mlog, out = _run_job(img, 256, 32, 8, True, {"w1": _oracle_worker(img, 256, 32, 8, True, started=started)},
                              master_delay=1.0, before_master_tile=_first_tile_of(started))
    w = out["w1"]
    assert not isinstance(w, BaseException), w
    assert len(w.pulled) >= 3
    assert w.chunks == (len(w.pulled) + 1) // 2
    assert np.array_equal(res, _replay(img, 256, 32, 8, True, [mlog, w.pulled])), (mlog, w.pulled)


@pytest.mark.timeout(600)
def test_worker_without_tiles_sends_only_the_completion_signal():
    """w2 starts pulling once every tile has an owner (the master, or w1, which stalls on its first tile until w2 is
    done): it gets no tile and posts the empty completion signal, nothing else; w1 then finishes the job."""
    img = make_input("noise", 21, 1, 520, 700)
    n = _n_tiles(img, 256, 32, True)
    w2_done = threading.Event()
    w1_obj, mlog = [], []

    def stall(w, tid):
        if not w1_obj:
            w1_obj.append(w)
            assert w2_done.wait(120)

    def w2(env, name, url):
        try:
            deadline = time.monotonic() + 120
            while time.monotonic() < deadline and not (w1_obj and len(mlog) + len(w1_obj[0].pulled) == n):
                time.sleep(0.05)
            w = HttpStaticWorker(url, JOB, name, 32, [(0, 0, 1, 1)] * n, 1)
            posts = []
            post = w._post_form
            w._post_form = lambda parts, retries: (posts.append({k: v for k, v, _, _ in parts}), post(parts, retries))
            w.run(lambda tid: pytest.fail("w2 must not get a tile"))
            return w, posts
        finally:
            w2_done.set()

    started = threading.Event()
    workers = {"w1": _oracle_worker(img, 256, 32, 8, True, stall, started), "w2": w2}
    res, mlog, out = _run_job(img, 256, 32, 8, True, workers, master_log=mlog, before_master_tile=_first_tile_of(started))
    assert not isinstance(out["w1"], BaseException), out["w1"]
    assert not isinstance(out["w2"], BaseException), out["w2"]
    w, posts = out["w2"]
    assert w.pulled == [] and w.chunks == 0
    assert posts == [{"multi_job_id": JOB.encode(), "worker_id": b"w2", "is_last": b"true", "batch_size": b"0"}]
    assert np.array_equal(res, _replay(img, 256, 32, 8, True, [mlog, out["w1"].pulled, []]))


class Interrupted(Exception):
    pass


@pytest.mark.timeout(600)
def test_interrupt_propagates_out_of_run(monkeypatch):
    """ComfyUI's cancel, raised at w1's third poll (after two tiles, none uploaded yet), leaves run() as is; the master
    re-queues w1's tiles once its heartbeat is overdue and computes them itself."""
    monkeypatch.setenv("COMFYUI_HEARTBEAT_INTERVAL", "0.5")      # read when _Env loads the reference's constants
    monkeypatch.setenv("COMFYUI_HEARTBEAT_TIMEOUT", "1")
    img = make_input("noise", 22, 1, 520, 700)
    polls = []

    def w1(env, name, url):
        def poll():             # the stand-in comfy module is shared with the master: only this thread is cancelled
            if threading.current_thread().name == name:
                polls.append(1)
                if len(polls) == 3:
                    raise Interrupted()
        monkeypatch.setattr(sys.modules["comfy.model_management"],
                            "throw_exception_if_processing_interrupted", poll)
        return _oracle_worker(img, 256, 32, 8, True, started=started)(env, name, url)

    started = threading.Event()
    res, mlog, out = _run_job(img, 256, 32, 8, True, {"w1": w1}, master_delay=0.5, before_master_tile=_first_tile_of(started))
    err = out["w1"]
    assert isinstance(err, Interrupted), err
    assert len(err.worker.pulled) == 2 and err.worker.chunks == 0
    assert sorted(mlog) == list(range(_n_tiles(img, 256, 32, True)))
    assert np.array_equal(res, _replay(img, 256, 32, 8, True, [mlog]))


# --------------------------------------------------------------------------------------
# GPU: this package's node as a worker beside a reference worker, one master
# --------------------------------------------------------------------------------------
def _gpu_worker(img, first_tile: threading.Event, before_second_tile: threading.Event):
    """This package's node as an HTTP worker, T0 sampler on the device.  It sets `first_tile` when its first tile reaches
    the sampler and holds its second tile until `before_second_tile` is set."""
    from comfyui_distributed_b200.denoise import T0Denoiser
    from comfyui_distributed_b200.nodes import UltimateSDUpscaleDistributed

    class GatedT0:
        def as_usdu_denoiser(self, seed, denoise, **_):
            t0, calls = T0Denoiser(seed, denoise), []

            def fn(tiles, rows):
                calls.append(len(rows))
                if len(calls) == 1:
                    first_tile.set()
                elif len(calls) == 2:
                    assert before_second_tile.wait(120), "the reference worker never started a tile"
                return t0(tiles, rows)

            return fn

    def fn(env, name, url, tile, pad, blur, uniform):
        x = torch.from_numpy(img)
        node = UltimateSDUpscaleDistributed()
        (out,) = node.run(x, GatedT0(), None, None, None, SEED, 20, 8.0, "euler", "normal", DENOISE, tile, tile, pad,
                          blur, uniform, False, multi_job_id=JOB, is_worker=True, master_url=url, worker_id=name,
                          enabled_worker_ids=json.dumps(["w1", "w2"]))
        assert out is x                              # a worker hands its input through (static.py:314)
        return node.last_stats["pulled"]

    return fn


def _ref_worker(img, start: threading.Event, first_tile: threading.Event):
    """The reference's worker; it starts once `start` is set and sets `first_tile` when it crops its first tile."""
    def fn(env, name, url, tile, pad, blur, uniform):
        B, H, W, _ = img.shape
        _, _, plan = orc.make_plan(W, H, tile, tile, pad, uniform)
        by_origin = {(t.x, t.y): t.idx for t in plan}
        node = env.node_cls()
        extract, log = node.extract_batch_tile_with_padding, []

        def spy(image, tx, ty, *rest):
            log.append(by_origin[(int(tx), int(ty))])
            first_tile.set()
            return extract(image, tx, ty, *rest)

        node.extract_batch_tile_with_padding = spy
        cond = [[torch.zeros(1, 77, 8), {}]]
        assert start.wait(120), "the GPU worker never started a tile"
        node.run(torch.from_numpy(img), None, cond, cond, None, SEED, 20, 8.0, "euler", "normal", DENOISE, tile, tile,
                 pad, blur, uniform, False, multi_job_id=JOB, is_worker=True, master_url=url, worker_id=name,
                 enabled_worker_ids=json.dumps(["w1", "w2"]))
        return log

    return fn


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("kind,seed,B,H,W,tile,pad,blur,uniform", [
    ("noise", 4, 1, 1100, 1300, 512, 32, 8, True),       # the geometry of the recorded HTTP runs
    ("smooth", 5, 5, 300, 420, 128, 16, 8, True),
])
def test_gpu_node_worker_in_a_mixed_fleet(kind, seed, B, H, W, tile, pad, blur, uniform):
    """Every participant gets a tile, whatever the start-up times: the master holds its first tile until the GPU worker
    has one in its sampler, and its second until the reference worker (started then) has one; the GPU worker holds its
    second tile until then too.  After that all three pull freely."""
    img = make_input(kind, seed, B, H, W)
    geo = (tile, pad, blur, uniform)
    w1_started, w2_started = threading.Event(), threading.Event()

    def gate_master(k):
        if k < 2:
            assert (w1_started, w2_started)[k].wait(120), "a worker never started a tile"

    workers = {"w1": lambda env, n, url: _gpu_worker(img, w1_started, w2_started)(env, n, url, *geo),
               "w2": lambda env, n, url: _ref_worker(img, w1_started, w2_started)(env, n, url, *geo)}
    res, mlog, out = _run_job(img, tile, pad, blur, uniform, workers, master_delay=0.0, before_master_tile=gate_master)
    for n in workers:
        assert not isinstance(out[n], BaseException), (n, out[n])
    assert mlog and out["w1"] and out["w2"], (mlog, out["w1"], out["w2"])
    assert sorted(mlog + out["w1"] + out["w2"]) == list(range(_n_tiles(img, tile, pad, uniform)))
    want = _replay(img, tile, pad, blur, uniform, [mlog, out["w1"], out["w2"]])
    assert np.array_equal(res, want), (mlog, out["w1"], out["w2"])
