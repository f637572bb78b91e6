"""This package's node as the static-mode master of HTTP workers (http_master.py, csrc/usdu_png_decode.cu): the PNG
decode kernel against PIL, and whole jobs served from an aiohttp app on 127.0.0.1 behind a server.PromptServer stand-in
(oracle/ref_static_run._Env), with the reference's workers, this package's workers or both.  Each job's result must equal
`usdu_oracle.replay_static` of the effective assignment the master records, bit for bit."""
import io
import json
import threading
import time

import numpy as np
import pytest
import torch
from PIL import Image

import ref_static_run
import usdu_oracle as orc
from __graft_entry__ import load_package
from inputs import make_input
from test_http_master import image, png_of

load_package()
from comfyui_distributed_b200 import _native as nat  # noqa: E402
from comfyui_distributed_b200 import engine  # noqa: E402
from comfyui_distributed_b200 import http_master as hm  # noqa: E402
from comfyui_distributed_b200.http_worker import HttpStaticWorker, _call, encode_png, multipart  # noqa: E402
from comfyui_distributed_b200.testing import T0Model  # noqa: E402

SEED, DENOISE = 5, 0.5
JOB = "jobG"


# --------------------------------------------------------------------------------------
# the decode kernel
# --------------------------------------------------------------------------------------
def decode_on_gpu(pngs, dst_offsets, dst_bytes, pad_between=7):
    """One launch over `pngs` (bytes), frame i written at dst_offsets[i] of a fresh u8 buffer; the files sit at odd
    offsets of the upload."""
    blobs, segs, descs, pos, max_row = [], [], [], 3, 1
    for data, off in zip(pngs, dst_offsets):
        info = hm.parse_png(data)
        blob = info.inflated if info.inflated is not None else data
        descs.append([len(segs), len(info.segs), info.H, info.W, info.C, off, 0, 0])
        segs += [(pos + o, r) for o, r in info.segs]
        blobs.append((pos, blob))
        pos += len(blob) + pad_between
        max_row = max(max_row, info.W * info.C)
    src = np.zeros(pos, np.uint8)
    for p, b in blobs:
        src[p: p + len(b)] = np.frombuffer(b, np.uint8)
    d_src = torch.from_numpy(src).cuda()
    d_segs = torch.tensor(np.asarray(segs, np.int64).reshape(-1)).cuda()
    d_descs = torch.tensor(np.asarray(descs, np.int64).reshape(-1)).cuda()
    dst = torch.full((dst_bytes,), 0xA5, dtype=torch.uint8, device="cuda")
    nat.png_decode_u8(d_src.data_ptr(), d_segs.data_ptr(), len(segs), d_descs.data_ptr(), len(descs), max_row,
                      dst.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return dst.cpu().numpy()


def _pil(data):
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


@pytest.mark.gpu
def test_decode_kernel_equals_pil_many_per_launch():
    files = []
    for level in (0, 1, 6, 9):
        for mode in ("L", "LA", "RGB", "RGBA"):
            for h, w in ((1, 1), (1, 77), (53, 1), (37, 70), (100, 33)):
                files.append(png_of(image(mode, h, w, h + w + level), level))
        files.append(png_of(image("RGB", 544, 544, level), level))
    files.append(png_of(image("RGBA", 40, 2560, 1), 0))                 # the widest processing tile, 4 channels
    files.append(png_of(image("RGB", 576, 576, 2), 0))
    rng = np.random.default_rng(0)
    offs, cur = [], 5
    for f in files:
        info = hm.parse_png(f)
        offs.append(cur)
        cur += info.H * info.W * 3 + int(rng.integers(0, 40))
    out = decode_on_gpu(files, offs, cur + 16)
    for f, o in zip(files, offs):
        want = _pil(f)
        got = out[o: o + want.size].reshape(want.shape)
        assert np.array_equal(got, want), (hm.parse_png(f).C, want.shape)
    assert (out[:5] == 0xA5).all()                                     # nothing outside the frames is written


@pytest.mark.gpu
def test_decode_kernel_b_frames_of_worker_tiles():
    """What workers post: B = 5 frames per tile at processing size, decoded into one tile's [B, ph, pw, 3] slot."""
    img = make_input("noise", 3, 5, 200, 260)
    tiles = [encode_png((img[b, :144, :144] * 255).astype(np.uint8)) for b in range(5)]
    frame = 144 * 144 * 3
    out = decode_on_gpu(tiles, [16 + b * frame for b in range(5)], 16 + 5 * frame)
    for b in range(5):
        assert np.array_equal(out[16 + b * frame: 16 + (b + 1) * frame].reshape(144, 144, 3), _pil(tiles[b]))


# --------------------------------------------------------------------------------------
# whole jobs
# --------------------------------------------------------------------------------------
class Master:
    """The reference's ComfyUI stand-ins (server, comfy, nodes) from _Env, with THIS package's routes served from a
    second aiohttp app on the same loop."""

    def __init__(self):
        from aiohttp import web
        self.env = ref_static_run._Env()
        self.env.sampler = ref_static_run.torch_t0
        hm.reset_for_tests()
        routes = web.RouteTableDef()
        hm.register(routes, hm.STORE, self.env.loop)
        app = web.Application(client_max_size=1 << 30)
        app.add_routes(routes)
        self.runner = web.AppRunner(app)
        self.port = ref_static_run._free_port()
        self.env._call(self.runner.setup())
        self.env._call(web.TCPSite(self.runner, "127.0.0.1", self.port).start())
        self.url = f"http://127.0.0.1:{self.port}"
        assert hm.serving()

    def close(self):
        try:
            self.env._call(self.runner.cleanup())
        finally:
            hm.reset_for_tests()
            self.env.close()


def _node_args(tile, pad, blur, uniform):
    return (T0Model(), None, None, None, SEED, 20, 8.0, "euler", "normal", DENOISE, tile, tile, pad, blur, uniform, False)


def _n_tiles(img, geo):
    tile, pad, _, uniform = geo
    return len(orc.make_plan(img.shape[2], img.shape[1], tile, tile, pad, uniform)[2])


def _replay(img, tile, pad, blur, uniform, assignment):
    return orc.replay_static(img, orc.make_t0_denoiser(SEED, DENOISE), tile, tile, pad, blur, uniform, assignment)


def _ref_worker(img, geo, started):
    tile, pad, blur, uniform = geo

    def fn(m, name, names):
        B, H, W, _ = img.shape
        _, _, plan = orc.make_plan(W, H, tile, tile, pad, uniform)
        by_origin = {(t.x, t.y): t.idx for t in plan}
        node = m.env.node_cls()
        extract, log = node.extract_batch_tile_with_padding, []

        def spy(image_, tx, ty, *rest):
            log.append(by_origin[(int(tx), int(ty))])
            started.set()
            return extract(image_, tx, ty, *rest)

        node.extract_batch_tile_with_padding = spy
        cond = [[torch.zeros(1, 77, 8), {}]]
        node.run(torch.from_numpy(img), None, cond, cond, None, SEED, 20, 8.0, "euler", "normal", DENOISE, tile, tile,
                 pad, blur, uniform, False, multi_job_id=JOB, is_worker=True, master_url=m.url, worker_id=name,
                 enabled_worker_ids=json.dumps(names))
        return log

    return fn


def _gpu_worker(img, geo, started):
    from comfyui_distributed_b200.denoise import T0Denoiser
    from comfyui_distributed_b200.nodes import UltimateSDUpscaleDistributed

    class Flagged:
        def as_usdu_denoiser(self, seed, denoise, **_):
            t0 = T0Denoiser(seed, denoise)

            def fn(tiles, rows):
                started.set()
                return t0(tiles, rows)
            return fn

    def fn(m, name, names):
        node = UltimateSDUpscaleDistributed()
        args = (Flagged(),) + _node_args(*geo)[1:]
        (out,) = node.run(torch.from_numpy(img), *args, multi_job_id=JOB, is_worker=True, master_url=m.url,
                          worker_id=name, enabled_worker_ids=json.dumps(names))
        return node.last_stats["pulled"]

    return fn


def _run_master_job(img, geo, workers, monkeypatch, master_delay=0.3, gate=(), timeout=600, cuda_input=False):
    """Our node as the master, `workers` = {name: fn(master, name, names)} in threads.  The master sleeps
    `master_delay` s before each of its tiles and holds its first one until every event in `gate` is set.
    -> (result numpy, node.last_stats, {name: worker result or exception})."""
    from comfyui_distributed_b200.nodes import UltimateSDUpscaleDistributed
    m = Master()
    try:
        step = engine.WorkerJob.step_device
        count = [0]

        def slow_step(self, tid):
            if count[0] == 0:
                for ev in gate:
                    assert ev.wait(180), "a worker never started a tile"
            count[0] += 1
            time.sleep(master_delay)
            return step(self, tid)

        monkeypatch.setattr(engine.WorkerJob, "step_device", slow_step)
        names = list(workers)
        out = {}

        def call(name, fn):
            try:
                out[name] = fn()
            except BaseException as e:      # noqa: BLE001 -- handed to the test
                out[name] = e

        node = UltimateSDUpscaleDistributed()
        x = torch.from_numpy(img)
        x = x.cuda() if cuda_input else x

        def master():
            return node.run(x, *_node_args(*geo), multi_job_id=JOB, is_worker=False,
                            enabled_worker_ids=json.dumps(names))[0]

        threads = [threading.Thread(target=call, args=("master", master), daemon=True)]
        threads += [threading.Thread(target=call, args=(n, lambda n=n: workers[n](m, n, names)), name=n, daemon=True)
                    for n in names]
        for t in threads:
            t.start()
        for t in threads:
            t.join(timeout)
        assert not any(t.is_alive() for t in threads), "job did not finish"
        res = out.pop("master")
        if isinstance(res, BaseException):
            raise res
        assert res.is_cuda == cuda_input and (cuda_input or res.is_pinned())
        return res.cpu().numpy(), node.last_stats, out
    finally:
        m.close()


@pytest.mark.gpu
@pytest.mark.timeout(1200)
@pytest.mark.parametrize("kind,seed,B,H,W,tile,pad,blur,uniform,fleet", [
    ("noise", 1, 1, 520, 700, 256, 32, 8, True, ("ref",)),
    ("smooth", 2, 5, 200, 260, 128, 16, 4, True, ("gpu",)),
    ("noise", 3, 1, 640, 900, 256, 0, 0, False, ("ref", "gpu")),
    ("noise", 4, 5, 300, 420, 128, 16, 16, False, ("gpu", "ref")),
])
def test_master_with_http_workers_equals_replay(monkeypatch, kind, seed, B, H, W, tile, pad, blur, uniform, fleet):
    img = make_input(kind, seed, B, H, W)
    geo = (tile, pad, blur, uniform)
    events = [threading.Event() for _ in fleet]
    workers = {f"w{i + 1}": (_ref_worker if k == "ref" else _gpu_worker)(img, geo, events[i]) for i, k in enumerate(fleet)}
    res, stats, out = _run_master_job(img, geo, workers, monkeypatch, gate=events, cuda_input=(seed % 2 == 0))
    for n, v in out.items():
        assert not isinstance(v, BaseException), (n, v)
    asg = stats["assignment"]
    n_tiles = len(orc.make_plan(W, H, tile, tile, pad, uniform)[2])
    assert sorted(t for a in asg for t in a) == list(range(n_tiles))
    assert asg[1:] == [out[n] for n in workers], (asg, out)          # every worker tile was kept, in arrival order
    assert all(asg[1:]), asg
    assert stats["tiles_received"] == B * sum(len(a) for a in asg[1:]) and stats["bytes_received"] > 0
    assert np.array_equal(res, _replay(img, tile, pad, blur, uniform, asg)), asg


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_no_worker_connects(monkeypatch):
    img = make_input("noise", 5, 1, 520, 700)
    geo = (256, 32, 8, True)
    # an enabled worker that never comes: the master drains the queue alone
    res, stats, out = _run_master_job(img, geo, {"w1": lambda m, n, names: None}, monkeypatch, master_delay=0.0)
    n = _n_tiles(img, geo)
    assert stats["assignment"] == [list(range(n)), []]
    assert np.array_equal(res, _replay(img, *geo, [list(range(n))]))
    assert np.array_equal(res, orc.process_single(img, orc.make_t0_denoiser(SEED, DENOISE), 256, 256, 32, 8, True))


def _rogue(img, geo, action, got):
    """A worker that takes one tile and then goes silent; action 'corrupt' first posts that tile as a broken PNG."""
    tile, pad, blur, uniform = geo

    def fn(m, name, names):
        B, H, W, _ = img.shape
        _, _, plan = orc.make_plan(W, H, tile, tile, pad, uniform)
        w = HttpStaticWorker(m.url, JOB, name, pad, [(t.x1, t.y1, t.ew, t.eh) for t in plan], B)
        assert w.wait_ready()
        tid = w.request_tile()
        got.append(tid)
        if action == "corrupt":
            t = plan[tid]
            png = bytearray(encode_png(np.zeros((t.ph, t.pw, 3), np.uint8)))
            png[-18] ^= 0x40                                   # the Adler-32
            meta = [{"tile_idx": tid, "x": t.x1, "y": t.y1, "extracted_width": t.ew, "extracted_height": t.eh,
                     "batch_idx": 0, "global_idx": tid}]
            body, ctype = multipart([("multi_job_id", JOB.encode(), None, None), ("worker_id", name.encode(), None, None),
                                     ("tile_0", bytes(png), "t.png", "image/png"), ("batch_size", b"1", None, None),
                                     ("tiles_metadata", json.dumps(meta).encode(), None, None)])
            status, text = _call(m.url + "/distributed/submit_tiles", "POST", body, ctype)
            got.append((status, json.loads(text)))
        return name

    return fn


@pytest.mark.gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("action", ["silent", "corrupt"])
def test_timed_out_worker_tiles_are_requeued(monkeypatch, action):
    monkeypatch.setenv("COMFYUI_HEARTBEAT_TIMEOUT", "1")
    monkeypatch.setenv("COMFYUI_HEARTBEAT_INTERVAL", "0.5")
    img = make_input("noise", 6, 1, 520, 700)
    geo = (256, 32, 8, True)
    got = []
    started = threading.Event()

    def worker(m, name, names):
        r = _rogue(img, geo, action, got)(m, name, names)
        started.set()
        return r

    res, stats, out = _run_master_job(img, geo, {"w1": worker}, monkeypatch, master_delay=0.2, gate=[started])
    assert out["w1"] == "w1"
    if action == "corrupt":
        status, body = got[1]
        assert status == 400 and body["error"].startswith("Invalid image data for tile 0: "), got
    asg = stats["assignment"]
    assert asg[1] == [] and sorted(asg[0]) == list(range(_n_tiles(img, geo))) and asg[0][-1] == got[0], (asg, got)
    assert np.array_equal(res, _replay(img, *geo, asg))


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_interrupt_during_collection_cleans_up(monkeypatch):
    img = make_input("noise", 7, 1, 520, 700)
    geo = (256, 32, 8, True)
    got, status = [], {}
    started = threading.Event()

    def worker(m, name, names):
        _rogue(img, geo, "silent", got)(m, name, names)
        started.set()
        mm = __import__("sys").modules["comfy.model_management"]
        time.sleep(6.0)                                        # the master is collecting by now (5 tiles x 0.2 s)
        monkeypatch.setattr(mm, "processing_interrupted", lambda: True)
        deadline = time.monotonic() + 60
        while time.monotonic() < deadline:                   # the master leaves; its job is gone
            s, body = _call(m.url + "/distributed/job_status?multi_job_id=" + JOB, "GET")
            status["after"] = (s, json.loads(body))
            if not status["after"][1]["ready"]:
                break
            time.sleep(0.2)
        return name

    with pytest.raises(Exception) as ei:
        _run_master_job(img, geo, {"w1": worker}, monkeypatch, master_delay=0.2, gate=[started])
    assert type(ei.value).__name__ == "_Interrupt", ei.value        # the stand-in InterruptProcessingException
    assert status["after"] == (200, {"ready": False})
    assert hm.STORE.jobs == {}


@pytest.mark.gpu
@pytest.mark.timeout(300)
def test_without_routes_behaviour_is_unchanged():
    from comfyui_distributed_b200.nodes import UltimateSDUpscaleDistributed
    hm.reset_for_tests()
    assert not hm.serving()
    img = make_input("noise", 8, 1, 300, 420)
    geo = (128, 16, 8, True)
    x = torch.from_numpy(img)
    (a,) = UltimateSDUpscaleDistributed().run(x, *_node_args(*geo), multi_job_id=JOB, is_worker=False,
                                              enabled_worker_ids='["w1", "w2"]')
    (b,) = UltimateSDUpscaleDistributed().run(x, *_node_args(*geo))
    assert np.array_equal(a.numpy(), b.numpy())
    assert np.array_equal(a.numpy(), orc.process_single(img, orc.make_t0_denoiser(SEED, DENOISE), 128, 128, 16, 8, True))
