"""The HTTP tile worker's PNG encoder on the GPU (csrc/usdu_png.cu, usdu_png_encode_u8; http_worker.png_layout,
engine.WorkerJob.step_png): byte for byte what encode_png (Pillow, compress_level=0) writes, for single frames, batches,
worker tiles and the whole worker role; and the PIL fallback when a shape's layout check fails."""
import io
import json
import re
import threading
import warnings
from http.server import BaseHTTPRequestHandler, ThreadingHTTPServer

import numpy as np
import pytest
import torch

from __graft_entry__ import load_package
from inputs import make_input
from png_filter_model import rechunk, split_cuts
from test_png_filtered_encoder import PROCESSING, SMALL, _contents

load_package()
from comfyui_distributed_b200 import _native as nat  # noqa: E402
from comfyui_distributed_b200 import engine  # noqa: E402
from comfyui_distributed_b200 import http_worker as hw  # noqa: E402
from comfyui_distributed_b200.denoise import T0Denoiser  # noqa: E402

GUARD = 64
SEED, DENOISE = 5, 0.5


def gpu_files(frames: np.ndarray, layout) -> list:
    """Encode u8 [B, H, W, 3] in one call into an output with guard bytes on both sides; the guards must survive."""
    B = frames.shape[0]
    n = layout.png_len
    buf = torch.full((2 * GUARD + B * n,), 0x5A, dtype=torch.uint8, device="cuda")
    hw.encode_png_gpu(torch.from_numpy(np.ascontiguousarray(frames)).cuda(), layout, buf[GUARD: GUARD + B * n])
    out = buf.cpu().numpy()
    assert (out[:GUARD] == 0x5A).all() and (out[GUARD + B * n:] == 0x5A).all()
    data = out[GUARD: GUARD + B * n].tobytes()
    return [data[b * n:(b + 1) * n] for b in range(B)]


@pytest.fixture(autouse=True)
def fresh_layouts():
    hw._LAYOUTS.clear()
    yield
    hw._LAYOUTS.clear()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_kernel_equals_encode_png_b1_and_b5():
    shapes = SMALL + PROCESSING + [(40, 2560), (1088, 1088)]
    for H, W in shapes:
        layout = hw.png_layout(H, W)
        assert layout is not None, (H, W)
        frames = np.stack([img for _, img in _contents(H, W, H + 5 * W)])       # 7 different frames
        for name, f in zip(["noise", "zeros", "constant", "gradient", "duplicated", "near128", "probe"], frames):
            assert gpu_files(f[None], layout) == [hw.encode_png(f)], (H, W, name)
        assert gpu_files(frames[:5], layout) == [hw.encode_png(f) for f in frames[:5]], (H, W)


@pytest.mark.gpu
def test_kernel_on_split_and_long_chunks():
    """Layouts Pillow does not produce but the tables allow: the Adler trailer and every stored-block header cut
    across two IDAT chunks, and the whole stream in one chunk several CRC spans long."""
    for H, W in [(1, 1), (19, 576), (40, 577), (200, 300)]:
        frames = np.stack([hw.png_probe(H, W, v) for v in range(3)])
        pil = [hw.encode_png(f) for f in frames]
        for cuts in (split_cuts(pil[0]), []):
            layout = hw.layout_from_png(rechunk(pil[0], cuts))
            assert gpu_files(frames, layout) == [rechunk(p, cuts) for p in pil], (H, W, len(cuts))


@pytest.mark.gpu
def test_entry_point_refuses():
    layout = hw.png_layout(8, 8)
    src = torch.zeros(8 * 8 * 4, dtype=torch.uint8, device="cuda")
    out = torch.empty(layout.png_len, dtype=torch.uint8, device="cuda")
    scratch = torch.empty(nat.png_encode_scratch_bytes(1, 8, 8), dtype=torch.uint8, device="cuda")
    tmpl, runs, chunks = layout.device_tables(src.device)
    args = [tmpl.data_ptr(), layout.png_len, runs.data_ptr(), len(layout.runs), chunks.data_ptr(), len(layout.chunks)]
    for B, H, W, C, at in [(1, 8, 8, 4, layout.adler_at), (1, 8, 8, 1, layout.adler_at),
                           (1, 1, 65536 // 3 + 1, 3, layout.adler_at), (-1, 8, 8, 3, layout.adler_at),
                           (1, 8, 8, 3, [0, 1, 2, layout.png_len])]:
        with pytest.raises(nat.NativeError, match="usdu_png_encode_u8"):
            nat.png_encode_u8(src.data_ptr(), B, H, W, C, *args, at, scratch.data_ptr(), out.data_ptr(),
                              torch.cuda.current_stream().cuda_stream)


def _jobs(kind, seed, B, H, W, tile, pad, blur, uniform):
    x = torch.from_numpy(make_input(kind, seed, B, H, W))
    return [engine.WorkerJob(x, T0Denoiser(SEED, DENOISE), tile, tile, pad, blur, uniform) for _ in range(2)]


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("kind,seed,B,H,W,tile,pad,blur,uniform", [
    ("noise", 1, 1, 1080, 1920, 512, 32, 8, True),       # cfg-like: 576 x 576 processing tiles
    ("smooth", 2, 5, 300, 420, 128, 16, 4, True),
    ("noise", 3, 2, 700, 900, 256, 0, 0, False),          # non-uniform: edge tiles of several shapes
])
def test_step_png_equals_pil_of_step(kind, seed, B, H, W, tile, pad, blur, uniform):
    a, b = _jobs(kind, seed, B, H, W, tile, pad, blur, uniform)
    shapes = set()
    for t in range(len(a.plan.tiles)):
        u8 = a.step(t)
        files = b.step_png(t)
        assert isinstance(files, list) and len(files) == B
        assert files == [hw.encode_png(u8[i]) for i in range(B)], t
        shapes.add(u8.shape[1:3])
    assert not uniform or len(shapes) == 1
    assert uniform or len(shapes) > 1
    assert b.times["encode_ms"] > 0 and b.times["tiles"] == len(b.plan.tiles)


# --------------------------------------------------------------------------------------
# the node's worker role against a stub master that records what is posted
# --------------------------------------------------------------------------------------
class StubMaster:
    """The four routes a static-mode worker calls; hands out tiles 0..n-1 and keeps every posted tile file by
    (tile_idx, batch_idx)."""

    def __init__(self, n_tiles):
        self.queue = list(range(n_tiles))
        self.files = {}
        self.posts = 0
        stub = self

        class H(BaseHTTPRequestHandler):
            def log_message(self, *a):
                pass

            def _reply(self, obj):
                body = json.dumps(obj).encode()
                self.send_response(200)
                self.send_header("Content-Type", "application/json")
                self.send_header("Content-Length", str(len(body)))
                self.end_headers()
                self.wfile.write(body)

            def do_GET(self):
                self._reply({"ready": True})

            def do_POST(self):
                body = self.rfile.read(int(self.headers["Content-Length"]))
                if self.path.endswith("request_image"):
                    self._reply({"tile_idx": stub.queue.pop(0) if stub.queue else None})
                elif self.path.endswith("submit_tiles"):
                    stub.record(self.headers["Content-Type"], body)
                    self._reply({"status": "ok"})
                else:
                    self._reply({"status": "ok"})

        self.server = ThreadingHTTPServer(("127.0.0.1", 0), H)
        self.thread = threading.Thread(target=self.server.serve_forever, daemon=True)
        self.thread.start()
        self.url = f"http://127.0.0.1:{self.server.server_address[1]}"

    def record(self, ctype, body):
        boundary = re.search(r"boundary=(\S+)", ctype).group(1).encode()
        parts = {}
        for part in body.split(b"--" + boundary)[1:-1]:
            head, value = part[2:].split(b"\r\n\r\n", 1)
            parts[re.search(rb'name="([^"]+)"', head).group(1).decode()] = value[:-2]
        self.posts += 1
        meta = json.loads(parts.get("tiles_metadata", b"[]"))
        for i, m in enumerate(meta):
            self.files[(m["tile_idx"], m["batch_idx"])] = parts[f"tile_{i}"]

    def close(self):
        self.server.shutdown()
        self.server.server_close()


def _worker_role(img, geo, url):
    from comfyui_distributed_b200.nodes import UltimateSDUpscaleDistributed
    from comfyui_distributed_b200.testing import T0Model
    tile, pad, blur, uniform = geo
    node = UltimateSDUpscaleDistributed()
    node.run(torch.from_numpy(img), T0Model(), None, None, None, SEED, 20, 8.0, "euler", "normal", DENOISE, tile, tile,
             pad, blur, uniform, False, multi_job_id="jobP", is_worker=True, master_url=url, worker_id="w1",
             enabled_worker_ids='["w1"]')
    return node.last_stats


def _n_tiles(img, geo):
    return len(engine.get_plan(img.shape[2], img.shape[1], geo[0], geo[0], geo[1], geo[2], geo[3]).tiles)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_worker_role_posts_pil_bytes(monkeypatch):
    img = make_input("noise", 9, 5, 300, 420)
    geo = (128, 16, 8, False)
    n = _n_tiles(img, geo)
    got = {}
    for arm in ("gpu", "pil"):
        if arm == "pil":
            monkeypatch.setattr(engine.WorkerJob, "step_png", engine.WorkerJob.step)
        m = StubMaster(n)
        try:
            stats = _worker_role(img, geo, m.url)
        finally:
            m.close()
        assert sorted(stats["pulled"]) == list(range(n)) and m.posts >= 1
        got[arm] = m.files
    assert len(got["gpu"]) == 5 * n
    assert got["gpu"] == got["pil"]


@pytest.mark.gpu
@pytest.mark.timeout(1200)
def test_worker_role_same_master_result_as_pil(monkeypatch):
    """This package's master with one of this package's workers: the result equals the replay of the assignment,
    whether the worker encodes on the GPU or with PIL."""
    import test_gpu_http_master as tm
    img = make_input("smooth", 12, 1, 520, 700)
    geo = (256, 32, 8, True)
    for arm in ("gpu", "pil"):
        with monkeypatch.context() as mp:
            if arm == "pil":
                mp.setattr(engine.WorkerJob, "step_png", engine.WorkerJob.step)
            ev = threading.Event()
            res, stats, out = tm._run_master_job(img, geo, {"w1": tm._gpu_worker(img, geo, ev)}, mp, gate=[ev])
        assert not isinstance(out["w1"], BaseException), out
        asg = stats["assignment"]
        assert asg[1], asg
        assert np.array_equal(res, tm._replay(img, *geo, asg)), (arm, asg)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_failed_layout_check_falls_back_to_pil_and_warns_once(monkeypatch):
    real = hw.encode_png_gpu

    def broken(frames, layout, out, scratch=None):
        real(frames, layout, out, scratch)
        out[3] ^= 1                                         # a GPU encoder whose bytes differ from Pillow's
        return out

    monkeypatch.setattr(hw, "encode_png_gpu", broken)
    with pytest.warns(RuntimeWarning, match="encoded with PIL") as rec:
        assert hw.png_layout(64, 48) is None
    assert len(rec) == 1
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        assert hw.png_layout(64, 48) is None               # cached: no second warning
    monkeypatch.setattr(hw, "encode_png_gpu", real)

    img = make_input("noise", 10, 2, 300, 420)
    geo = (128, 16, 8, True)
    n = _n_tiles(img, geo)
    monkeypatch.setattr(hw, "_checked_layout", lambda H, W, device: (_ for _ in ()).throw(ValueError("forced")))
    m = StubMaster(n)
    try:
        with pytest.warns(RuntimeWarning, match="forced") as rec:
            stats = _worker_role(img, geo, m.url)
    finally:
        m.close()
    assert len([w for w in rec if "forced" in str(w.message)]) == 1      # one shape, one warning
    assert sorted(stats["pulled"]) == list(range(n))
    a, = _jobs("noise", 10, 2, 300, 420, *geo)[:1]
    for t in range(n):
        u8 = a.step(t)
        assert [m.files[(t, b)] for b in range(2)] == [hw.encode_png(u8[b]) for b in range(2)], t
