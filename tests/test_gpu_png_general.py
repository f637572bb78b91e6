"""The general PNG decode on the GPU (usdu_png_decode_general_u8): every colour type, bit depth and interlace method of
the generated corpus in one launch and large frames against the installed Pillow; a static-mode HttpStaticMaster job
and a collector master job whose workers post palette, 16-bit and Adam7 PNGs against the same jobs with 8-bit PNGs of
the same pixels."""
import asyncio
import io
import json
import threading
import warnings

import numpy as np
import pytest
import torch
from PIL import Image

import png_general_model as M
from __graft_entry__ import load_package
from test_http_collector import JOB, Ours, body, post

load_package()
from comfyui_distributed_b200 import engine  # noqa: E402
from comfyui_distributed_b200 import http_master as hm  # noqa: E402
from comfyui_distributed_b200.denoise import T0Denoiser  # noqa: E402
from comfyui_distributed_b200.http_worker import _call, encode_png, multipart  # noqa: E402
from comfyui_distributed_b200.nodes import collector  # noqa: E402

pytestmark = pytest.mark.gpu


def pil_rgb(data: bytes) -> np.ndarray:
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


def decode_general(infos):
    """One launch over every frame of `infos` -> [u8 [H, W, 3]], with guard bytes between the frames."""
    offs, cur = [], 0
    for info in infos:
        offs.append(cur)
        cur += info.H * info.W * 3 + 13
    dst = torch.full((cur + 16,), 0xA5, dtype=torch.uint8, device="cuda")
    dec = hm.PngDecoder(torch.device("cuda"))
    dec.decode_general(list(zip(infos, offs)), dst)
    torch.cuda.synchronize()
    host = dst.cpu().numpy()
    for o, info in zip(offs, infos):                 # nothing written outside the frames
        assert (host[o + info.H * info.W * 3: o + info.H * info.W * 3 + 13] == 0xA5).all()
    dec.release()
    return [host[o: o + i.H * i.W * 3].reshape(i.H, i.W, 3) for o, i in zip(offs, infos)]


def test_corpus_in_one_launch():
    corpus = M.corpus(seed=7)
    infos = [hm.parse_png_general(d) for _, d in corpus]
    for (name, data), got in zip(corpus, decode_general(infos)):
        assert np.array_equal(got, pil_rgb(data)), name


@pytest.mark.parametrize("what", ["rgb16_4k", "pal8_adam7_4k", "grey16_4k", "rgba16_row_65536", "grey1_row_65536",
                                  "pal4_adam7_row_65536"])
def test_large_frames(what):
    rng = np.random.default_rng(11)
    if what == "rgb16_4k":
        data = M.make_png(rng, 2, 16, 3840, 2160, 0, 1, 4)
    elif what == "pal8_adam7_4k":
        data = M.make_png(rng, 3, 8, 3840, 2160, 1, 1, 4, plte_entries=200)
    elif what == "grey16_4k":
        data = M.make_png(rng, 0, 16, 3840, 2160, 0, 1, 4)
    elif what == "rgba16_row_65536":
        data = M.make_png(rng, 6, 16, 8192, 9, 0, 1, 2)
    elif what == "grey1_row_65536":
        data = M.make_png(rng, 0, 1, 65536 * 8, 3, 0, 1, 2)
    else:
        data = M.make_png(rng, 3, 4, 65536 * 2, 9, 1, 1, 2, plte_entries=9)
    info = hm.parse_png_general(data)
    if "row_65536" in what:
        assert max(info.row_bytes(p[4]) for p in info.passes()) == 65536
    (got,) = decode_general([info])
    assert np.array_equal(got, pil_rgb(data))


# --------------------------------------------------------------------------------------
# a static-mode job: every tile posted by a worker, as 8-bit RGB or in the new formats
# --------------------------------------------------------------------------------------
TILE_FORMATS = ["rgb16", "pal8_i", "rgba16_i", "pal4", "grey16", "rgb8", "rgb16_i", "la16_i", "grey2", "rgb8_i"]


def _tile_pixels(rng, fmt, h, w):
    base = fmt.partition("_")[0]
    if base.startswith("pal"):
        return M.palette_image(rng, h, w, 1 << int(base[3:]))
    if base in ("grey16", "la16"):
        return M.grey_image(rng, h, w, 8)
    if base.startswith("grey"):
        return M.grey_image(rng, h, w, int(base[4:]))
    return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)


def _encode(rng, x, fmt):
    if fmt == "rgb8":                                 # parse_png's 8-bit fast path, in the same batches
        return encode_png(x)
    if fmt == "rgb8_i":
        return M.make_png(rng, 2, 8, x.shape[1], x.shape[0], 1, 6, 2, raw=M.pack_passes(x, 8, 1))
    return M.encode_as(rng, x, fmt)


def _static_job(general: bool):
    """A 2-frame job whose worker takes every tile and posts it; frame b of tile t is _tile_pixels(TILE_FORMATS[t]),
    as 8-bit RGB (general False) or in that format.  -> (result numpy, master stats)."""
    from aiohttp import web
    loop = asyncio.new_event_loop()
    th = threading.Thread(target=loop.run_forever, daemon=True)
    th.start()
    call = lambda c: asyncio.run_coroutine_threadsafe(c, loop).result(60)     # noqa: E731
    store = hm.JobStore()
    routes = web.RouteTableDef()
    hm.register(routes, store, loop)
    app = web.Application(client_max_size=1 << 30)
    app.add_routes(routes)
    runner = web.AppRunner(app)
    call(runner.setup())
    import socket
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    call(web.TCPSite(runner, "127.0.0.1", port).start())
    url = f"http://127.0.0.1:{port}"
    try:
        x = torch.from_numpy(np.random.default_rng(2).random((2, 300, 420, 3), dtype=np.float32))
        job = engine.WorkerJob(x, T0Denoiser(5, 0.5), 128, 128, 16, 8, True)
        master = hm.HttpStaticMaster(job, "jobS", ["w1"], store, loop)
        call(store.init_job("jobS", master.B, master.geometry, ["w1"]))
        tids = []
        while True:                                   # the worker takes every tile before the master asks for one
            st, text = _call(url + "/distributed/request_image", "POST",
                             json.dumps({"worker_id": "w1", "multi_job_id": "jobS"}).encode(), "application/json")
            tid = json.loads(text)["tile_idx"]
            if tid is None:
                break
            tids.append(tid)
        assert sorted(tids) == list(range(master.T)) and master.T >= 6
        rng = np.random.default_rng(9)
        for k, tid in enumerate(tids):
            x1, y1, ew, eh, pw, ph = master.geometry[tid]
            fmt = TILE_FORMATS[tid % len(TILE_FORMATS)]
            fields = [("multi_job_id", b"jobS", None, None), ("worker_id", b"w1", None, None),
                      ("is_last", b"true" if k == len(tids) - 1 else b"false", None, None),
                      ("batch_size", b"2", None, None), ("padding", b"16", None, None)]
            meta = []
            for b in range(2):
                px = _tile_pixels(np.random.default_rng(1000 * tid + b), fmt, ph, pw)
                png = _encode(rng, px, fmt) if general else encode_png(px)
                assert np.array_equal(pil_rgb(png), px)
                fields.append((f"tile_{b}", png, f"t{b}.png", "image/png"))
                meta.append({"tile_idx": tid, "x": x1, "y": y1, "extracted_width": ew, "extracted_height": eh,
                             "batch_idx": b, "global_idx": b * master.T + tid})
            fields.append(("tiles_metadata", json.dumps(meta).encode(), None, "application/json"))
            st, text = _call(url + "/distributed/submit_tiles", "POST", *multipart(fields))
            assert st == 200, text
        out = master.run()
        torch.cuda.synchronize()
        return out.cpu().numpy(), dict(master.stats), master.assignment()
    finally:
        call(runner.cleanup())
        loop.call_soon_threadsafe(loop.stop)
        th.join(10)


def test_static_master_job_with_general_tiles():
    want, st8, a8 = _static_job(False)
    got, stg, ag = _static_job(True)
    assert a8 == ag and a8[0] == []                  # every tile came from the worker
    assert stg["tiles_received"] == st8["tiles_received"] == 2 * len(a8[1])
    assert stg["decode_launches"] >= 2                # the general entry and the 8-bit one, per drained batch
    assert np.array_equal(got, want)


# --------------------------------------------------------------------------------------
# a collector job: frames posted in the new formats, through the device checks
# --------------------------------------------------------------------------------------
def _collector(master, posts):
    with Ours() as ours:
        out = {}
        t = threading.Thread(target=lambda: out.update(r=collector.DistributedCollectorNode().run(
            master, multi_job_id=JOB, enabled_worker_ids=json.dumps(["w1", "w2"]))))
        t.start()
        for raw in posts:
            assert post(ours.url, raw)[0] == 200
        t.join(300)
        assert "r" in out
        return out["r"][0]


@pytest.mark.timeout(600)
def test_collector_job_with_general_frames():
    H, W = 180, 260
    fmts = ["pal8_i", "rgb16", "grey16_i", "rgba16", "pal2", "rgb8_i", "la16"]
    frames = [_tile_pixels(np.random.default_rng(50 + i), f, H, W) for i, f in enumerate(fmts)]
    rng = np.random.default_rng(4)
    general = [_encode(rng, x, f) for x, f in zip(frames, fmts)]
    eight = [encode_png(x) for x in frames]
    master = torch.rand(1, H, W, 3, device="cuda")

    def posts(pngs):
        return [body("w1" if i % 2 else "w2", i // 2, p, i >= len(pngs) - 2) for i, p in enumerate(pngs)]

    want = _collector(master, posts(eight))
    got = _collector(master, posts(general))
    assert got.shape == (1 + len(fmts), H, W, 3)
    assert torch.equal(got, want)
