"""The baseline JPEG decode on the GPU (usdu_jpeg_decode_u8) against the installed Pillow: the host corpus frame by
frame, batches of up to 81 frames in one launch, batches that mix PNG and JPEG frames; a static-mode HttpStaticMaster
job whose worker posts JPEG tiles, and a collector master job fed JPEG POSTs, each against the same job fed PNGs of
PIL's decode of those JPEGs."""
import io

import numpy as np
import pytest
import torch
from PIL import Image

import jpeg_model as jm
from __graft_entry__ import load_package
from test_gpu_png_general import _collector, pil_rgb
from test_http_collector import body
from test_jpeg_host import SIZES, corruption_corpus, picture, pillow

load_package()
from comfyui_distributed_b200 import http_master as hm  # noqa: E402
from comfyui_distributed_b200.http_worker import encode_png  # noqa: E402

pytestmark = pytest.mark.gpu


def decode(items):
    """items: (info, posted bytes) -> [u8 [H, W, 3]], every frame in one PngDecoder.decode call (one launch per kind),
    with guard bytes between the frames."""
    offs, cur = [], 0
    for info, _ in items:
        offs.append(cur)
        cur += info.H * info.W * 3 + 13
    dst = torch.full((cur + 16,), 0xA5, dtype=torch.uint8, device="cuda")
    dec = hm.PngDecoder(torch.device("cuda"))
    launches = dec.decode([(info, raw, o) for (info, raw), o in zip(items, offs)], dst)
    torch.cuda.synchronize()
    host = dst.cpu().numpy()
    for o, (info, _) in zip(offs, items):
        assert (host[o + info.H * info.W * 3: o + info.H * info.W * 3 + 13] == 0xA5).all()
    dec.release()
    return [host[o: o + i.H * i.W * 3].reshape(i.H, i.W, 3) for o, (i, _) in zip(offs, items)], launches


def corpus():
    out = []
    for W, H in SIZES:
        a = picture(np.random.default_rng(W + H), W, H)
        for sub in (0, 1, 2):
            for q in (1, 75, 100):
                out.append(pillow(a, quality=q, subsampling=sub, optimize=q == 75))
        out.append(pillow(a[:, :, 0], quality=90))
        out.append(pillow(a, quality=85, restart_marker_rows=1, keep_rgb=W % 2 == 1))
    rng = np.random.default_rng(3)
    for nc, h0, v0 in [(1, 1, 1), (3, 1, 1), (3, 2, 1), (3, 1, 2), (3, 2, 2)]:
        for W, H in [(3, 5), (17, 33), (200, 70)]:
            for scale, dc, qmax in [(40, 120, 40), (2000, 16000, 255)]:
                blocks = jm.random_blocks(rng, W, H, nc, h0, v0, scale, (-dc, dc))
                for b in blocks:
                    np.clip(b, -32767, 32767, out=b)
                quant = [rng.integers(1, qmax + 1, 64) for _ in range(nc)]
                out.append(jm.encode(blocks, quant, W, H, h0, v0, jfif=W != 17, adobe=0 if W == 17 else None))
    return out


def test_corpus_frame_by_frame_and_in_batches():
    files = corpus()
    infos = [(hm.parse_jpeg(d), d) for d in files]
    refs = [pil_rgb(d) for d in files]
    for item, ref in zip(infos, refs):
        (got,), n = decode([item])
        assert n == 1 and np.array_equal(got, ref)
    for k in range(0, len(infos), 81):               # batches of up to 81 frames
        got, n = decode(infos[k: k + 81])
        assert n == 1
        for g, ref in zip(got, refs[k: k + 81]):
            assert np.array_equal(g, ref)


def test_corruption_corpus_taken_files():
    taken = []
    for d in corruption_corpus():
        try:
            taken.append((hm.parse_jpeg(d), d))
        except ValueError:
            pass
    got, _ = decode(taken)
    for g, (_, d) in zip(got, taken):
        assert np.array_equal(g, pil_rgb(d))


def test_batches_mixing_png_and_jpeg():
    rng = np.random.default_rng(5)
    items, refs = [], []
    for i in range(40):
        W, H = int(rng.integers(1, 300)), int(rng.integers(1, 200))
        a = picture(rng, W, H)
        if i % 3 == 0:
            raw = encode_png(a)
            refs.append(a)
        else:
            raw = pillow(a, quality=int(rng.integers(10, 100)), subsampling=int(rng.integers(0, 3)))
            refs.append(pil_rgb(raw))
        items.append((hm.parse_image_any(raw), raw))
    got, n = decode(items)
    assert n == 2
    for g, ref in zip(got, refs):
        assert np.array_equal(g, ref)


@pytest.mark.parametrize("W,H,sub", [(3840, 2160, 2), (3840, 2160, 0), (1920, 1080, 1), (4001, 37, 2)])
def test_large_frames(W, H, sub):
    data = pillow(picture(np.random.default_rng(1), W, H), quality=90, subsampling=sub)
    (got,), _ = decode([(hm.parse_jpeg(data), data)])
    assert np.array_equal(got, pil_rgb(data))


# --------------------------------------------------------------------------------------
# the masters
# --------------------------------------------------------------------------------------
def test_static_master_job_with_jpeg_tiles(monkeypatch):
    """Every third tile of the worker arrives as a JPEG: the result equals the same job with every tile a PNG of
    PIL's decode of what was posted (test_gpu_http_master holds that job to usdu_oracle.replay_static)."""
    import test_gpu_png_general as G
    encs, source = {}, {}

    def as_jpeg(rng, x, fmt):
        key = x.tobytes()
        if key not in encs:
            encs[key] = pillow(x, quality=int(rng.integers(40, 96)), subsampling=int(rng.integers(0, 3)))
            source[encs[key]] = x
        return encs[key]

    monkeypatch.setattr(G, "_tile_pixels", lambda rng, fmt, h, w: picture(rng, w, h))
    monkeypatch.setattr(G, "TILE_FORMATS", ["jpeg", "png", "png"])
    monkeypatch.setattr(G, "_encode", lambda rng, x, fmt: as_jpeg(rng, x, fmt) if fmt == "jpeg" else encode_png(x))
    # the harness checks each posted file against its pixels: a JPEG stands for the pixels it was made from
    monkeypatch.setattr(G, "pil_rgb", lambda data: source[data] if data in source else pil_rgb(data))
    got, stj, aj = G._static_job(True)
    # the same job, each JPEG tile replaced by the PNG of PIL's decode of it
    def as_png_of_jpeg(rng, x, fmt):
        png = encode_png(pil_rgb(as_jpeg(rng, x, fmt)))
        source[png] = x
        return png

    monkeypatch.setattr(G, "_encode", lambda rng, x, fmt: as_png_of_jpeg(rng, x, fmt) if fmt == "jpeg" else
                        encode_png(x))
    want, stp, ap = G._static_job(True)
    assert aj == ap and aj[0] == []
    assert stj["tiles_received"] == stp["tiles_received"] and stj["decode_launches"] > stp["decode_launches"]
    assert np.array_equal(got, want)


@pytest.mark.timeout(600)
def test_collector_job_with_jpeg_frames():
    H, W = 180, 260
    rng = np.random.default_rng(4)
    frames = [picture(rng, W, H) for _ in range(7)]
    jpegs = [pillow(x, quality=q, subsampling=s) for x, q, s in zip(frames, (95, 75, 50, 90, 30, 85, 99),
                                                                     (2, 0, 1, 2, 2, 0, 1))]
    pngs = [encode_png(pil_rgb(j)) for j in jpegs]
    master = torch.rand(1, H, W, 3, device="cuda")

    def posts(raws):
        return [body("w1" if i % 2 else "w2", i // 2, p, i >= len(raws) - 2) for i, p in enumerate(raws)]

    want = _collector(master, posts(pngs))
    got = _collector(master, posts(jpegs))
    assert got.shape == (1 + len(jpegs), H, W, 3)
    assert torch.equal(got, want)
