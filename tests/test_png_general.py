"""The general PNG path on the host (http_master.parse_png_general): its filtered stream and a numpy model of the
decode against the installed Pillow's convert("RGB") on every colour type, bit depth and interlace method; its verdict
against PIL's on corrupted files; and both masters' routes answering these files as they answer 8-bit RGB PNGs of the
same pixels."""
import asyncio
import base64
import io
import json
import struct
import warnings
import zlib

import numpy as np
import pytest
from PIL import Image

import png_general_model as M
from __graft_entry__ import load_package

load_package()
from comfyui_distributed_b200 import http_collector as hc  # noqa: E402
from comfyui_distributed_b200 import http_master as hm  # noqa: E402
from comfyui_distributed_b200.http_worker import encode_png, multipart  # noqa: E402

CORPUS = M.corpus()


def pil_rgb(data: bytes) -> np.ndarray:
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")             # Pillow's note on palette transparency
        return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


def test_corpus_covers_the_issue():
    names = [n for n, _ in CORPUS]
    assert {n.split("_")[0] for n in names} == {f"c{c}d{d}i{i}" for c, d in M.MODES for i in (0, 1)}
    assert len(M.MODES) == 15
    levels = {n.rsplit("_z", 1)[1] for n in names}
    assert levels == {"0", "6", "9"}


def test_model_equals_pil_on_the_corpus():
    for name, data in CORPUS:
        info = hm.parse_png_any(data)
        eight = name.split("_")[0] in ("c0d8i0", "c2d8i0", "c4d8i0", "c6d8i0")
        if eight:                                   # parse_png's fast path keeps these
            assert isinstance(info, hm.PngInfo), name
            info = hm.parse_png_general(data)
        else:
            assert isinstance(info, hm.PngGeneral), name
            with pytest.raises(hm.UnsupportedPng):
                hm.parse_png(data)
        want = pil_rgb(data)
        assert np.array_equal(M.decode_model(info), want), name
        assert len(info.inflated) == info.raw_len


def test_every_filter_on_every_pass_of_the_corpus():
    seen = set()
    for name, data in CORPUS:
        info = hm.parse_png_general(data)
        R = np.frombuffer(info.inflated, np.uint8)
        for p, (_, _, _, _, pw, ph, at) in enumerate(info.passes()):
            n = 1 + info.row_bytes(pw)
            for f in R[at: at + ph * n: n]:
                seen.add((info.color, info.depth, info.interlace, p, int(f)))
    for c, d in M.MODES:
        for i, passes in ((0, 1), (1, 7)):
            for p in range(passes):
                assert {f for cc, dd, ii, pp, f in seen if (cc, dd, ii, pp) == (c, d, i, p)} == set(range(5)), \
                    (c, d, i, p)


def _rechunk(data: bytes, fn) -> bytes:
    """Rebuild `data` with fn(type, body) -> [(type, body)] applied to every chunk (CRCs recomputed)."""
    out, pos = data[:8], 8
    while pos < len(data):
        ln, ct = struct.unpack_from(">I4s", data, pos)
        for t, b in fn(ct, data[pos + 8: pos + 8 + ln]):
            out += M.chunk(t, b)
        pos += 12 + ln
    return out


def _with_stream(data: bytes, edit, edit_z=lambda z: z) -> bytes:
    """`data` with its filtered stream R replaced by edit(R), recompressed into one IDAT (then edit_z of that)."""
    info = hm.parse_png_general(data)
    z = edit_z(zlib.compress(edit(bytearray(info.inflated)), 6))
    first = []

    def fn(t, b):
        if t != b"IDAT":
            return [(t, b)]
        if first:
            return []
        first.append(1)
        return [(b"IDAT", z)]
    return _rechunk(data, fn)


def _cut_stream(data: bytes) -> bytes:
    """`data` with its zlib stream cut short (the stream never ends), IEND kept."""
    z = hm._IdatStream(data, hm._walk_chunks(data, hm._ihdr_general)[1]).joined()
    first = []

    def fn(t, b):
        if t != b"IDAT":
            return [(t, b)]
        if first:
            return []
        first.append(1)
        return [(b"IDAT", z[: max(3, len(z) - 7)])]
    return _rechunk(data, fn)


def _flip_crc(data: bytes, ctype: bytes) -> bytes:
    at = data.index(ctype) - 4
    ln = struct.unpack_from(">I", data, at)[0]
    q = at + 8 + ln
    return data[:q] + bytes([data[q] ^ 0x40]) + data[q + 1:]


def _corruptions(data: bytes, color: int):
    def set_filter(R, v):
        R[0] = v
        return bytes(R)

    out = [("ihdr_crc", _flip_crc(data, b"IHDR")),
           ("truncated_file", data[: len(data) // 2]),
           ("truncated_stream", _cut_stream(data)),
           ("filter_5", _with_stream(data, lambda R: set_filter(R, 5))),
           ("comp_method", _rechunk(data, lambda t, b: [(t, b[:10] + b"\x01" + b[11:] if t == b"IHDR" else b)])),
           ("interlace_2", _rechunk(data, lambda t, b: [(t, b[:12] + bytes([2 * b[12]]) if t == b"IHDR" else b)])),
           ("filter_method", _rechunk(data, lambda t, b: [(t, b[:11] + b"\x01" + b[12:] if t == b"IHDR" else b)]))]
    # a compressed stream in one IDAT chunk with a broken Adler-32 (PIL checks it when the last row and the checksum
    # reach its decoder together; parse_png_general always checks it)
    out.append(("adler", _with_stream(data, bytes, lambda z: z[:-1] + bytes([z[-1] ^ 1]))))
    if color == 3:
        out += [("plte_crc", _flip_crc(data, b"PLTE")),
                ("no_plte", _rechunk(data, lambda t, b: [] if t == b"PLTE" else [(t, b)])),
                ("odd_plte", _rechunk(data, lambda t, b: [(t, b[:7] if t == b"PLTE" else b)])),
                ("plte_257", _rechunk(data, lambda t, b: [(t, bytes(771) if t == b"PLTE" else b)])),
                ("plte_256_odd", _rechunk(data, lambda t, b: [(t, bytes(770) if t == b"PLTE" else b)]))]
    trns = {0: b"\x00", 2: b"\x00\x01\x00\x02\x00"}.get(color)
    if trns is not None:
        out.append(("short_trns", _rechunk(data, lambda t, b: [(t, b)] + ([(b"tRNS", trns)] if t == b"IHDR" else []))))
    out.append(("trns_crc", _flip_crc(_rechunk(data, lambda t, b: [(t, b)] + (
        [(b"tRNS", M.trns_for(np.random.default_rng(0), color, 8) or b"\x00")] if t == b"IHDR" else [])), b"tRNS")))
    return out


def test_refused_exactly_when_pil_refuses():
    checked = 0
    for name, data in CORPUS[::3]:
        color = data[8 + 8 + 9]
        for what, bad in _corruptions(data, color):
            try:
                want = pil_rgb(bad)
            except Exception:
                want = None
            try:
                info = hm.parse_png_general(bad)
            except ValueError:
                info = None
            assert (info is None) == (want is None), (name, what, want is None)
            if info is not None:
                assert np.array_equal(M.decode_model(info), want), (name, what)
            checked += 1
    assert checked > 1000


def test_other_refusals_stay():
    rng = np.random.default_rng(3)
    x = M.palette_image(rng, 9, 7, 16)
    pal = M.encode_as(rng, x, "pal4")
    with pytest.raises(hm.UnsupportedPng, match="^unsupported PNG: bit depth 4, colour type 3$"):
        hm.parse_png(pal)
    assert isinstance(hm.parse_png_any(pal), hm.PngGeneral)
    # a depth no colour type takes, and rows past the limit, keep their refusals
    bad = _rechunk(pal, lambda t, b: [(t, b[:8] + b"\x03" + b[9:] if t == b"IHDR" else b)])
    with pytest.raises(ValueError, match="bit depth 3, colour type 3"):
        hm.parse_png_any(bad)
    wide = M.make_png(rng, 2, 16, 10923, 1, 0, 1)            # 65,538 filtered bytes
    with pytest.raises(ValueError, match="rows of 65538 bytes"):
        hm.parse_png_any(wide)
    ok = M.make_png(rng, 6, 16, 8192, 1, 1, 1)               # exactly 65,536 bytes, interlaced
    assert hm.parse_png_any(ok).row_bytes(8192) == 65536


# --------------------------------------------------------------------------------------
# both masters' routes
# --------------------------------------------------------------------------------------
FORMATS = ["rgb16", "rgb16_i", "rgba16", "rgba16_i", "la16", "la16_i", "grey16", "grey16_i", "grey1", "grey2_i",
           "grey4", "pal1_i", "pal2", "pal4_i", "pal8", "pal8_i", "rgb8_i"]


def same_pixels(fmt: str, H=24, W=40, seed=0):
    """(u8 RGB image, PNG in `fmt` of it, 8-bit RGB PNG of it)."""
    rng = np.random.default_rng(seed)
    base = fmt.partition("_")[0]
    if base.startswith("pal"):
        x = M.palette_image(rng, H, W, 1 << int(base[3:]))
    elif base in ("grey16", "la16"):
        x = M.grey_image(rng, H, W, 8)
    elif base.startswith("grey"):
        x = M.grey_image(rng, H, W, int(base[4:]))
    else:
        x = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    if base == "rgb8":                               # 8-bit RGB, Adam7
        data = M.make_png(rng, 2, 8, W, H, 1, 6, 2, raw=M.pack_passes(x, 8, 1))
    else:
        data = M.encode_as(rng, x, fmt)
    assert np.array_equal(pil_rgb(data), x)
    return x, data, encode_png(x)


async def _serve(handlers, requests):
    from aiohttp import web
    from aiohttp.test_utils import TestClient, TestServer
    app = web.Application(client_max_size=1 << 30)
    for (method, path), fn in handlers.items():
        app.router.add_route(method, path, fn)
    out = []
    async with TestClient(TestServer(app)) as client:
        for method, path, body, ctype in requests:
            r = await client.request(method, path, data=body, headers={"Content-Type": ctype})
            out.append((r.status, await r.json()))
    return out


def _tile_form(png: bytes, job="jobP"):
    meta = [{"tile_idx": 0, "x": 0, "y": 0, "extracted_width": 40, "extracted_height": 24, "batch_idx": 0,
             "global_idx": 0}]
    fields = [("multi_job_id", job, None, None), ("worker_id", "w1", None, None), ("is_last", "false", None, None),
              ("batch_size", "1", None, None), ("padding", "0", None, None), ("tile_0", png, "t.png", "image/png"),
              ("tiles_metadata", json.dumps(meta), None, "application/json")]
    return multipart([(k, v if isinstance(v, bytes) else str(v).encode(), fn, ct) for k, v, fn, ct in fields])


@pytest.mark.parametrize("fmt", FORMATS)
def test_static_master_routes_take_the_format(fmt):
    x, data, rgb8 = same_pixels(fmt)
    bad = _flip_crc(data, b"IHDR")

    async def go():
        store = hm.JobStore()
        await store.init_job("jobP", 1, [(0, 0, 40, 24, 40, 24)], ["w1"])
        reqs = []
        for png in (data, rgb8, bad):
            reqs.append(("POST", "/distributed/submit_tiles", *_tile_form(png)))
            body, ctype = multipart([("multi_job_id", b"jobP", None, None), ("worker_id", b"w1", None, None),
                                     ("image_idx", b"0", None, None), ("full_image", png, "i.png", "image/png")])
            reqs.append(("POST", "/distributed/submit_image", body, ctype))
        answers = await _serve(hm.make_handlers(store), reqs)
        q = store.jobs["jobP"].queue
        return answers, [q.get_nowait() for _ in range(q.qsize())]

    answers, queued = asyncio.run(go())
    assert answers[0] == answers[2] == (200, {"status": "success"})
    assert answers[1] == answers[3] == (400, {"error": "Job not configured for image submissions"})
    assert answers[4][0] == 400 and answers[4][1]["error"].startswith("Invalid image data for tile 0: bad CRC in IHDR")
    assert answers[5] == (500, {"error": "bad CRC in IHDR"})
    info = queued[0]["tiles"][0]["info"]
    assert isinstance(info, hm.PngGeneral) and np.array_equal(M.decode_model(info), x)
    assert isinstance(queued[1]["tiles"][0]["info"], hm.PngInfo)


@pytest.mark.parametrize("fmt", FORMATS)
def test_collector_route_takes_the_format(fmt):
    x, data, rgb8 = same_pixels(fmt, seed=1)

    def post(png, raw=False):
        image = base64.b64encode(png).decode() if raw else "data:image/png;base64," + base64.b64encode(png).decode()
        return ("POST", "/distributed/job_complete", json.dumps(
            {"job_id": "jobQ", "worker_id": "w1", "batch_idx": 0, "image": image, "is_last": False}).encode(),
            "application/json")

    async def go():
        store = hc.CollectorStore()
        await store.prepare("jobQ")
        answers = await _serve(hc.make_handlers(store, checks=False),
                               [post(data), post(data, True), post(rgb8), post(_flip_crc(data, b"IHDR"))])
        return answers, await store.drain("jobQ")

    answers, items = asyncio.run(go())
    assert answers[0] == answers[1] == answers[2] == (200, {"status": "success"})
    assert answers[3] == (500, {"error": "Failed to decode PNG image payload: bad CRC in IHDR"})
    for it in items[:2]:
        assert isinstance(it["info"], hm.PngGeneral) and it["png"] == data
        assert np.array_equal(M.decode_model(it["info"]), x)
    host = hc.png_of_payload(base64.b64encode(data).decode())
    assert host[0] == data and isinstance(host[1], hm.PngGeneral)
