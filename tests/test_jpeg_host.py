"""The baseline JPEG path on the host: the library's marker parse and Huffman decode (csrc/usdu_jpeg.cpp) followed by
the numpy restatement of the device stages (jpeg_model.py) equals PIL's open().convert("RGB") byte for byte, on files
from Pillow, cv2 and a test-side encoder of arbitrary coefficients; files outside the subset, and damaged files, keep
the refusal every JPEG had before (the PNG parse's), or decode to PIL's bytes, and are never taken where PIL raises."""
import io
import json
import warnings
import zlib

import numpy as np
import pytest
from PIL import Image

import jpeg_model as jm
from __graft_entry__ import load_package

load_package()
from comfyui_distributed_b200 import _native as nat  # noqa: E402
from comfyui_distributed_b200 import http_collector as hc  # noqa: E402
from comfyui_distributed_b200 import http_master as hm  # noqa: E402


def pil_rgb(data: bytes) -> np.ndarray:
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


def model(data: bytes) -> np.ndarray:
    info = hm.parse_jpeg(data)
    return jm.model_decode(info.info, info.quant, info.coefs)


def picture(rng, W, H):
    """Gradients and edges with noise: every quality gives busy and flat blocks."""
    y, x = np.mgrid[:H, :W]
    a = np.stack([x * 255 // max(W - 1, 1), y * 255 // max(H - 1, 1), ((x // 5 + y // 3) * 37) % 256], 2)
    return (a + rng.integers(-40, 41, a.shape)).clip(0, 255).astype(np.uint8)


def pillow(a, **kw) -> bytes:
    b = io.BytesIO()
    Image.fromarray(a).save(b, "JPEG", **kw)
    return b.getvalue()


SIZES = [(1, 1), (7, 7), (8, 8), (9, 9), (15, 15), (16, 16), (17, 17), (33, 33), (577, 433), (1283, 721)]


@pytest.mark.parametrize("W,H", SIZES)
def test_pillow_files_equal_pil(W, H):
    rng = np.random.default_rng(W * 1000 + H)
    a = picture(rng, W, H)
    big = W * H > 100000
    for sub in (0, 1, 2):
        for q in ((75, 95) if big else (1, 50, 75, 95, 100)):
            for opt in ((False,) if big else (False, True)):
                try:
                    data = pillow(a, quality=q, subsampling=sub, optimize=opt)
                except OSError:                       # Pillow's optimize cannot write some 1-row frames
                    continue
                assert np.array_equal(model(data), pil_rgb(data)), (sub, q, opt)
    data = pillow(a[:, :, 1], quality=90)
    assert hm.parse_jpeg(data).info[nat.JI_COMPONENTS] == 1
    assert np.array_equal(model(data), pil_rgb(data))


@pytest.mark.parametrize("kw", [dict(restart_marker_blocks=5), dict(restart_marker_rows=1), dict(keep_rgb=True),
                                dict(keep_rgb=True, subsampling=0, optimize=True), dict(restart_marker_blocks=1)])
def test_pillow_options_equal_pil(kw):
    a = picture(np.random.default_rng(3), 203, 99)
    data = pillow(a, quality=85, **kw)
    info = hm.parse_jpeg(data)
    if "keep_rgb" in kw:
        assert info.info[nat.JI_COLOUR] == nat.JPEG_RGB
    else:
        assert info.info[nat.JI_RESTART] > 0
    assert np.array_equal(model(data), pil_rgb(data))


@pytest.mark.parametrize("W,H", [(9, 9), (577, 433), (1283, 721)])
def test_cv2_files_equal_pil(W, H):
    cv2 = pytest.importorskip("cv2")
    a = picture(np.random.default_rng(5), W, H)
    for q in (30, 90):
        for extra in ([], [cv2.IMWRITE_JPEG_RST_INTERVAL, 3], [cv2.IMWRITE_JPEG_OPTIMIZE, 1]):
            ok, buf = cv2.imencode(".jpg", a, [cv2.IMWRITE_JPEG_QUALITY, q] + extra)
            data = buf.tobytes()
            assert np.array_equal(model(data), pil_rgb(data)), (q, extra)


KINDS = {"ycc": {}, "rgb_adobe": dict(jfif=False, adobe=0), "ycc_adobe": dict(jfif=False, adobe=1),
         "rgb_ids": dict(jfif=False, ids=(82, 71, 66)), "ycc_other_ids": dict(jfif=False, ids=(7, 8, 9))}


@pytest.mark.parametrize("sampling", ["grey", "444", "422", "440", "420"])
@pytest.mark.parametrize("kind", list(KINDS))
def test_encoder_files_equal_pil(sampling, kind):
    """Arbitrary coefficients: small to 16-bit overflowing dequantised values and IDCT sums (libjpeg's SIMD IDCT
    wraps and saturates them), every sampling mode incl. 4:4:0, RGB-coded files, restarts, 16-bit DQT."""
    if sampling == "grey" and kind != "ycc":
        pytest.skip("one component: no colour space")
    nc, h0, v0 = {"grey": (1, 1, 1), "444": (3, 1, 1), "422": (3, 2, 1), "440": (3, 1, 2), "420": (3, 2, 2)}[sampling]
    rng = np.random.default_rng(zlib.crc32(f"{sampling}/{kind}".encode()))
    for W, H in [(1, 1), (3, 5), (9, 9), (17, 33), (64, 48)]:
        for scale, dc, qmax in [(3, 60, 8), (40, 120, 40), (300, 2000, 255), (2000, 16000, 255), (30000, 16000, 3)]:
            blocks = jm.random_blocks(rng, W, H, nc, h0, v0, scale, (-dc, dc))
            for b in blocks:
                np.clip(b, -32767, 32767, out=b)
            quant = [rng.integers(1, qmax + 1, 64) for _ in range(nc)]
            for rst in (0, 1, 3):
                data = jm.encode(blocks, quant, W, H, h0, v0, restart=rst, q16=rst == 3, **KINDS[kind])
                info = hm.parse_jpeg(data)
                assert np.array_equal(info.coefs.reshape(-1, 64), np.concatenate([b.reshape(-1, 64) for b in blocks]))
                assert np.array_equal(jm.model_decode(info.info, info.quant, info.coefs), pil_rgb(data)), \
                    (W, H, scale, rst)


# --------------------------------------------------------------------------------------
# verdicts: outside the subset, and damaged files
# --------------------------------------------------------------------------------------
def today(data: bytes) -> str:
    """The answer every JPEG got before this path: parse_png_any's refusal."""
    with pytest.raises(ValueError) as e:
        hm.parse_png_any(data)
    return str(e.value)


class _Field:
    def __init__(self, raw):
        self.file = io.BytesIO(raw)


def route_answers(data: bytes):
    """-> (submit_tiles' parse, submit_image's parse, job_complete's host path) answers: 'ok' or the error text."""
    import base64
    out = []
    form = {"tiles_metadata": json.dumps([{"tile_idx": 0}]), "tile_0": _Field(data)}
    for fn in (lambda: hm.parse_tiles_from_form(form), lambda: hm.parse_image_any(data),
               lambda: hc.png_of_payload(base64.b64encode(data).decode())):
        try:
            fn()
            out.append("ok")
        except ValueError as e:
            out.append(str(e))
    return out


def refused_as_today(data: bytes):
    msg = today(data)
    assert route_answers(data) == [f"Invalid image data for tile 0: {msg}", msg, f"{hc.PNG_FAILED}{msg}"]


def test_outside_the_subset_keeps_todays_answer():
    a = picture(np.random.default_rng(8), 64, 40)
    cmyk = io.BytesIO()
    Image.fromarray(a).convert("CMYK").save(cmyk, "JPEG", quality=80)
    rng = np.random.default_rng(9)
    files = {"progressive": pillow(a, quality=80, progressive=True), "cmyk": cmyk.getvalue(),
             "411": jm.encode(jm.random_blocks(rng, 64, 40, 3, 4, 1, 5), [np.full(64, 4)] * 3, 64, 40, 4, 1)}
    for name, data in files.items():
        pil_rgb(data)                                 # PIL opens every one of them
        with pytest.raises(ValueError):
            hm.parse_jpeg(data)
        refused_as_today(data)


def test_valid_jpeg_at_the_routes():
    import base64
    data = pillow(picture(np.random.default_rng(1), 40, 30), quality=90)
    assert route_answers(data) == ["ok", "ok", "ok"]
    png, info = hc.png_of_payload(base64.b64encode(data).decode())
    assert png == data and isinstance(info, hm.JpegInfo) and (info.W, info.H) == (40, 30)


def _markers(data: bytes):
    at, out = 2, [2]
    while at < len(data) - 1:
        if data[at] == 0xFF and data[at + 1] not in (0x00, 0xFF):
            out.append(at)
        at += 1
    return out


def corruption_corpus():
    rng = np.random.default_rng(12)
    a = picture(rng, 97, 61)
    bases = [pillow(a, quality=80, restart_marker_blocks=4), pillow(a[:, :, 0], quality=60),
             pillow(a, quality=95, subsampling=0, optimize=True)]
    out = []
    for base in bases:
        ms = _markers(base)
        for m in ms:                                  # truncation at every marker and inside each segment
            out += [base[:m], base[:m + 1], base[:m + 3]]
        scan = base.rindex(b"\xff\xda")
        for _ in range(40):                           # bit flips in the entropy-coded data
            b = bytearray(base)
            k = int(rng.integers(scan + 20, len(b) - 2))
            b[k] ^= 1 << int(rng.integers(0, 8))
            out.append(bytes(b))
        out += [base[:-2], base + b"\x00", base + b"\xff\xd9", base[:-2] + b"\x12\xff\xd9"]
        rst = [i for i in ms if 0xD0 <= base[i + 1] <= 0xD7]
        if len(rst) >= 2:
            b = bytearray(base)
            b[rst[0] + 1], b[rst[1] + 1] = b[rst[1] + 1], b[rst[0] + 1]
            out.append(bytes(b))
            out.append(base[:rst[0]] + base[rst[0] + 2:])
    return out


def test_corruption_corpus_never_taken_where_pil_raises():
    taken = refused = 0
    for data in corruption_corpus():
        try:
            info = hm.parse_jpeg(data)
        except ValueError:
            refused_as_today(data)
            refused += 1
            continue
        taken += 1
        got = jm.model_decode(info.info, info.quant, info.coefs)
        assert np.array_equal(got, pil_rgb(data))     # PIL opens it, to the same bytes
    assert refused > 100 and taken > 0
