"""Verdicts at the edges of the JPEG subset: sides over libjpeg's 65,500 limit, and APPn segments PIL's Python header
parse (Image.open) raises on.  Each such file keeps the answer every JPEG had before (the PNG parse's refusal) at all
three routes; the files next to them that PIL opens decode to PIL's bytes."""
import io
import warnings

import numpy as np
import pytest
from PIL import Image

import jpeg_model as jm
from __graft_entry__ import load_package
from test_jpeg_host import pil_rgb, refused_as_today

load_package()
from comfyui_distributed_b200 import _native as nat  # noqa: E402
from comfyui_distributed_b200 import http_master as hm  # noqa: E402


def pil_raises(data: bytes) -> bool:
    try:
        pil_rgb(data)
        return False
    except Exception:
        return True


def grey(W, H) -> bytes:
    rng = np.random.default_rng(W + H)
    return jm.encode(jm.random_blocks(rng, W, H, 1, 1, 1, 2), [np.full(64, 3)], W, H)


def taken_as_pil(data: bytes):
    info = hm.parse_jpeg(data)
    assert np.array_equal(jm.model_decode(info.info, info.quant, info.coefs), pil_rgb(data))


@pytest.mark.parametrize("W,H", [(65501, 1), (65535, 1), (1, 65535), (1, 65501)])
def test_side_over_65500_is_refused(W, H):
    data = grey(W, H)
    assert pil_raises(data)
    with pytest.raises(ValueError, match="65,500|65500"):
        nat.jpeg_parse(data)
    refused_as_today(data)


@pytest.mark.parametrize("W,H", [(65500, 1), (1, 65500)])
def test_side_of_65500_is_taken(W, H):
    taken_as_pil(grey(W, H))


def with_segment(marker: int, body: bytes) -> bytes:
    rng = np.random.default_rng(16)
    base = jm.encode(jm.random_blocks(rng, 16, 16, 3, 2, 2, 5), [np.full(64, 4)] * 3, 16, 16, 2, 2)
    return base[:2] + bytes([0xFF, marker]) + (len(body) + 2).to_bytes(2, "big") + body + base[2:]


BAD_EXIF = bytes.fromhex("4578696600004d4d002a000000080003010f00020000000463616d00011a00070000000100000067012800030000"
                         "000100020000000000000000004800000001")
REFUSED = {"jfif_4": (0xE0, b"JFIF"), "jfif_6": (0xE0, b"JFIF\0\x01"), "adobe_5": (0xEE, b"Adobe"),
           "adobe_6": (0xEE, b"Adobe\0"), "icc_12": (0xE2, b"ICC_PROFILE\0"), "icc_13": (0xE2, b"ICC_PROFILE\0\x01"),
           "photoshop_cut": (0xED, b"Photoshop 3.0\0" + b"8BIM\x04\x04"), "bad_exif": (0xE1, BAD_EXIF)}


@pytest.mark.parametrize("name", list(REFUSED))
def test_app_segments_pil_raises_on_are_refused(name):
    data = with_segment(*REFUSED[name])
    assert pil_raises(data)
    with pytest.raises(ValueError):
        hm.parse_jpeg(data)
    refused_as_today(data)
    if name != "bad_exif":                          # the library alone refuses these; Exif is PIL's header verdict
        with pytest.raises(ValueError):
            nat.jpeg_parse(data)


def test_mpf_segment_is_refused():
    data = with_segment(0xE2, b"MPF\0" + bytes(16))
    with pytest.raises(ValueError, match="MPF"):
        nat.jpeg_parse(data)
    refused_as_today(data)


def _exif() -> bytes:
    ex = Image.Exif()
    ex[0x011A], ex[0x0128], ex[0x010F] = (72, 1), 2, "camera"
    return ex.tobytes()


TAKEN = {"jfif_7": (0xE0, b"JFIF\0\x01\x02"), "adobe_7": (0xEE, b"Adobe\0\x64"), "icc_14": (0xE2, b"ICC_PROFILE\0\x01\x01"),
         "photoshop": (0xED, b"Photoshop 3.0\0" + b"8BIM\x03\xed\x00\x00" + (16).to_bytes(4, "big") + bytes(16)),
         "photoshop_short_info": (0xED, b"Photoshop 3.0\0" + b"8BIM\x03\xed\x00\x00" + (4).to_bytes(4, "big") + bytes(4)),
         "exif": (0xE1, _exif()), "xmp": (0xE1, b"http://ns.adobe.com/xap/1.0/\0<x/>"), "app9": (0xE9, b"")}


@pytest.mark.parametrize("name", list(TAKEN))
def test_app_segments_pil_reads_are_taken(name):
    data = with_segment(*TAKEN[name])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        assert not pil_raises(data)
    taken_as_pil(data)
