"""The collector master's device checks, modelled in numpy (tests/b64_model.py): the base64 verdict and bytes against
this interpreter's b64decode(validate=True) on a generated corpus, and the split parse_png (the device table, then
http_collector.check_png_tables on the host) against png_of_payload on the static master's corruption corpus."""
import base64
import struct
import zlib

import numpy as np
import pytest

import b64_model as bm
from test_http_master import _corruptions, image, png_of

hc = bm.hc


def test_corpus_covers_the_cases():
    names = {n for n, _ in bm.corpus()}
    assert {f"len{n}_pad{k}" for n in range(4, 8) for k in range(4)} <= names
    assert {f"byte{v}_{w}" for v in range(256) for w in ("start", "mid", "end")} <= names
    assert {"empty", "non_ascii", "space_inside", "newline_inside", "leading_pad", "after_quad"} <= names


def test_model_agrees_with_the_interpreter():
    accepted = 0
    for name, text in bm.corpus():
        want = bm.interpreter(text)
        assert bm.b64_model(text) == want, name
        accepted += want is not None
    assert accepted > 40


@pytest.mark.parametrize("text,want", [("QUJD=", b"ABC"), ("QUJD===", b"ABC"), ("QR==", b"A"), ("=QUJD", None),
                                       ("QU=D", None), ("QQ=", None), ("QUI", None), ("QQ===", None), ("Q", None),
                                       ("", b""), ("QUI=", b"AB")])
def test_probed_cases(text, want):
    assert bm.interpreter(text) == want
    assert bm.b64_model(text) == want


def _host(image_field):
    try:
        png, info = hc.png_of_payload(image_field)
    except ValueError as e:
        return str(e)
    return png, (info.W, info.H, info.C, info.segs, info.inflated, info.idat, info.trailer)


def _split(text: bytes):
    try:
        png, info = bm.check_model(text)
    except ValueError as e:
        return str(e)
    return png, (info.W, info.H, info.C, info.segs, info.inflated, info.idat, info.trailer)


def _files():
    out = []
    for mode, h, w, level in (("RGB", 544, 544, 0), ("RGBA", 37, 70, 0), ("L", 53, 1, 0), ("LA", 37, 70, 0),
                              ("RGB", 37, 70, 6), ("RGB", 1, 1, 0)):
        data = png_of(image(mode, h, w, 3), level)
        out.append((f"{mode}_{h}x{w}_{level}_good", data))
        out += [(f"{mode}_{h}x{w}_{level}_{name}", bad) for name, bad in _corruptions(data)]
    return out


@pytest.mark.parametrize("name,data", _files(), ids=[n for n, _ in _files()])
def test_split_parse_png_gives_parse_pngs_answer(name, data):
    text = base64.b64encode(data)
    assert _split(text) == _host(text.decode()), name


def _chunk(t, d):
    return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d))


def test_split_on_truncations_and_odd_layouts():
    data = png_of(image("RGBA", 37, 70, 8), 0)
    cases = [data[:k] for k in (1, 7, 8, 12, 20, 33, 40, 41, 45, 47, 60, len(data) - 20, len(data) - 16,
                                len(data) - 12, len(data) - 1)]
    sig, ihdr = data[:8], data[8:33]
    idat = [c for c in _chunks(data) if c[:4] != b"IEND"]
    body = b"".join(c[4:] for c in idat)
    text = _chunk(b"tEXt", b"k\x00" + b"v" * 5000)
    cases += [sig + ihdr + text + b"".join(_chunk(b"IDAT", body[i:i + 999]) for i in range(0, len(body), 999))
              + _chunk(b"IEND", b""),                                    # a chunk before IDAT past the prefix
              sig + ihdr + _chunk(b"IDAT", body[:10]) + _chunk(b"IDAT", body[10:]) + _chunk(b"IHDR", data[16:29]),
              sig + ihdr + _chunk(b"IEND", b""), sig + _chunk(b"IDAT", body),
              sig + ihdr + _chunk(b"IDAT", b"") + _chunk(b"IDAT", body) + _chunk(b"IDAT", b"") + _chunk(b"IEND", b"")]
    for i, bad in enumerate(cases):
        text = base64.b64encode(bad)
        assert _split(text) == _host(text.decode()), i


def _chunks(data):
    pos, out = 8, []
    while pos < len(data):
        ln, = struct.unpack_from(">I", data, pos)
        out.append(data[pos + 4: pos + 12 + ln])
        pos += 12 + ln
    return out


def test_b64_length_rule():
    assert bm.b64_length(0, False, 0, 0) == 0
    assert bm.b64_length(4, False, 4, 4) == 3
    assert bm.b64_length(4, False, 2, 2) == 1 and bm.b64_length(4, False, 3, 3) == 2
    assert bm.b64_length(5, False, 4, 4) == 3                      # '=' after a whole quad
    assert bm.b64_length(3, False, 2, 2) == -1 and bm.b64_length(5, False, 2, 2) == -1
    assert bm.b64_length(4, False, 1, 1) == -1 and bm.b64_length(4, True, 4, 4) == -1
    assert bm.b64_length(4, False, 0, 4) == -1 and bm.b64_length(4, False, 2, 4) == -1


def test_device_png_behaves_as_its_bytes():
    class Ready:
        def synchronize(self):
            pass

    class Buf:
        def __init__(self, b):
            self.b = b

        def __getitem__(self, k):
            return self

        def cpu(self):
            return self

        def numpy(self):
            return np.frombuffer(self.b, np.uint8)

    p = hc.DevicePng(Buf(b"\x89PNGxyz"), 7, Ready())
    assert len(p) == 7 and p == b"\x89PNGxyz" and bytes(p) == b"\x89PNGxyz" and p[1:4] == b"PNG"
    assert p != b"other" and not (p == 3)


def test_pool_bound():
    pool = hc.DevicePool(100)
    pool.used = 90
    assert pool.take(11, None, None) is None and pool.used == 90
    pool.give(90)
    assert pool.used == 0 and hc.POOL_BYTES == 4 << 30
