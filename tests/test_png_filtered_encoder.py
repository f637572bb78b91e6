"""The HTTP tile worker's PNG encoder on the host: Pillow's level-0 RGB PNG is a content-free framing (http_worker.
PngLayout, read off the installed Pillow) filled with the filtered stream and the checksums.  The numpy filter rule
(tests/png_filter_model.py) must give Pillow's decompressed stream, and the host model of the whole encoder -- rule,
layout tables, zlib.adler32 / crc32, i.e. what usdu_png_encode_u8 consumes -- must give encode_png's bytes."""
import io
import struct
import zlib

import numpy as np
import pytest

import usdu_oracle as orc
from __graft_entry__ import load_package
from png_filter_model import filter_choice, filtered_stream, host_encode, rechunk, split_cuts

load_package()
from comfyui_distributed_b200 import http_worker as hw  # noqa: E402


def _idat_stream(data: bytes) -> bytes:
    pos, out = 8, b""
    while pos < len(data):
        n, kind = struct.unpack_from(">I4s", data, pos)
        if kind == b"IDAT":
            out += data[pos + 8: pos + 8 + n]
        pos += 12 + n
    return zlib.decompress(out)


def _contents(H, W, seed):
    """The adversarial contents: noise, zeros, a constant, gradients, duplicated rows, values 126..130, the probe."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W]
    dup = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    dup[1::2] = dup[0::2][: H // 2]
    yield "noise", rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    yield "zeros", np.zeros((H, W, 3), np.uint8)
    yield "constant", np.full((H, W, 3), 201, np.uint8)
    yield "gradient", np.stack([(x * 3 + y) % 256, (y * 5) % 256, (x * 7 + y * 2) % 256], -1).astype(np.uint8)
    yield "duplicated", dup
    yield "near128", rng.integers(126, 131, (H, W, 3), dtype=np.uint8)
    yield "probe", hw.png_probe(H, W, seed)


def _processing_sizes():
    """Every distinct tile processing size (ph, pw) the planner gives for the sweep cases and for cfg2 / cfg5."""
    geos = [(7680, 4320, 512, 512, 32, True), (3840, 2160, 1024, 1024, 32, True)]      # cfg2, cfg5
    for W, H in ((520, 700), (700, 520), (900, 640), (300, 420), (1000, 1000)):
        for tile, pad, uniform in ((256, 32, True), (128, 16, False), (384, 0, False), (512, 64, True)):
            geos.append((W, H, tile, tile, pad, uniform))
    sizes = set()
    for W, H, tw, th, pad, uniform in geos:
        for t in orc.make_plan(W, H, tw, th, pad, uniform)[2]:
            sizes.add((t.ph, t.pw))
    return sorted(sizes)


SMALL = [(1, 1), (1, 9), (1, 700), (9, 1), (700, 1), (2, 2), (3, 5), (7, 13), (37, 53), (101, 67), (6, 2560), (3, 2560)]
PROCESSING = _processing_sizes()


def _scan_shapes():
    return SMALL + PROCESSING + [(40, 2560), (1088, 1088), (33, 1999), (29, 2047)]


@pytest.fixture(scope="module")
def framing_scan():
    """Per shape: the layouts of three different contents (noise, a gradient, the probe)."""
    out = {}
    for H, W in _scan_shapes():
        lays = [hw.layout_from_png(hw.encode_png(img)) for _, img in list(_contents(H, W, 3))[::3]]
        out[(H, W)] = lays
    return out


def _split_shapes(scan):
    """Shapes whose Adler trailer or a 5-byte stored-block header straddles two IDAT chunks."""
    found = []
    for shape, lays in scan.items():
        lay = lays[0]
        # the zlib stream = the IDAT data in order; per stream byte its file offset and its chunk
        files = np.concatenate([np.arange(off + 8, off + 8 + n) for off, n in lay.chunks.tolist()])
        chunk = np.concatenate([np.full(n, i) for i, (_, n) in enumerate(lay.chunks.tolist())])
        at = {int(f): i for i, f in enumerate(files)}
        heads = []
        is_r = np.zeros(len(files), bool)
        for f, _, n in lay.runs.tolist():
            is_r[at[f]: at[f] + n] = True
        for f, _, _ in lay.runs.tolist():
            i = at[f]
            if i >= 5 and not is_r[i - 1]:          # a run that starts a stored block follows its 5-byte header
                heads.append(chunk[i - 5: i])
        trailer = chunk[[at[p] for p in lay.adler_at]]
        if any(len(set(h.tolist())) > 1 for h in heads + [trailer]):
            found.append(shape)
    return found


def test_framing_does_not_depend_on_content(framing_scan):
    for shape, lays in framing_scan.items():
        key = lays[0].framing()
        assert all(lay.framing() == key for lay in lays[1:]), shape
        lay = lays[0]
        assert lay.template[lay.chunks[0, 0] + 8: lay.chunks[0, 0] + 10] == b"\x78\x01", shape   # the zlib header
        assert (lay.chunks[:-1, 1] == 65536).all(), shape                  # Pillow's IDAT chunks hold 64 KiB


def test_filter_rule_equals_pillow():
    n = 0
    for H, W in SMALL + PROCESSING[::3] + [(40, 2560)]:
        for name, img in _contents(H, W, H * 7 + W):
            assert filtered_stream(img) == _idat_stream(hw.encode_png(img)), (H, W, name)
            n += 1
    assert n > 100


def test_probe_makes_every_filter_win():
    for H, W in [(7, 4), (12, 40), (64, 2560)] + PROCESSING:
        if H < 7 or W < 4:
            continue
        for v in (0, 1):
            assert set(filter_choice(hw.png_probe(H, W, v)).tolist()) == {0, 1, 2, 4}, (H, W, v)
    p0, p1 = hw.png_probe(40, 30, 0), hw.png_probe(40, 30, 1)
    assert not p0[3].any() and (p0[1] == p0[0]).all() and (p0 != p1).any()


def test_host_model_equals_encode_png(framing_scan):
    split = _split_shapes(framing_scan)          # none so far (test_host_model_on_split_and_long_chunks covers them)
    shapes = SMALL + PROCESSING + [(40, 2560), (1088, 1088)] + split
    for H, W in shapes:
        lay = hw.layout_from_png(hw.encode_png(hw.png_probe(H, W, 0)))
        for name, img in _contents(H, W, H + 3 * W):
            assert host_encode(img, lay) == hw.encode_png(img), (H, W, name)


def test_host_model_on_split_and_long_chunks():
    """No Pillow shape seen splits the trailer or a block header across IDAT chunks; the tables allow it, and a file
    re-cut that way (or into one chunk longer than a CRC span) is reproduced from its own layout."""
    for H, W in [(1, 1), (19, 576), (40, 577), (200, 300)]:
        img = hw.png_probe(H, W, 5)
        pil = hw.encode_png(img)
        for cuts in (split_cuts(pil), []):
            f = rechunk(pil, cuts)
            lay = hw.layout_from_png(f)
            assert host_encode(img, lay) == f, (H, W, cuts)
            other = hw.png_probe(H, W, 6)
            assert host_encode(other, lay) == rechunk(hw.encode_png(other), cuts), (H, W, cuts)


def test_layout_tables():
    lay = hw.layout_from_png(hw.encode_png(hw.png_probe(576, 576, 0)))
    assert lay.raw_len == 576 * 1729 and lay.runs[:, 2].sum() == lay.raw_len
    assert lay.png_len == len(hw.encode_png(np.zeros((576, 576, 3), np.uint8)))
    assert len(lay.chunks) == -(-(lay.chunks[:, 1].sum()) // 65536)
    assert sorted(lay.adler_at) == lay.adler_at and lay.adler_at[3] - lay.adler_at[0] in (3, 15)
    with pytest.raises(ValueError):
        hw.PngLayout(lay.H, lay.W, lay.template, lay.runs[1:], lay.chunks, lay.adler_at)       # R not covered
    with pytest.raises(ValueError):
        hw.PngLayout(lay.H, lay.W, lay.template, lay.runs, lay.chunks, [lay.runs[0, 0]] * 4)  # Adler over R
    with pytest.raises(ValueError):
        hw.layout_from_png(zlib.compress(b"x"))                                                  # not a PNG
    bio = io.BytesIO()
    from PIL import Image
    Image.fromarray(np.zeros((8, 8, 3), np.uint8)).save(bio, format="PNG", compress_level=6)
    with pytest.raises(ValueError):
        hw.layout_from_png(bio.getvalue())                                                      # compressed blocks


def test_step_result_may_be_png_files(monkeypatch):
    """HttpStaticWorker.run takes a step's PNG files as they are and still PIL-encodes a step's u8 tiles."""
    w = hw.HttpStaticWorker("http://127.0.0.1:9", "j", "w", 8, [(0, 0, 4, 4)] * 2, 2)
    sent = []
    queue = [0, 1]
    monkeypatch.setattr(w, "wait_ready", lambda: True)
    monkeypatch.setattr(w, "request_tile", lambda: queue.pop(0) if queue else None)
    monkeypatch.setattr(w, "heartbeat", lambda: None)
    monkeypatch.setattr(w, "send", lambda tiles, final: sent.extend(tiles))
    tiles = np.random.default_rng(0).integers(0, 256, (2, 2, 6, 5, 3), dtype=np.uint8)
    assert w.run(lambda t: [b"png-%d-%d" % (t, b) for b in range(2)] if t == 0 else tiles[t])
    assert [p for p, _ in sent] == [b"png-0-0", b"png-0-1", hw.encode_png(tiles[1][0]), hw.encode_png(tiles[1][1])]
    assert [m["global_idx"] for _, m in sent] == [0, 2, 1, 3]
    queue[:] = [0]
    with pytest.raises(ValueError):
        w.run(lambda t: [b"only one"])
