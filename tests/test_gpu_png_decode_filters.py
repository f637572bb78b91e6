"""The PNG decode kernel (usdu_png_decode_u8, csrc/usdu_png_decode.cu) on synthetic files whose filters, stored blocks and
IDAT chunks the test chooses (test_png_layouts.cases): every filter sequence, chunk edge, ring depth, segment layout and
launch shape there must decode to the pixels the file was written from, with nothing written outside the frames.  And
the GPU encoder (usdu_png_base64_u8) round-tripped through PIL and through parse_png + the decode kernel."""
import base64
import io

import numpy as np
import pytest
import torch
from PIL import Image

import usdu_oracle as orc
from __graft_entry__ import load_package
from test_gpu_collector_master import _steps
from test_gpu_http_master import decode_on_gpu
from test_png_layouts import STORED_MAX, depth_steps, launches, rgb, ring_depth

load_package()
from comfyui_distributed_b200 import _native as nat  # noqa: E402
from comfyui_distributed_b200 import http_master as hm  # noqa: E402
from comfyui_distributed_b200.nodes import collector  # noqa: E402

pytestmark = pytest.mark.gpu
SENTINEL = 0xA5


def _decode_and_check(pngs, wants, names, seed):
    """One launch over `pngs`; frame i lands at an odd byte offset after a gap of 1..9 bytes and must equal wants[i]
    ([H, W, 3] u8); every other byte of the output keeps the sentinel."""
    rng = np.random.default_rng(seed)
    offs, cur = [], 1
    for w in wants:
        offs.append(cur)
        cur += w.size + int(rng.integers(0, 5)) * 2 + 1
    out = decode_on_gpu(pngs, offs, cur + 8)
    outside = np.ones(out.size, bool)
    for o, w, name in zip(offs, wants, names):
        got = out[o: o + w.size].reshape(w.shape)
        if not np.array_equal(got, w):
            bad = np.argwhere(got != w)
            pytest.fail(f"{name}: {len(bad)} wrong bytes, first at (row, x, channel) {tuple(bad[0])}")
        outside[o: o + w.size] = False
    assert (out[outside] == SENTINEL).all(), "bytes outside the frames were written"


@pytest.mark.timeout(120)
def test_depth_model_is_the_device():
    """The ring depths test_png_layouts builds its cases for are the ones the kernel picks on this device."""
    assert _steps() == depth_steps()
    for name, cases in launches().items():
        row = max(c.shape[1] * c.shape[2] for c in cases)
        assert nat.png_decode_warps(row) == ring_depth(row), name


@pytest.mark.timeout(300)
@pytest.mark.parametrize("launch", list(launches()))
def test_decode_equals_source_pixels(launch):
    cases = launches()[launch]
    _decode_and_check([c.data for c in cases], [rgb(c.px) for c in cases], [repr(c) for c in cases],
                      seed=len(cases))


# --------------------------------------------------------------------------------------
# the GPU encoder, decoded by PIL and by the decode kernel
# --------------------------------------------------------------------------------------
def _shape_with_raw_len(C, raw, rows_on_blocks=False):
    """(H, W) with H * (1 + W * C) == raw, W as large as possible below 600, H >= 2; None if there is none.
    rows_on_blocks: also a row boundary at every multiple of 65535 (a row's filter byte opens each stored block)."""
    for W in range(600, 0, -1):
        L = 1 + W * C
        if raw % L == 0 and raw // L >= 2 and (not rows_on_blocks or STORED_MAX % L == 0):
            return raw // L, W
    return None


def _round_trip_shapes():
    """For C in 2..4: |R| = k * 65535 - 1, k * 65535 and k * 65535 + 1, each with the smallest k that has a shape, and
    |R| = 2 * 65535 with the second stored block starting at a row's filter byte."""
    out = []
    for C in (2, 3, 4):
        for delta in (-1, 0, 1):
            shape = next(s for k in range(1, 64) if (s := _shape_with_raw_len(C, k * STORED_MAX + delta)))
            out.append((C,) + shape)
        out.append((C,) + _shape_with_raw_len(C, 2 * STORED_MAX, rows_on_blocks=True))
    return out


@pytest.mark.timeout(300)
def test_encoder_round_trip():
    shapes = _round_trip_shapes()
    rows_on_block_starts = 0
    pngs, wants, names = [], [], []
    for i, (C, H, W) in enumerate(shapes):
        g = torch.Generator().manual_seed(40 + i)
        x = (torch.rand((3, H, W, C), generator=g) * 1.02 - 0.01).cuda()      # a few values outside [0, 1]
        q = orc.quantize_u8(x.cpu().numpy())
        L = 1 + W * C
        rows_on_block_starts += sum(r * L % STORED_MAX == 0 for r in range(1, H))
        for b, text in enumerate(collector._native_png_b64(collector._native_pack(x))):
            data = base64.b64decode(bytes(text), validate=True)
            pil = np.asarray(Image.open(io.BytesIO(data)))
            assert np.array_equal(pil, q[b]), (C, H, W, b)
            info = hm.parse_png(data)
            assert (info.H, info.W, info.C, info.inflated) == (H, W, C, None)
            assert len(info.segs) == -(-info.raw_len // STORED_MAX)          # each stored block in its own IDAT
            pngs.append(data)
            wants.append(rgb(q[b]))
            names.append(f"C{C} {H}x{W} frame {b}")
    assert rows_on_block_starts > 0                      # a row's filter byte opens a stored block
    assert {(H * (1 + W * C)) % STORED_MAX for C, H, W in shapes} == {STORED_MAX - 1, 0, 1}
    _decode_and_check(pngs, wants, names, seed=7)
