"""Synthetic PNGs for the decode kernel (csrc/usdu_png_decode.cu): a writer that controls each row's filter, the stored
deflate blocks and the IDAT chunks, and the case list test_gpu_png_decode_filters.py decodes on the GPU.  Filtering is
invertible, so a correct decode returns the pixels a case started from.  On the host: every file opens in PIL as those
pixels, passes http_master.parse_png, and its filtered stream and http_master.unfilter_model match the writer's; and the
case list reaches every filter pair, ring depth, chunk edge and segment layout the kernel handles differently."""
import functools
import io
import struct
import zlib
from collections import defaultdict

import numpy as np
import pytest
from PIL import Image

from __graft_entry__ import load_package

load_package()
from comfyui_distributed_b200 import http_master as hm  # noqa: E402

NONE, SUB, UP, AVG, PAETH = range(5)
COLOUR_TYPE = {1: 0, 2: 4, 3: 2, 4: 6}       # L, LA, RGB, RGBA
STORED_MAX = 65535

# The decode kernel's ring depth (warps per CTA) on an H100: min(16, (opt-in shared memory per block - the kernel's
# static shared memory) // widest row bytes of the launch).  test_gpu_png_decode_filters.py checks this model against
# usdu_png_decode_warps on the device.
H100_SMEM_OPTIN = 232448
DECODE_STATIC_SMEM = 64                      # the 16 progress counters
MAX_DEPTH, MAX_ROW = 16, 65536


def ring_depth(row_bytes: int) -> int:
    return min(MAX_DEPTH, (H100_SMEM_OPTIN - DECODE_STATIC_SMEM) // row_bytes)


def depth_steps():
    """(depth, widest row bytes at that depth) for every depth up to MAX_ROW, deepest first."""
    return [(d, min(MAX_ROW, (H100_SMEM_OPTIN - DECODE_STATIC_SMEM) // d)) for d in range(MAX_DEPTH, 2, -1)]


# --------------------------------------------------------------------------------------
# the writer
# --------------------------------------------------------------------------------------
def predictors(px: np.ndarray):
    """(a, b, c) per byte of [H, W, C] u8 pixels as int32 [H, W*C]: left, up and upper-left, zero outside the image."""
    H, W, C = px.shape
    x = px.reshape(H, W * C).astype(np.int32)
    b = np.vstack([np.zeros((1, W * C), np.int32), x[:-1]])
    a = np.hstack([np.zeros((H, C), np.int32), x[:, :-C]])
    c = np.hstack([np.zeros((H, C), np.int32), b[:, :-C]])
    return x, a, b, c


def paeth(a, b, c):
    """The PNG Paeth predictor; ties go to a, then b, then c."""
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def filter_rows(px: np.ndarray, filters) -> bytes:
    """The filtered stream R of [H, W, C] u8 pixels: row r is filters[r], then its W*C bytes filtered with it."""
    H = px.shape[0]
    assert len(filters) == H and all(0 <= f <= 4 for f in filters)
    x, a, b, c = predictors(px)
    pred = np.stack([np.zeros_like(x), a, b, (a + b) >> 1, paeth(a, b, c)])      # [filter, H, W*C]
    f = np.asarray(filters, np.int64)
    res = (x - pred[f, np.arange(H)]) & 0xFF
    return np.hstack([f[:, None].astype(np.uint8), res.astype(np.uint8)]).tobytes()


def cut(n: int, sizes) -> list:
    """n bytes cut into pieces of sizes[0], sizes[1], ... (cycling; zeros give empty pieces), the last one short."""
    assert any(sizes)
    out, i = [], 0
    while n > 0:
        s = min(sizes[i % len(sizes)], n)
        out.append(s)
        n -= s
        i += 1
    return out


def zlib_stored(R: bytes, blocks) -> bytes:
    """A zlib stream holding R in stored deflate blocks of the given sizes (cut), the last one marked final."""
    assert max(blocks) <= STORED_MAX
    out, pos = [b"\x78\x01"], 0
    pieces = cut(len(R), blocks)
    for i, ln in enumerate(pieces):
        out.append(bytes([i == len(pieces) - 1]) + struct.pack("<HH", ln, ln ^ 0xFFFF) + R[pos: pos + ln])
        pos += ln
    out.append(struct.pack(">I", zlib.adler32(R)))
    return b"".join(out)


def _chunk(kind: bytes, data: bytes) -> bytes:
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(kind + data))


def png(px: np.ndarray, filters, blocks=(STORED_MAX,), chunks=(1 << 20,), compressed=False) -> bytes:
    """An 8-bit PNG of [H, W, C] u8 pixels (C = 1..4: L, LA, RGB, RGBA) with row r filtered by filters[r], R stored in
    deflate blocks of the sizes `blocks` (or deflated by zlib at level 9 if `compressed`), and the zlib stream cut into
    IDAT chunks of the sizes `chunks`."""
    H, W, C = px.shape
    R = filter_rows(px, filters)
    z = zlib.compress(R, 9) if compressed else zlib_stored(R, blocks)
    out = [hm.PNG_SIGNATURE, _chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, 8, COLOUR_TYPE[C], 0, 0, 0))]
    pos = 0
    for ln in cut(len(z), chunks):
        out.append(_chunk(b"IDAT", z[pos: pos + ln]))
        pos += ln
    out.append(_chunk(b"IEND", b""))
    return b"".join(out)


def rgb(px: np.ndarray) -> np.ndarray:
    """What PIL's convert("RGB") gives for [H, W, C] pixels: grey replicated, alpha dropped."""
    return np.repeat(px[:, :, :1], 3, 2) if px.shape[2] < 3 else np.ascontiguousarray(px[:, :, :3])


# --------------------------------------------------------------------------------------
# pixel content
# --------------------------------------------------------------------------------------
def content(kind: str, H: int, W: int, C: int, seed: int) -> np.ndarray:
    """u8 [H, W, C].  random: any byte.  small: values 0..3, so Paeth's pa, pb and pc tie often.  high: 224..255, so
    a + b > 255 in Avg and the sums of Sub and Up wrap.  ramp: linear ramps mod 256 (Paeth predicts them exactly).
    patches: 3x5 constant patches.  mixed: all five, in diagonal bands."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    kinds = {
        "random": lambda: rng.integers(0, 256, (H, W, C)),
        "small": lambda: rng.integers(0, 4, (H, W, C)),
        "high": lambda: rng.integers(224, 256, (H, W, C)),
        "ramp": lambda: (xx[..., None] * rng.integers(1, 40, C) + yy[..., None] * rng.integers(1, 40, C)
                         + rng.integers(0, 256, C)) % 256,
        "patches": lambda: rng.integers(0, 256, ((H + 2) // 3, (W + 4) // 5, C)).repeat(3, 0).repeat(5, 1)[:H, :W],
    }
    if kind != "mixed":
        return kinds[kind]().astype(np.uint8)
    parts = [kinds[k]() for k in ("random", "small", "high", "ramp", "patches")]
    band = ((xx // 7 + yy // 3) % 5)[..., None]
    return np.choose(band, parts).astype(np.uint8)


# --------------------------------------------------------------------------------------
# the cases
# --------------------------------------------------------------------------------------
class Case:
    """One file of the GPU test: pixels, filters per row, layout, and the launch it is decoded in (one launch per
    `launch` name; the widest row of a launch sets its ring depth)."""

    def __init__(self, launch, name, px, filters, blocks=(STORED_MAX,), chunks=(1 << 20,), compressed=False):
        self.launch, self.name, self.px, self.filters = launch, name, px, list(filters)
        self.blocks, self.chunks, self.compressed = tuple(blocks), tuple(chunks), compressed

    @property
    def shape(self):
        return self.px.shape

    @functools.cached_property
    def data(self) -> bytes:
        return png(self.px, self.filters, self.blocks, self.chunks, self.compressed)

    @functools.cached_property
    def stream(self) -> bytes:
        return filter_rows(self.px, self.filters)

    def block_starts(self):
        """Raw positions in R where a stored block starts (none for the compressed variant)."""
        if self.compressed:
            return []
        return np.cumsum([0] + cut(len(self.stream), self.blocks)[:-1]).tolist()

    def __repr__(self):
        return f"{self.launch}/{self.name}{tuple(self.shape)}"


def de_bruijn_pairs(first: int) -> list:
    """26 filters, starting with `first`, in which every ordered pair of the five filters follows on consecutive rows."""
    seq = [0, 0, 1, 0, 2, 0, 3, 0, 4, 1, 1, 2, 1, 3, 1, 4, 2, 2, 3, 2, 4, 3, 3, 4, 4]      # B(5, 2), cyclic
    i = seq.index(first)
    rot = seq[i:] + seq[:i]
    return rot + rot[:1]


def ring_filters(D: int) -> list:
    """At least 3 D + 2 rows for ring depth D: Paeth only, then alternating Avg / Paeth, then a run of D + 1 rows that
    read no row above, then dependent rows with None rows between them."""
    rows = [PAETH] * (D + 1) + [AVG, PAETH] * ((D + 2) // 2) + [NONE] * D + [SUB]
    rows += [PAETH, NONE, AVG, NONE, NONE, UP, PAETH, SUB, AVG]
    assert len(rows) >= 3 * D + 2
    return rows


def stored_sizes_for_every_offset(L: int) -> int:
    """A block size whose multiples fall on every offset of an L-byte row."""
    return next(s for s in range(3, L + 3) if np.gcd(s, L) == 1)


@functools.lru_cache(maxsize=1)
def cases():
    out, seed = [], iter(range(1, 1 << 30))
    kinds = ("random", "small", "high", "ramp", "patches", "mixed")
    rng = np.random.default_rng(2024)

    # filter sequences (one launch at depth 16)
    for C in (1, 2, 3, 4):
        for f in range(5):
            for kind in ("mixed", "small", "high"):
                out.append(Case("filters", f"all{f}-{kind}", content(kind, 9, 45, C, next(seed)), [f] * 9))
        for first in range(5):
            out.append(Case("filters", f"pairs{first}", content(kinds[first], 26, 40, C, next(seed)),
                            de_bruijn_pairs(first)))
        for kind in kinds:
            out.append(Case("filters", f"random-{kind}", content(kind, 40, 70, C, next(seed)),
                            rng.integers(0, 5, 40)))
        long_runs = [AVG] * 20 + [PAETH] * 20 + [AVG, PAETH] * 10
        out.append(Case("filters", "avg-paeth-runs", content("mixed", 60, 50, C, next(seed)), long_runs))

    # chunk edges: partial last chunks, left and upper-left pixels across chunk boundaries (depth 16)
    for C in (1, 2, 3, 4):
        for W in (1, 2, 31, 32, 33, 63, 64, 65, 97):
            fl = [SUB, AVG, PAETH, SUB, PAETH, AVG, UP, PAETH, SUB, SUB, AVG, AVG, PAETH, PAETH]
            for kind in ("random", "high", "small"):
                out.append(Case("chunks", f"W{W}-{kind}", content(kind, len(fl), W, C, next(seed)), fl))

    # every ring depth: the widest row at that depth, wrapping the ring several times; and, in the same launch (so at
    # the same depth), frames of fewer rows than the ring and of one row more
    for k, (D, widest) in enumerate(depth_steps()):
        C = 4 if D == 3 else k % 4 + 1                                  # depth 3: 16,384 RGBA pixels
        W = widest // C
        fl = ring_filters(D)
        out.append(Case(f"depth{D}", "wide", content("mixed", len(fl), W, C, next(seed)), fl))
        for H in (D - 1, D + 1):
            fl = [PAETH if r % 3 else AVG for r in range(H)]
            out.append(Case(f"depth{D}", f"H{H}", content("mixed", H, 77 + k, (k + 1) % 4 + 1, next(seed)), fl))

    # segment layouts (depth 16)
    def layout(name, H, W, C, **kw):
        out.append(Case("segments", name, content("mixed", H, W, C, next(seed)), rng.integers(0, 5, H), **kw))

    layout("idat-1-0", 12, 37, 3, chunks=(1, 0, 1, 2, 7))
    layout("blocks-0-1-2-3", 12, 37, 4, blocks=(0, 1, 0, 2, 3), chunks=(1, 0, 1, 2, 7))
    layout("blocks-1", 9, 21, 2, blocks=(1,))
    layout("blocks-1-idat-1", 5, 13, 3, blocks=(1,), chunks=(1,))
    for W, C in ((5, 3), (33, 4), (7, 1), (40, 2)):
        L = 1 + W * C
        s = stored_sizes_for_every_offset(L)
        layout(f"every-offset-L{L}", s + 2, W, C, blocks=(s,), chunks=(11, 0, 3))
    layout("big-blocks", 60, 1200, 4, blocks=(3, STORED_MAX, 0, 2, 40000), chunks=(65536, 1, 0, 9000))
    layout("empty-first-idat", 6, 30, 3, blocks=(0, 5), chunks=(0, 4, 0))
    layout("compressed", 20, 90, 3, compressed=True)
    layout("compressed-idat-1-0", 11, 33, 4, compressed=True, chunks=(1, 0, 2))
    layout("compressed-L", 30, 61, 1, compressed=True, chunks=(100,))

    # launch shapes: narrow frames beside one of the widest (all at depth 3), and more frames than SMs
    out.append(Case("mixed-widths", "wide", content("mixed", 7, 16384, 4, next(seed)), [PAETH, AVG, SUB, UP, PAETH,
                                                                                        NONE, AVG]))
    for H, W, C in ((9, 1, 1), (33, 31, 2), (12, 33, 3), (20, 64, 4), (5, 100, 1), (3, 2000, 3), (40, 3, 4)):
        out.append(Case("mixed-widths", "narrow", content("mixed", H, W, C, next(seed)), rng.integers(0, 5, H),
                        blocks=(int(rng.integers(1, 300)),), chunks=(int(rng.integers(1, 500)),)))
    for i in range(300):
        H, W, C = int(rng.integers(1, 9)), int(rng.integers(1, 70)), int(rng.integers(1, 5))
        out.append(Case("many-frames", f"f{i}", content(kinds[i % 6], H, W, C, next(seed)), rng.integers(0, 5, H),
                        blocks=(int(rng.integers(1, 200)), 0), chunks=(int(rng.integers(1, 300)),)))
    return out


def launches():
    """{launch name: its cases, in order}."""
    by = defaultdict(list)
    for c in cases():
        by[c.launch].append(c)
    return dict(by)


# --------------------------------------------------------------------------------------
# host checks
# --------------------------------------------------------------------------------------
def _pil(data: bytes) -> np.ndarray:
    return np.asarray(Image.open(io.BytesIO(data)))


@pytest.mark.parametrize("launch", list(launches()))
def test_files_open_as_their_pixels(launch):
    for case in launches()[launch]:
        got = _pil(case.data)
        want = case.px[:, :, 0] if case.shape[2] == 1 else case.px
        assert np.array_equal(got, want), case
        assert np.array_equal(np.asarray(Image.open(io.BytesIO(case.data)).convert("RGB")), rgb(case.px)), case
        info = hm.parse_png(case.data)
        assert (info.H, info.W, info.C) == case.shape, case
        assert (info.inflated is not None) == case.compressed, case
        assert hm.filtered_stream(info, case.data) == case.stream, case
        assert np.array_equal(hm.unfilter_model(info, case.data), rgb(case.px)), case


def test_writer_layout():
    """The blocks and IDAT chunks are the sizes asked for, including empty ones."""
    px = content("random", 4, 6, 3, 1)
    data = png(px, [SUB, AVG, PAETH, UP], blocks=(0, 1, 0, 2, 3), chunks=(1, 0, 1, 2, 7))
    pos, idat = 8, []
    while pos < len(data):
        ln, kind = struct.unpack_from(">I4s", data, pos)
        if kind == b"IDAT":
            idat.append(ln)
        pos += 12 + ln
    z = zlib_stored(filter_rows(px, [SUB, AVG, PAETH, UP]), (0, 1, 0, 2, 3))
    assert idat == cut(len(z), (1, 0, 1, 2, 7)) and idat[:6] == [1, 0, 1, 2, 7, 1]
    assert z[:12] == b"\x78\x01" + b"\x00\x00\x00\xff\xff" + b"\x00\x01\x00\xfe\xff"     # LEN 0, LEN 1
    assert z[13:18] == b"\x00\x00\x00\xff\xff"
    assert zlib.decompress(z) == filter_rows(px, [SUB, AVG, PAETH, UP])


def test_case_coverage():
    """The GPU test reaches what the kernel handles differently."""
    all_cases = cases()
    L = launches()

    # every ordered filter pair on consecutive rows, every filter on row 0
    pairs = {(c.filters[r - 1], c.filters[r]) for c in all_cases for r in range(1, len(c.filters))}
    assert pairs == {(i, j) for i in range(5) for j in range(5)}
    assert {c.filters[0] for c in all_cases} == set(range(5))

    # every ring depth, with the ring wrapping at least three times; fewer rows than the ring, and one row more
    depth_of = {name: ring_depth(max(c.shape[1] * c.shape[2] for c in cs)) for name, cs in L.items()}
    for D in range(3, 17):
        hs = [c.shape[0] for name, cs in L.items() if depth_of[name] == D for c in cs]
        assert any(h >= 3 * D + 2 for h in hs) and any(h < D for h in hs) and D + 1 in hs, D
    assert any(c.shape == (c.shape[0], 16384, 4) for name, cs in L.items() if depth_of[name] == 3 for c in cs)
    assert depth_of["mixed-widths"] == 3 and len(L["many-frames"]) > 132

    # partial last chunks and full ones, for every C, with Sub, Avg and Paeth rows
    for C in (1, 2, 3, 4):
        for f in (SUB, AVG, PAETH):
            mods = {c.shape[1] % 32 for c in all_cases if c.shape[2] == C and c.shape[1] > 32 and f in c.filters}
            assert {0, 1, 31} <= mods, (C, f)

    # empty and 1-byte stored blocks and IDAT chunks; a block starting at every offset of a row
    stored = [c for c in all_cases if not c.compressed]
    assert any(0 in c.blocks for c in stored) and any(1 in c.blocks for c in stored)
    assert any(0 in c.chunks for c in all_cases) and any(1 in c.chunks for c in all_cases)
    assert any(c.blocks == (1,) for c in stored)
    assert any(c.compressed for c in all_cases)
    for C in (1, 2, 3, 4):
        assert any({s % (1 + c.shape[1] * c.shape[2]) for s in c.block_starts()[1:]}
                   == set(range(1 + c.shape[1] * c.shape[2])) for c in stored if c.shape[2] == C), C

    # the arithmetic edges: Paeth ties that change the prediction, Avg sums above 255, Sub and Up sums that wrap
    seen = defaultdict(int)
    for c in all_cases:
        x, a, b, cc = predictors(c.px)
        f = np.asarray(c.filters)[:, None]
        p = a + b - cc
        pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - cc)
        res = (x - np.choose(f, [0 * x, a, b, (a + b) >> 1, paeth(a, b, cc)])) & 0xFF
        seen["paeth pa == pc < pb"] += int(((f == PAETH) & (pa == pc) & (pa < pb) & (a != cc)).sum())
        seen["paeth pb == pc < pa"] += int(((f == PAETH) & (pb == pc) & (pb < pa) & (b != cc)).sum())
        seen["paeth pa == pb == pc"] += int(((f == PAETH) & (pa == pb) & (pb == pc)).sum())
        seen["avg a + b > 255"] += int(((f == AVG) & (a + b > 255)).sum())
        seen["sub wraps"] += int(((f == SUB) & (a + res > 255)).sum())
        seen["up wraps"] += int(((f == UP) & (b + res > 255)).sum())
    assert all(v >= 100 for v in seen.values()), dict(seen)
