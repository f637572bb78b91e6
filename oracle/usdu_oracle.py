"""CPU oracle for the Ultimate-SD-Upscale tile hot path -- TEST INFRASTRUCTURE ONLY.

This file is a numpy restatement of the arithmetic that the reference
(robertvoy/ComfyUI-Distributed @ a91f9fb) performs on the CPU through Pillow.  It is
imported only by ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` legs, and only as the checker.  The product
package (``comfyui-distributed_b200/``) never imports it.

Where the algorithm lives
-------------------------
* tile grid / crop geometry ..... ``upscale/tile_ops.py:14-32`` (round_to_multiple,
  calculate_tiles), ``:51-78`` / ``:108-135`` (uniform / non-uniform target size),
  ``utils/usdu_utils.py:49-62`` (get_crop_region), ``:65-73`` (fix_crop_region),
  ``:76-112`` (expand_crop).
* float <-> u8 .................. ``utils/image.py:8-18`` (truncating cast, /255).
* LANCZOS resize ................ Pillow ``Image.resize(..., Image.LANCZOS)`` called at
  ``upscale/tile_ops.py:88,148,329``, ``upscale/modes/single_gpu.py:63``,
  ``upscale/modes/static.py:182,271``.
* feather mask .................. Pillow ``ImageDraw.rectangle`` + ``ImageFilter.GaussianBlur``
  at ``upscale/tile_ops.py:289-308``.
* seam blend .................... Pillow paste / putalpha / alpha_composite at
  ``upscale/tile_ops.py:310-349``.
* progressive single-GPU driver . ``upscale/modes/single_gpu.py:8-72``.
* static (multi-worker) driver .. ``upscale/modes/static.py:191-314`` (worker),
  ``:371-570`` (master, sorted final blend ``:521-553``).
* collector ordering ............ ``nodes/collector.py:193-236``.

Third-party dependency
----------------------
The pixel arithmetic is Pillow's (not vendored in /root/reference; the reference does
not pin a version -- ``pyproject.toml`` has ``dependencies = []``).  The restatement
below follows Pillow 12.2.0 (the version in this image): ``src/libImaging/Resample.c``
(precompute_coeffs, normalize_coeffs_8bpc, ImagingResampleHorizontal_8bpc /
Vertical_8bpc), ``src/libImaging/BoxBlur.c`` (ImagingGaussianBlur -> 3 extended box
passes per axis) and ``src/libImaging/AlphaComposite.c`` / ``Paste.c``.

Pinning
-------
``tests/test_oracle_vs_pillow.py`` checks every primitive here bit-exactly against the
installed Pillow on random data; ``tests/test_oracle_golden.py`` checks the drivers
against fixtures in ``tests/golden/`` that were produced by importing and running the
REAL reference modules from /root/reference (``oracle/gen_golden.py``).  The reference
itself ships no known-answer test for this path (SURVEY.md section 4).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Callable, Dict, List, Sequence, Tuple

import numpy as np

PRECISION_BITS = 32 - 8 - 2  # Pillow Resample.c


# --------------------------------------------------------------------------------------
# geometry
# --------------------------------------------------------------------------------------
def round_to_multiple(value: int, multiple: int = 8) -> int:
    """upscale/tile_ops.py:14-16 -- Python round() => banker's rounding on .5 cases."""
    return round(value / multiple) * multiple


def calculate_tiles(W: int, H: int, tw: int, th: int) -> List[Tuple[int, int]]:
    """upscale/tile_ops.py:18-32 -- row-major (x, y) grid origins."""
    rows = math.ceil(H / th)
    cols = math.ceil(W / tw)
    return [(xi * tw, yi * th) for yi in range(rows) for xi in range(cols)]


def _rect_bbox(W: int, H: int, x: int, y: int, tw: int, th: int):
    """bbox of PIL's *inclusive* rectangle [x, y, x+tw, y+th] clipped to the canvas
    (ImageDraw.rectangle + Image.getbbox, upscale/tile_ops.py:51-54, usdu_utils.py:52)."""
    bx1, by1 = max(x, 0), max(y, 0)
    bx2, by2 = min(x + tw + 1, W), min(y + th + 1, H)
    if bx2 <= bx1 or by2 <= by1:  # nothing drawn -> getbbox() is None (usdu_utils.py:55-56)
        return W, H, 0, 0
    return bx1, by1, bx2, by2


def _expand_crop(region, W, H, target_w, target_h):
    """utils/usdu_utils.py:76-112."""
    x1, y1, x2, y2 = region
    diff = target_w - (x2 - x1)
    x2 = min(x2 + diff // 2, W)
    diff = target_w - (x2 - x1)
    x1 = max(x1 - diff, 0)
    diff = target_w - (x2 - x1)
    x2 = min(x2 + diff, W)
    diff = target_h - (y2 - y1)
    y2 = min(y2 + diff // 2, H)
    diff = target_h - (y2 - y1)
    y1 = max(y1 - diff, 0)
    diff = target_h - (y2 - y1)
    y2 = min(y2 + diff, H)
    return (x1, y1, x2, y2)


def crop_geometry(W: int, H: int, x: int, y: int, tw: int, th: int, padding: int,
                  uniform: bool) -> Tuple[int, int, int, int, int, int]:
    """Crop window (x1, y1, x2, y2) and processing size (pw, ph) of the tile at (x, y).

    upscale/tile_ops.py:51-82 (== :108-138 for the batched twin)."""
    bx1, by1, bx2, by2 = _rect_bbox(W, H, x, y, tw, th)
    x1, y1 = max(bx1 - padding, 0), max(by1 - padding, 0)
    x2, y2 = min(bx2 + padding, W), min(by2 + padding, H)
    if x2 < W:  # fix_crop_region, usdu_utils.py:65-73
        x2 -= 1
    if y2 < H:
        y2 -= 1
    if uniform:
        pw = round_to_multiple(tw + padding, 8)
        ph = round_to_multiple(th + padding, 8)
        cw, ch = x2 - x1, y2 - y1
        crop_ratio = cw / ch if ch != 0 else 1.0
        proc_ratio = pw / ph if ph != 0 else 1.0
        if crop_ratio > proc_ratio:
            tgt_w = cw
            tgt_h = round(cw / proc_ratio) if proc_ratio != 0 else ch
        else:
            tgt_w = round(ch * proc_ratio)
            tgt_h = ch
        x1, y1, x2, y2 = _expand_crop((x1, y1, x2, y2), W, H, tgt_w, tgt_h)
    else:
        cw, ch = x2 - x1, y2 - y1
        pw = max(8, math.ceil(cw / 8) * 8)
        ph = max(8, math.ceil(ch / 8) * 8)
        x1, y1, x2, y2 = _expand_crop((x1, y1, x2, y2), W, H, pw, ph)
    return x1, y1, x2, y2, pw, ph


# --------------------------------------------------------------------------------------
# float <-> u8   (utils/image.py:8-18)
# --------------------------------------------------------------------------------------
def quantize_u8(x: np.ndarray) -> np.ndarray:
    """(255 * x).astype(uint8) as the reference runs it: the multiply rounds in x's own dtype (fp16, fp32 or fp64;
    anything else is taken as fp32), then numpy's x86 cast truncates and keeps the low byte.  NaN, +-inf and products
    outside [-2^31, 2^31) give 0 (tests/test_u8_cast_model.py pins this on the host)."""
    x = np.asarray(x)
    if x.dtype not in (np.float16, np.float64):
        x = x.astype(np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        return (x.dtype.type(255) * x).astype(np.uint8)


def dequantize_u8(u: np.ndarray) -> np.ndarray:
    return u.astype(np.float32) / np.float32(255.0)


# --------------------------------------------------------------------------------------
# Pillow LANCZOS, 8 bits per channel   (Resample.c)
# --------------------------------------------------------------------------------------
def _sinc(x: float) -> float:
    if x == 0.0:
        return 1.0
    x = x * math.pi
    return math.sin(x) / x


def _lanczos3(x: float) -> float:
    if -3.0 <= x < 3.0:
        return _sinc(x) * _sinc(x / 3)
    return 0.0


def _bicubic(x: float) -> float:
    """Resample.c bicubic_filter, a = -0.5 (Keys), support 2."""
    a = -0.5
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


_FILTERS = {"lanczos": (_lanczos3, 3.0), "bicubic": (_bicubic, 2.0)}
_COEFF_CACHE: Dict[Tuple[int, int, str], Tuple[np.ndarray, np.ndarray]] = {}


def lanczos_coeffs(in_size: int, out_size: int) -> Tuple[np.ndarray, np.ndarray]:
    return resample_coeffs(in_size, out_size, "lanczos")


def resample_coeffs(in_size: int, out_size: int, filt: str = "lanczos") -> Tuple[np.ndarray, np.ndarray]:
    """precompute_coeffs + normalize_coeffs_8bpc for a full-axis resize (box = whole axis).

    Returns bounds int32[out,2] = (xmin, n) and kk int32[out, ksize] (22-bit fixed point)."""
    key = (in_size, out_size, filt)
    if key in _COEFF_CACHE:
        return _COEFF_CACHE[key]
    _lanczos3, fsupport = _FILTERS[filt]
    scale = filterscale = in_size / out_size
    if filterscale < 1.0:
        filterscale = 1.0
    support = fsupport * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), dtype=np.int32)
    kk = np.zeros((out_size, ksize), dtype=np.int32)
    ss = 1.0 / filterscale
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = int(center - support + 0.5)
        if xmin < 0:
            xmin = 0
        xmax = int(center + support + 0.5)
        if xmax > in_size:
            xmax = in_size
        n = xmax - xmin
        w = [_lanczos3((i + xmin - center + 0.5) * ss) for i in range(n)]
        ww = 0.0
        for v in w:
            ww += v
        for i in range(n):
            v = w[i] / ww if ww != 0.0 else w[i]
            if v < 0:
                kk[xx, i] = int(-0.5 + v * (1 << PRECISION_BITS))
            else:
                kk[xx, i] = int(0.5 + v * (1 << PRECISION_BITS))
        bounds[xx, 0] = xmin
        bounds[xx, 1] = n
    _COEFF_CACHE[key] = (bounds, kk)
    return bounds, kk


def _resample_axis0(img: np.ndarray, out_size: int, filt: str = "lanczos") -> np.ndarray:
    """One 8bpc resample pass along axis 0 of img[u8, n_in, ...]."""
    n_in = img.shape[0]
    bounds, kk = resample_coeffs(n_in, out_size, filt)
    ksize = kk.shape[1]
    idx = bounds[:, 0:1] + np.arange(ksize, dtype=np.int32)[None, :]
    idx = np.minimum(idx, n_in - 1)  # taps past n have coefficient 0
    acc = np.full((out_size,) + img.shape[1:], 1 << (PRECISION_BITS - 1), dtype=np.int64)
    src = img.astype(np.int64)
    for t in range(ksize):
        k = kk[:, t].astype(np.int64).reshape((out_size,) + (1,) * (img.ndim - 1))
        acc += src[idx[:, t]] * k
    acc >>= PRECISION_BITS
    return np.clip(acc, 0, 255).astype(np.uint8)


def lanczos_resize_u8(img: np.ndarray, out_w: int, out_h: int) -> np.ndarray:
    return resize_u8(img, out_w, out_h, "lanczos")


def resize_u8(img: np.ndarray, out_w: int, out_h: int, filt: str = "lanczos") -> np.ndarray:
    """Image.resize((out_w, out_h), LANCZOS | BICUBIC) on an u8 image [H, W, C] (or [H, W]).

    Horizontal pass first with a u8 intermediate, then vertical; a pass is skipped when
    that axis keeps its size (Resample.c ImagingResampleInner)."""
    h, w = img.shape[:2]
    out = img
    if out_w != w:
        out = np.swapaxes(_resample_axis0(np.swapaxes(out, 0, 1), out_w, filt), 0, 1)
    if out_h != h:
        out = _resample_axis0(out, out_h, filt)
    return np.ascontiguousarray(out)


# --------------------------------------------------------------------------------------
# conditioning mask crop   (utils/usdu_utils.py:415-442, :242-266, :169-203)
# --------------------------------------------------------------------------------------
def nearest_index(in_size: int, out_size: int) -> np.ndarray:
    """Source index of every output sample of Image.resize(..., NEAREST) along one axis
    (Geometry.c ImagingScaleAffine: xo = a/2, then xo += a per sample, index = (int)xo --
    the additions accumulate in double exactly like the C loop)."""
    a = in_size / out_size
    xo = 0.0 + a * 0.5
    out = np.zeros(out_size, dtype=np.int32)
    for x in range(out_size):
        xin = -1 if xo < 0.0 else int(xo)
        out[x] = min(max(xin, 0), in_size - 1)
        xo += a
    return out


def pad_fill_u8(img: np.ndarray, hp: int, vp: int) -> np.ndarray:
    """pad_image2(img, hp, hp, vp, vp, fill=True) on a mode-L image [h, w] (usdu_utils.py:169-203):
    left/right columns = the edge column WITHOUT its first and last pixel, NEAREST-stretched to the
    new height; then top/bottom rows likewise (they overwrite the corners)."""
    h, w = img.shape
    nh, nw = h + 2 * vp, w + 2 * hp
    out = np.zeros((nh, nw), dtype=np.uint8)
    out[vp:vp + h, hp:hp + w] = img
    if hp > 0:
        iy = 1 + nearest_index(h - 2, nh)
        out[:, :hp] = img[iy, 0][:, None]
        out[:, nw - hp:] = img[iy, w - 1][:, None]
    if vp > 0:
        ix = 1 + nearest_index(w - 2, nw)
        out[:vp, :] = img[0, ix][None, :]
        out[nh - vp:, :] = img[h - 1, ix][None, :]
    return out


def py_round(x: float) -> int:
    return int(round(x))       # Python 3 round(): half to even, like the reference's call


def mask_fit_geometry(cw: int, ch: int, pw: int, ph: int):
    """resize_and_pad_image's sizes (usdu_utils.py:242-266): -> (rw, rh, hp, vp)."""
    width_ratio, height_ratio = pw / cw, ph / ch
    ratio = width_ratio if height_ratio > width_ratio else height_ratio
    rw, rh = py_round(cw * ratio), py_round(ch * ratio)
    return rw, rh, (pw - rw) // 2, (ph - rh) // 2


def crop_mask_u8(mask: np.ndarray, region, canvas_size, tile_size) -> np.ndarray:
    """crop_mask for ONE mask frame already cast to u8 [Hm, Wm] (usdu_utils.py:415-442):
    BICUBIC to the canvas size, crop the region, LANCZOS to the tile's aspect-preserving size,
    edge-fill pad, LANCZOS to the tile size, BICUBIC if that still is not the tile size."""
    W, H = canvas_size
    pw, ph = tile_size
    x1, y1, x2, y2 = region
    m = resize_u8(mask, W, H, "bicubic")[y1:y2, x1:x2]
    ch, cw = m.shape
    rw, rh, hp, vp = mask_fit_geometry(cw, ch, pw, ph)
    m = resize_u8(m, rw, rh, "lanczos")
    m = pad_fill_u8(m, hp, vp)
    m = resize_u8(m, pw, ph, "lanczos")
    if m.shape != (ph, pw):
        m = resize_u8(m, pw, ph, "bicubic")
    return m


# --------------------------------------------------------------------------------------
# Pillow GaussianBlur on mode L   (BoxBlur.c)
# --------------------------------------------------------------------------------------
def box_blur_params(radius: float) -> Tuple[int, int, int]:
    """_gaussian_blur_radius (3 passes) + ImagingHorizontalBoxBlur's integer weights.

    All intermediate arithmetic is C ``float`` (fp32), as in BoxBlur.c."""
    f = np.float32
    r = f(radius)
    sigma2 = f(r * r / f(3))
    L = f(math.sqrt(12.0 * float(sigma2) + 1.0))
    l = f(math.floor((float(L) - 1.0) / 2.0))
    a = f(f(f(2) * l + f(1)) * f(f(l * f(l + f(1))) - f(f(3) * sigma2)))
    a = f(a / f(f(6) * f(sigma2 - f(f(l + f(1)) * f(l + f(1))))))
    R = f(l + a)
    rad = int(R)
    ww = int(f(f(1 << 24) / f(R * f(2) + f(1))))
    fw = ((1 << 24) - (rad * 2 + 1) * ww) // 2
    return rad, ww, fw


def box_blur_pass_1d(line: np.ndarray, rad: int, ww: int, fw: int) -> np.ndarray:
    """One extended-box pass along the last axis, edge-replicated, u8 in / u8 out."""
    n = line.shape[-1]
    src = line.astype(np.int64)
    pos = np.arange(n)
    acc = np.zeros(line.shape, dtype=np.int64)
    for i in range(-rad, rad + 1):
        acc += src[..., np.clip(pos + i, 0, n - 1)]
    far = src[..., np.clip(pos - rad - 1, 0, n - 1)] + src[..., np.clip(pos + rad + 1, 0, n - 1)]
    out = (acc * ww + far * fw + (1 << 23)) >> 24
    return out.astype(np.uint8)


def gaussian_blur_L(img: np.ndarray, radius: float) -> np.ndarray:
    """ImageFilter.GaussianBlur(radius) on an L image [H, W]: 3 horizontal passes, then
    3 vertical passes, u8 rounding after every pass."""
    rad, ww, fw = box_blur_params(radius)
    out = img
    for _ in range(3):
        out = box_blur_pass_1d(out, rad, ww, fw)
    out = out.T
    for _ in range(3):
        out = box_blur_pass_1d(out, rad, ww, fw)
    return np.ascontiguousarray(out.T)


def tile_mask_full(W: int, H: int, x: int, y: int, tw: int, th: int, blur: int) -> np.ndarray:
    """create_tile_mask, upscale/tile_ops.py:289-308 -- the literal full-canvas form."""
    m = np.zeros((H, W), dtype=np.uint8)
    bx1, by1, bx2, by2 = _rect_bbox(W, H, x, y, tw, th)
    if bx2 > bx1 and by2 > by1:
        m[by1:by2, bx1:bx2] = 255
    if blur > 0:
        m = gaussian_blur_L(m, blur)
    return m


def _blur_profile_1d(n: int, lo: int, hi: int, amp: np.ndarray, params) -> np.ndarray:
    """3 passes over a length-n line that is ``amp`` on [lo, hi) and 0 elsewhere.
    amp may be an array of amplitudes -> result [len(amp), n]."""
    rad, ww, fw = params
    amp = np.atleast_1d(np.asarray(amp, dtype=np.uint8))
    line = np.zeros((amp.shape[0], n), dtype=np.uint8)
    line[:, lo:hi] = amp[:, None]
    for _ in range(3):
        line = box_blur_pass_1d(line, rad, ww, fw)
    return line


def tile_mask_window(W: int, H: int, x: int, y: int, tw: int, th: int, blur: int,
                     window: Tuple[int, int, int, int]) -> np.ndarray:
    """The feather mask restricted to ``window`` = (x1, y1, x2, y2), computed without a
    full canvas.  The rectangle is an outer product of two indicator lines, the three
    horizontal passes act row-wise (rows outside the rectangle stay 0, rows inside all
    become the same u8 profile hx), so every column x entering the vertical passes is a
    step of amplitude hx[x]; the result is v_{hx[x]}(y).  Bit-identical to
    ``tile_mask_full(...)[y1:y2, x1:x2]`` (tests/test_oracle_vs_pillow.py)."""
    x1, y1, x2, y2 = window
    bx1, by1, bx2, by2 = _rect_bbox(W, H, x, y, tw, th)
    if bx2 <= bx1 or by2 <= by1:
        return np.zeros((y2 - y1, x2 - x1), dtype=np.uint8)
    if blur <= 0:
        m = np.zeros((y2 - y1, x2 - x1), dtype=np.uint8)
        m[max(by1, y1) - y1:max(min(by2, y2) - y1, 0), max(bx1, x1) - x1:max(min(bx2, x2) - x1, 0)] = 255
        return m
    params = box_blur_params(blur)
    hx = _blur_profile_1d(W, bx1, bx2, np.array([255]), params)[0]          # [W]
    vt = _blur_profile_1d(H, by1, by2, np.arange(256), params)              # [256, H]
    return np.ascontiguousarray(vt[hx[x1:x2]][:, y1:y2].T)


# --------------------------------------------------------------------------------------
# seam blend   (blend_tile, upscale/tile_ops.py:310-349)
# --------------------------------------------------------------------------------------
def composite_u8(S: np.ndarray, D: np.ndarray, A: np.ndarray) -> np.ndarray:
    """alpha_composite of an RGBA layer (rgb=S, alpha=A) over an opaque base D, u8.

    AlphaComposite.c with dst alpha 255: blend = A*255, outa255 = 255*255,
    coef1 = A*255*255*128 / (255*255) = A*128, coef2 = 255*128 - coef1;
    tmp = S*coef1 + D*coef2 + (0x80 << 7); out = SHIFTFORDIV255(tmp) >> 7."""
    a = A.astype(np.uint32)
    if a.ndim == S.ndim - 1:
        a = a[..., None]
    c1 = a * 128
    c2 = (255 - a) * 128
    tmp = S.astype(np.uint32) * c1 + D.astype(np.uint32) * c2 + (0x80 << 7)
    tmp = ((tmp >> 8) + tmp) >> 8
    return (tmp >> 7).astype(np.uint8)


# --------------------------------------------------------------------------------------
# drivers
# --------------------------------------------------------------------------------------
@dataclass
class TilePlan:
    """Everything integer about one tile position (identical for every frame)."""
    idx: int
    x: int
    y: int
    x1: int
    y1: int
    x2: int
    y2: int
    pw: int
    ph: int

    @property
    def ew(self) -> int:
        return self.x2 - self.x1

    @property
    def eh(self) -> int:
        return self.y2 - self.y1


def make_plan(W, H, tile_width, tile_height, padding, uniform) -> Tuple[int, int, List[TilePlan]]:
    tw = round_to_multiple(tile_width)      # single_gpu.py:13-14, static.py:198-199
    th = round_to_multiple(tile_height)
    plan = []
    for i, (x, y) in enumerate(calculate_tiles(W, H, tw, th)):
        x1, y1, x2, y2, pw, ph = crop_geometry(W, H, x, y, tw, th, padding, uniform)
        plan.append(TilePlan(i, x, y, x1, y1, x2, y2, pw, ph))
    return tw, th, plan


DenoiseFn = Callable[[np.ndarray, TilePlan], np.ndarray]
"""denoise(tile_batch fp32 [B, ph, pw, 3] in [0,1], plan row) -> fp32 [B, ph, pw, 3]."""


def extract_tile(canvas: np.ndarray, t: TilePlan) -> np.ndarray:
    """extract_batch_tile_with_padding on an u8 canvas [B,H,W,3] -> fp32 [B,ph,pw,3]."""
    out = []
    for b in range(canvas.shape[0]):
        crop = canvas[b, t.y1:t.y2, t.x1:t.x2]
        if (t.ew, t.eh) != (t.pw, t.ph):
            crop = lanczos_resize_u8(crop, t.pw, t.ph)
        out.append(dequantize_u8(crop))
    return np.stack(out, 0)


def blend_processed(canvas: np.ndarray, processed: np.ndarray, t: TilePlan, mask_win: np.ndarray):
    """tensor_to_pil (trunc) -> resize back -> blend_tile, in place on canvas[B,H,W,3]."""
    for b in range(canvas.shape[0]):
        q = quantize_u8(processed[b])
        if (t.pw, t.ph) != (t.ew, t.eh):
            q = lanczos_resize_u8(q, t.ew, t.eh)
        win = canvas[b, t.y1:t.y2, t.x1:t.x2]
        canvas[b, t.y1:t.y2, t.x1:t.x2] = composite_u8(q, win, mask_win)


def process_single(image: np.ndarray, denoise: DenoiseFn, tile_width: int, tile_height: int,
                   padding: int, mask_blur: int, uniform: bool = True) -> np.ndarray:
    """process_single_gpu (upscale/modes/single_gpu.py:8-72) as a window-only algorithm:
    tile k is cropped from the canvas AFTER tiles < k were blended (progressive)."""
    B, H, W, _ = image.shape
    tw, th, plan = make_plan(W, H, tile_width, tile_height, padding, uniform)
    canvas = quantize_u8(image)                                    # single_gpu.py:30-32
    for t in plan:
        tile_in = extract_tile(canvas, t)                          # :42-49
        out = denoise(tile_in, t)                                  # :52-55
        mask = tile_mask_window(W, H, t.x, t.y, tw, th, mask_blur, (t.x1, t.y1, t.x2, t.y2))
        blend_processed(canvas, out, t, mask)                      # :58-64
    return dequantize_u8(canvas)                                   # :67-68


def replay_static(image: np.ndarray, denoise: DenoiseFn, tile_width: int, tile_height: int,
                  padding: int, mask_blur: int, uniform: bool,
                  assignment: Sequence[Sequence[int]]) -> np.ndarray:
    """Deterministic replay of static (tile-queue) mode for a fixed pull order.

    ``assignment[r]`` is the ordered list of tile ids participant r processed; r == 0 is
    the master.  Every participant starts from u8(image) and crops from ITS OWN
    progressive canvas (static.py:209-212 + :242-280 worker, :382-385 + :151-183 master).
    The result is the master's canvas with all worker tiles blended on top in ascending
    (tile_idx, batch_idx) order (static.py:521-553)."""
    B, H, W, _ = image.shape
    tw, th, plan = make_plan(W, H, tile_width, tile_height, padding, uniform)
    masks = {}

    def mask_of(t):
        if t.idx not in masks:
            masks[t.idx] = tile_mask_window(W, H, t.x, t.y, tw, th, mask_blur, (t.x1, t.y1, t.x2, t.y2))
        return masks[t.idx]

    base = quantize_u8(image)
    master = None
    shipped = {}
    for r, tiles in enumerate(assignment):
        canvas = base.copy()
        for tid in tiles:
            t = plan[tid]
            out = denoise(extract_tile(canvas, t), t)
            blend_processed(canvas, out, t, mask_of(t))
            if r != 0:
                # the worker ships the raw processed tensor, PNG-encoded after the same
                # truncating cast (worker_comms.py:30-33) -> keep the fp32, quantise at blend
                shipped[tid] = out
        if r == 0:
            master = canvas
    if master is None:
        master = base.copy()
    for tid in sorted(shipped):
        blend_processed(master, shipped[tid], plan[tid], mask_of(plan[tid]))
    return dequantize_u8(master)


def collector_combine(master_images, worker_images: Dict[str, np.ndarray], worker_order: Sequence[str],
                      delegate_only: bool = False) -> np.ndarray:
    """DistributedCollector ordering (nodes/collector.py:193-236): master's images first
    (full-precision fp32, :276), then each enabled worker in ``worker_order``, then
    unexpected worker ids sorted.  Worker images went through trunc-u8 -> PNG -> /255
    (collector.py:95-98, api/job_routes.py:104-132), i.e. they are quantised."""
    parts = []
    if not delegate_only and master_images is not None:
        parts.append(np.asarray(master_images, dtype=np.float32))
    seen = set()
    for wid in [str(w) for w in worker_order]:
        seen.add(wid)
        if wid in worker_images:
            parts.append(dequantize_u8(quantize_u8(worker_images[wid])))
    for wid in sorted(worker_images):
        if wid not in seen:
            parts.append(dequantize_u8(quantize_u8(worker_images[wid])))
    if not parts:
        raise ValueError("No image data collected from master or workers")
    return np.concatenate(parts, 0)


# --------------------------------------------------------------------------------------
# the T0 test denoiser (BASELINE.md section 3): same callable on both sides of a parity test
# --------------------------------------------------------------------------------------
def t0_noise(seed: int, shape: Tuple[int, ...]) -> np.ndarray:
    """Seeded uniform noise; torch's CPU generator so that it is identical everywhere."""
    import torch
    g = torch.Generator().manual_seed(int(seed))
    return torch.rand(shape, generator=g, dtype=torch.float32).numpy()


def make_t0_denoiser(seed: int, denoise: float) -> DenoiseFn:
    """x' = clamp(x*(1-d) + noise*d, 0, 1); every step individually rounded in fp32 so
    that CPU and GPU agree bit-for-bit.  The same seed is used for every tile
    (upscale/tile_ops.py:430-431, single_gpu.py:53-55)."""
    d = np.float32(denoise)
    omd = np.float32(1.0) - d
    cache = {}

    def fn(tile: np.ndarray, t: TilePlan) -> np.ndarray:
        if tile.shape not in cache:
            cache[tile.shape] = t0_noise(seed, tile.shape)
        y = tile.astype(np.float32) * omd + cache[tile.shape] * d
        return np.clip(y, np.float32(0), np.float32(1))

    return fn
