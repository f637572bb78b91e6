"""Per-tile conditioning for the real ComfyUI sampler (SURVEY.md 8f rank 3).

Text embeddings are shared between tiles; entries that carry SPATIAL hints must be cut to the
tile's crop window before sampling, as the reference does for every tile
(upscale/conditioning.py:17-34 clone, utils/usdu_utils.py:297-312 ControlNet hints, :335-378
GLIGEN boxes, :381-412 areas, :445-503 reference latents, :506-517 crop_cond).  Everything
here is torch / integer arithmetic on whatever device the hints live on -- no PIL.  Mask
conditioning (:415-442: PIL BICUBIC upscale of the whole mask to the canvas size, crop, LANCZOS fit
with edge-fill padding -- per tile and per frame) runs on the GPU through the one-channel plane
kernels of libusdu_b200.so (csrc/usdu_plane.cu), window only, bit-identical to Pillow's 8bpc
arithmetic (`MaskCropper`).
"""
from __future__ import annotations

import copy
import math
from typing import Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

from .casts import reference_f32

Region = Tuple[int, int, int, int]


def scale_region(region: Region, from_size: Sequence[int], to_size: Sequence[int]) -> Region:
    """Map a rectangle from an image of `from_size` (w, h) to the same image at `to_size`:
    floor the near edges, ceil the far ones (utils/usdu_utils.py:115-124)."""
    x1, y1, x2, y2 = region
    fw, fh = from_size
    tw, th = to_size
    return (math.floor(x1 * tw / fw), math.floor(y1 * th / fh), math.ceil(x2 * tw / fw), math.ceil(y2 * th / fh))


def intersect(a: Region, b: Region) -> Optional[Region]:
    x1, y1, x2, y2 = max(a[0], b[0]), max(a[1], b[1]), min(a[2], b[2]), min(a[3], b[3])
    return None if (x1 >= x2 or y1 >= y2) else (x1, y1, x2, y2)


def _clone_control_chain(control, clone_hint: bool):
    if control is None:
        return None
    new = copy.copy(control)
    if clone_hint and getattr(control, "cond_hint_original", None) is not None:
        new.cond_hint_original = control.cond_hint_original.clone()
    if hasattr(control, "previous_controlnet"):
        new.previous_controlnet = _clone_control_chain(control.previous_controlnet, clone_hint)
    return new


def clone_conditioning(cond, clone_hints: bool = True, clone_masks: bool = True):
    """New list / dicts / hint tensors per tile, models shared (upscale/conditioning.py:17-34).
    clone_masks=False keeps the caller's mask tensors (the mask cropper never writes to them and
    keys its u8 cache on their identity)."""
    out = []
    for emb, opts in cond:
        d = dict(opts)
        if "control" in d:
            d["control"] = _clone_control_chain(d["control"], clone_hints)
        for key in ("mask", "pooled_output"):
            if d.get(key) is not None and (clone_masks or key != "mask"):
                d[key] = d[key].clone()
        if "area" in d:
            d["area"] = d["area"][:]
        out.append([emb.clone() if emb is not None else None, d])
    return out


def crop_control_hints(opts: dict, region: Region, canvas_size, tile_size):
    """Every ControlNet of the chain gets its hint [B,C,h,w] cut to the window (scaled to the
    hint's own resolution) and resized nearest-exact to the tile size."""
    c = opts.get("control")
    if c is None:
        return
    def _copy(ctrl):
        # ControlNet.copy() is what the reference calls (utils/usdu_utils.py:297-312): it creates a fresh control object
        # WITHOUT the cached cond_hint / timestep state a shallow copy would carry over; copy.copy is for test doubles
        return ctrl.copy() if callable(getattr(ctrl, "copy", None)) else copy.copy(ctrl)

    head = _copy(c)
    opts["control"] = head
    node = head
    while node is not None:
        hint = node.cond_hint_original
        hx1, hy1, hx2, hy2 = scale_region(region, canvas_size, (hint.shape[-1], hint.shape[-2]))
        hint = hint[:, :, hy1:hy2, hx1:hx2]
        node.cond_hint_original = F.interpolate(hint, size=(tile_size[1], tile_size[0]), mode="nearest-exact")
        prev = getattr(node, "previous_controlnet", None)
        prev = _copy(prev) if prev is not None else None
        if hasattr(node, "set_previous_controlnet"):
            node.set_previous_controlnet(prev)
        else:
            node.previous_controlnet = prev
        node = prev


def _to_tile_box(box: Region, region: Region, w_pad: int, h_pad: int) -> Region:
    return (box[0] - region[0] + w_pad, box[1] - region[1] + h_pad, box[2] - region[0] + w_pad, box[3] - region[1] + h_pad)


def crop_gligen(opts: dict, region: Region, init_size, canvas_size, w_pad: int = 0, h_pad: int = 0):
    if "gligen" not in opts:
        return
    kind, model, boxes = opts["gligen"]
    if kind != "position":
        return
    kept = []
    for emb, h, w, y, x in boxes:
        box = scale_region((x * 8, y * 8, (x + w) * 8, (y + h) * 8), init_size, canvas_size)
        hit = intersect(box, region)
        if hit is None:
            continue
        x1, y1, x2, y2 = _to_tile_box(hit, region, w_pad, h_pad)
        kept.append((emb, (y2 - y1) // 8, (x2 - x1) // 8, y1 // 8, x1 // 8))
    opts["gligen"] = (kind, model, kept)


def crop_area(opts: dict, region: Region, init_size, canvas_size, w_pad: int = 0, h_pad: int = 0):
    if "area" not in opts:
        return
    h, w, y, x = opts["area"]
    box = scale_region((8 * x, 8 * y, 8 * (x + w), 8 * (y + h)), init_size, canvas_size)
    hit = intersect(box, region)
    if hit is None:
        del opts["area"]
        opts.pop("strength", None)
        return
    x1, y1, x2, y2 = _to_tile_box(hit, region, w_pad, h_pad)
    opts["area"] = ((y2 - y1) // 8, (x2 - x1) // 8, y1 // 8, x1 // 8)


def crop_reference_latents(opts: dict, region: Region, canvas_size, tile_size, k: int = 8):
    lat = opts.get("reference_latents")
    if not isinstance(lat, list):
        return
    cw, chh = canvas_size[0] // k, canvas_size[1] // k
    tw, th = max(1, tile_size[0] // k), max(1, tile_size[1] // k)
    x1, y1, x2, y2 = region
    out = []
    for t in lat:
        five = t.ndim == 5
        if five:
            t = t.squeeze(2)
        if t.ndim != 4:
            raise ValueError(f"expected BCHW or BC1HW, got {tuple(t.shape)}")
        if tuple(t.shape[-2:]) != (chh, cw):
            t = F.interpolate(t, size=(chh, cw), mode="bilinear", align_corners=False)
        t = t[:, :, int(round(y1 / k)):int(round(y2 / k)), int(round(x1 / k)):int(round(x2 / k))]
        t = F.interpolate(t, size=(th, tw), mode="bilinear", align_corners=False)
        out.append(t.unsqueeze(2) if five else t)
    opts["reference_latents"] = out


def mask_fit_geometry(cw: int, ch: int, pw: int, ph: int):
    """Sizes of resize_and_pad_image (utils/usdu_utils.py:242-266) for a (cw, ch) crop that has to
    become a (pw, ph) tile: -> (rw, rh, hp, vp).  `round` is Python's (half to even), like there."""
    width_ratio, height_ratio = pw / cw, ph / ch
    ratio = width_ratio if height_ratio > width_ratio else height_ratio
    rw, rh = round(cw * ratio), round(ch * ratio)
    return rw, rh, (pw - rw) // 2, (ph - rh) // 2


class MaskCropper:
    """crop_mask (utils/usdu_utils.py:415-442) on the GPU.  One instance per job: the truncated u8
    copy of every mask tensor and the coefficient / index tables are built once and reused for
    every tile.  Returns CUDA tensors (the reference returns CPU tensors that ComfyUI then moves
    to the sampling device)."""

    def __init__(self, device=None):
        if not torch.cuda.is_available():
            from ._native import NativeError
            raise NativeError("mask conditioning is cropped by the CUDA library (csrc/usdu_plane.cu); "
                              "no CUDA device is visible and there is no CPU fallback")
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self._masks = {}     # id(tensor) -> (tensor kept alive, u8 copy on the device)
        self._tables = {}    # (filter, in, out) -> (host int32, device int32)
        self._index = {}     # (in, out) -> device int32

    # -- cached operands ---------------------------------------------------------------------
    def _quantised(self, mask: torch.Tensor) -> torch.Tensor:
        from . import _native as nat
        hit = self._masks.get(id(mask))
        if hit is not None and hit[0] is mask:
            return hit[1]
        x = reference_f32(mask.detach())
        if not x.is_cuda:
            x = x.contiguous()
            x = (x if x.is_pinned() else x.pin_memory()).to(self.device, non_blocking=True)
        x = x.contiguous()
        q = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
        nat.pack_tiles_u8(x.data_ptr(), q.data_ptr(), x.numel(), torch.cuda.current_stream().cuda_stream)
        self._masks[id(mask)] = (mask, q)
        return q

    def _table(self, filt: int, n_in: int, n_out: int):
        if n_in == n_out:
            return None, None            # Pillow skips a pass whose axis keeps its size
        key = (filt, n_in, n_out)
        if key not in self._tables:
            from . import _native as nat
            host = nat.build_filter_table(filt, n_in, n_out)
            self._tables[key] = (host, torch.from_numpy(host).to(self.device))
        return self._tables[key]

    def _nearest(self, n_in: int, n_out: int) -> torch.Tensor:
        key = (n_in, n_out)
        if key not in self._index:
            from . import _native as nat
            self._index[key] = torch.from_numpy(nat.nearest_index(n_in, n_out)).to(self.device)
        return self._index[key]

    # -- one resize of n planes, window [ox, ox+ow) x [oy, oy+oh) of the (out_w, out_h) result ---
    def _resize(self, src: torch.Tensor, filt: int, out_w: int, out_h: int, window=None) -> torch.Tensor:
        from . import _native as nat
        n, h, w = src.shape
        ox, oy, ow, oh = (0, 0, out_w, out_h) if window is None else window
        th_host, th_dev = self._table(filt, w, out_w)
        tv_host, tv_dev = self._table(filt, h, out_h)
        dst = torch.empty((n, oh, ow), dtype=torch.uint8, device=src.device)
        mid, y0, rows = None, 0, 0
        if th_dev is not None and tv_dev is not None:
            y0, rows = nat.table_input_span(tv_host, oy, oh)
            mid = torch.empty((n, rows, (ow + 3) // 4 * 4), dtype=torch.uint8, device=src.device)
        nat.plane_resample_u8(src.data_ptr(), n, h, w, src.stride(1), src.stride(0),
                              th_dev.data_ptr() if th_dev is not None else None, ox, ow,
                              tv_dev.data_ptr() if tv_dev is not None else None, oy, oh, y0, rows,
                              mid.data_ptr() if mid is not None else None,
                              dst.data_ptr(), dst.stride(1), dst.stride(0), torch.cuda.current_stream().cuda_stream)
        return dst

    def crop(self, mask: torch.Tensor, region: Region, canvas_size, tile_size) -> torch.Tensor:
        """mask fp32 [Bm, Hm, Wm] in [0,1] -> fp32 [Bm, ph, pw] (values k/255) on the GPU."""
        from . import _native as nat
        if mask.dim() != 3:
            raise ValueError(f"mask conditioning must be [B, H, W], got {tuple(mask.shape)}")
        W, H = int(canvas_size[0]), int(canvas_size[1])
        pw, ph = int(tile_size[0]), int(tile_size[1])
        x1, y1, x2, y2 = (int(v) for v in region)
        if not (0 <= x1 < x2 <= W and 0 <= y1 < y2 <= H):
            raise ValueError(f"crop region {region} outside the canvas {W}x{H}")
        with torch.cuda.device(self.device):
            q = self._quantised(mask)
            cw, ch = x2 - x1, y2 - y1
            m = self._resize(q, nat.FILTER_BICUBIC, W, H, window=(x1, y1, cw, ch))      # :424 + :427
            rw, rh, hp, vp = mask_fit_geometry(cw, ch, pw, ph)
            m = self._resize(m, nat.FILTER_LANCZOS, rw, rh)                              # :258
            if hp or vp:                                                                   # :262, pad_image2 fill
                n = m.shape[0]
                padded = torch.empty((n, rh + 2 * vp, rw + 2 * hp), dtype=torch.uint8, device=m.device)
                rows = self._nearest(rh - 2, rh + 2 * vp) if hp else None
                cols = self._nearest(rw - 2, rw + 2 * hp) if vp else None
                nat.plane_pad_fill_u8(m.data_ptr(), n, rh, rw, m.stride(1), m.stride(0), hp, vp,
                                      rows.data_ptr() if rows is not None else None,
                                      cols.data_ptr() if cols is not None else None,
                                      padded.data_ptr(), padded.stride(1), padded.stride(0),
                                      torch.cuda.current_stream().cuda_stream)
                m = padded
            m = self._resize(m, nat.FILTER_LANCZOS, pw, ph)                              # :263 (always ends at the tile size, so :434-435 never fires)
            out = torch.empty(m.shape, dtype=torch.float32, device=m.device)
            nat.unpack_tiles_f32(m.data_ptr(), out.data_ptr(), m.numel(), torch.cuda.current_stream().cuda_stream)
        return out


def crop_mask(opts: dict, region: Region, canvas_size, tile_size, cropper: Optional[MaskCropper] = None):
    mask = opts.get("mask")
    if mask is None:
        return
    opts["mask"] = (cropper or MaskCropper()).crop(mask, region, canvas_size, tile_size)


def crop_cond(cond, region: Region, init_size, canvas_size, tile_size, w_pad: int = 0, h_pad: int = 0,
              mask_cropper: Optional[MaskCropper] = None):
    """utils/usdu_utils.py:506-517 on an already cloned conditioning list."""
    out = []
    for emb, opts in cond:
        d = dict(opts)
        crop_control_hints(d, region, canvas_size, tile_size)
        crop_gligen(d, region, init_size, canvas_size, w_pad, h_pad)
        crop_area(d, region, init_size, canvas_size, w_pad, h_pad)
        crop_mask(d, region, canvas_size, tile_size, mask_cropper)
        crop_reference_latents(d, region, canvas_size, tile_size)
        out.append([emb, d])
    return out


def make_cond_cropper():
    """-> fn(positive, negative, tile, tile_size (w,h), image_size (w,h)) used by ComfySampler,
    mirroring process_tiles_batch (upscale/tile_ops.py:263-273).  Masks are cropped from the
    caller's tensors (cached u8 copy), everything else from a per-tile clone."""
    state = {}

    def _masks(cond):
        return [opts.get("mask") for _, opts in cond]

    def crop(positive, negative, tile, tile_size, image_size):
        region = (tile.x1, tile.y1, tile.x2, tile.y2)
        has_mask = any(m is not None for m in _masks(positive) + _masks(negative))
        cropper = None
        if has_mask:
            cropper = state.setdefault("cropper", MaskCropper())
        out = []
        for cond in (positive, negative):
            cloned = clone_conditioning(cond, clone_masks=False)
            out.append(crop_cond(cloned, region, image_size, image_size, tile_size, mask_cropper=cropper))
        return out[0], out[1]
    return crop
