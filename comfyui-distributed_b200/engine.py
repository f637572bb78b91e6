"""Device pipeline of the USDU tile path on one H100: u8 canvas resident in HBM, tiles
cropped / blended by the sm_90a kernels in libusdu_b200.so, the sampler injected as a
callable on device tensors.  torch is used for memory, streams and (in dist.py) NCCL.

Replaces upscale/modes/single_gpu.py:8-72 (progressive driver) and the pixel half of
upscale/modes/static.py (per-participant canvases, sorted final blend :521-553).
"""
from __future__ import annotations

import contextlib
import os
import threading
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _native as nat
from .casts import reference_f32
from .lru import LruCache
from .planner import Plan, Tile, WorkList, get_plan

Denoiser = Callable[[torch.Tensor, List[Tile]], torch.Tensor]
"""denoise(tiles fp32 cuda [n, B, ph, pw, 3] in [0,1], tile rows) -> same shape, fp32.
The n tiles of one call have pairwise disjoint crop windows (they are independent)."""


def _require_cuda(t: torch.Tensor, what: str):
    if not t.is_cuda:
        raise nat.NativeError(f"{what} must be a CUDA tensor: the USDU kernels have no CPU path")


def _stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


# Every frame of a batch is one grid.y index of the crop and blend launches, whose limit is 65,535.  A larger batch is
# refused before any device work.  It is not run in chunks: a sampler sees the whole batch per tile, so chunking would
# change the noise it draws.
MAX_BATCH = 65535


def check_batch(B: int):
    if B > MAX_BATCH:
        raise ValueError(f"Batch size {B} exceeds {MAX_BATCH} frames, the most one tile launch takes. "
                         "Please split the batch.")


class KernelProfile:
    """Optional per-launch CUDA-event timing on the launching stream (bench.py's roofline).
    Usage: prof = KernelProfile(); engine.PROFILE = prof; ...; prof.summary()."""

    def __init__(self):
        self.rec = []          # (name, ev0, ev1, algorithmic bytes) of eager launches since begin_step()
        self.graph_rec = []    # the same for launches captured into a CUDA graph (re-recorded on every replay)
        self.capturing = False

    def begin_step(self):
        """Forget the eager records of earlier steps: summary() then describes ONE step."""
        self.rec = []

    def launch(self, name: str, nbytes: int, fn):
        # external=True: inside a CUDA-graph capture these become event-record NODES, so the
        # timestamps are taken on the device between back-to-back kernels (no host gaps)
        e0 = torch.cuda.Event(enable_timing=True, external=True)
        e1 = torch.cuda.Event(enable_timing=True, external=True)
        e0.record()
        fn()
        e1.record()
        (self.graph_rec if self.capturing else self.rec).append((name, e0, e1, nbytes))

    def summary(self) -> dict:
        torch.cuda.synchronize()
        out = {}
        for name, e0, e1, nb in self.rec + self.graph_rec:
            d = out.setdefault(name, {"launches": 0, "ms": 0.0, "bytes": 0})
            d["launches"] += 1
            d["ms"] += e0.elapsed_time(e1)
            d["bytes"] += nb
        for d in out.values():
            d["gbps"] = d["bytes"] / (d["ms"] * 1e-3) / 1e9 if d["ms"] > 0 else 0.0
            d["avg_us"] = d["ms"] * 1e3 / max(d["launches"], 1)
        return out


PROFILE: Optional[KernelProfile] = None
FORCE_GENERIC = False     # tests: run the generic (any-scale) kernels even when the fast ones apply
FORCE_NO_MMA = os.environ.get("USDU_NO_MMA", "0") == "1"   # tests / A-B runs: integer-pipe fast kernels instead of the tensor-core ones
PATH_FLAGS = (0, nat.FLAG_FAST, nat.FLAG_MMA)
_PATHS = {"generic": 0, "fast": 1, "mma": 2}
PATH_CROP = _PATHS[os.environ.get("USDU_CROP_PATH", "mma")]      # best build per kernel (upper bound: the plan may not support it)
PATH_BLEND = _PATHS[os.environ.get("USDU_BLEND_PATH", "mma")]
USE_CUDA_GRAPHS = True    # capture the wave loop when the sampler is cuda_graph_safe


def _launch(name: str, nbytes: int, fn):
    if PROFILE is not None:
        PROFILE.launch(name, nbytes, fn)
    else:
        fn()


class DevicePlan:
    """Plan tables resident on one device (+ the feather templates, built there)."""

    _cache: "LruCache[DevicePlan]" = LruCache(8)

    def __init__(self, plan: Plan, device: torch.device):
        self.plan = plan
        self.device = device
        self.tiles = torch.from_numpy(plan.tile_desc).to(device)
        self.tabs = torch.from_numpy(plan.tabs).to(device)
        self.mask_pool = torch.empty(plan.mask_pool_bytes, dtype=torch.uint8, device=device)
        scratch = torch.empty(nat.mask_scratch_bytes(plan.mask_specs), dtype=torch.uint8, device=device)
        with torch.cuda.device(device):
            nat.build_feather_masks(plan.mask_specs, self.mask_pool.data_ptr(), scratch.data_ptr(), _stream_ptr())
        torch.cuda.current_stream(device).synchronize()   # scratch may be freed now
        self._wl: Dict[tuple, tuple] = {}

    @classmethod
    def get(cls, plan: Plan, device: torch.device) -> "DevicePlan":
        key = (id(plan), device.index)
        return cls._cache.get_or_build(key, lambda: DevicePlan(plan, device), lambda dp: dp.plan is plan)

    def _upload(self, wl: WorkList):
        items = torch.from_numpy(wl.items).to(self.device)
        cover = torch.from_numpy(wl.cover).to(self.device) if wl.cover is not None else None
        return items, cover

    def crop_list(self, tile_ids: Tuple[int, ...], B: int, use_fast: bool):
        key = ("crop", tile_ids, B, use_fast)
        if key not in self._wl:
            wl, offs, total = self.plan.crop_worklist(tile_ids, B, use_fast)
            self._wl[key] = (wl, offs, total) + self._upload(wl)
        return self._wl[key]

    def blend_list(self, tile_ids: Tuple[int, ...], offs: np.ndarray, src_u8: bool, use_fast: bool, B: int = 1,
                   part: Optional[Tuple[int, int]] = None):
        key = ("blend", tile_ids, tuple(int(o) for o in offs), src_u8, use_fast, B, part)
        if key not in self._wl:
            wl = self.plan.blend_worklist(tile_ids, offs, 1 if src_u8 else 4, use_fast, B, part)
            self._wl[key] = (wl,) + self._upload(wl)
        return self._wl[key]

    def split_lists(self, waves: Sequence[Sequence[int]], B: int, path_crop: int, path_blend: int):
        """Per dependency wave, the work lists of the split schedule (planner.split_lists), uploaded:
        dict(crop=(wl, items) on the chain, early=(wl, items) beside the previous wave or None, offs, total,
        blend=(wl, items)), or None when some list would not run on job records."""
        key = ("split", tuple(tuple(int(t) for t in w) for w in waves), B, path_crop, path_blend)
        if key not in self._wl:
            out = None
            if self.plan.kernel_path(path_crop) >= 1 and self.plan.kernel_path(path_blend) >= 1:
                out = []
                for k, wave in enumerate(waves):
                    offs, _ = self.plan.slot_offsets(wave, B)
                    chain, side, coffs, ctotal, bl = self.plan.split_lists(wave, offs, waves[k - 1] if k else None, B, path_crop)
                    if path_blend != path_crop:
                        bl = self.plan.blend_worklist(wave, offs, 4, path_blend, B)
                    out.append({"crop": (chain, self._upload(chain)[0]), "offs": coffs, "total": ctotal,
                                "early": None if side is None else (side, self._upload(side)[0]), "blend": (bl, self._upload(bl)[0])})
            self._wl[key] = out
        return self._wl[key]


class Canvas:
    """The progressive u8 canvas [B, H, pitch] of one participant."""

    def __init__(self, dplan: DevicePlan, B: int, buf: Optional[torch.Tensor] = None):
        self.dp = dplan
        self.plan = dplan.plan
        self.B = B
        self.pitch = self.pitch_of(self.plan.W)
        if buf is None:
            # 16 bytes of slack behind the last row: the LDG staging of the integer-pipe kernels reads whole 12-byte chunks
            # and, for widths that are not multiples of 4, may touch up to 4 bytes past the last row's pitch (discarded)
            n = B * self.plan.H * self.pitch
            buf = torch.empty(n + 16, dtype=torch.uint8, device=dplan.device)[:n].view(B, self.plan.H, self.pitch)
        elif tuple(buf.shape) != (B, self.plan.H, self.pitch) or buf.dtype != torch.uint8 or not buf.is_contiguous():
            raise ValueError(f"canvas buffer must be contiguous uint8 [{B},{self.plan.H},{self.pitch}]")
        self.buf = buf                      # caller-owned when given (dist.py: symmetric memory peers can address)
        self.launches = 0
        self.algo_bytes = 0
        self.path = 0 if FORCE_GENERIC else self.plan.kernel_path(1 if FORCE_NO_MMA else None)   # 0 generic, 1 fast, 2 tensor-core
        # per kernel: the tensor-core build where the plan supports it, the integer-pipe build otherwise;
        # both give identical bytes
        self.path_crop = min(self.path, PATH_CROP)
        self.path_blend = min(self.path, PATH_BLEND)

    @staticmethod
    def pitch_of(W: int) -> int:
        return (W * 3 + 127) // 128 * 128

    # Q0 (single_gpu.py:30-32)
    def load(self, image: torch.Tensor):
        _require_cuda(image, "image")
        p = self.plan
        if tuple(image.shape) != (self.B, p.H, p.W, 3) or image.dtype != torch.float32:
            raise ValueError(f"image must be float32 [{self.B},{p.H},{p.W},3], got {image.dtype} {tuple(image.shape)}")
        image = image.contiguous()
        _launch("quantize", self.B * p.H * p.W * 15,
                lambda: nat.quantize_canvas(image.data_ptr(), self.buf.data_ptr(), self.B, p.H, p.W, self.pitch,
                                            _stream_ptr()))
        self.launches += 1
        return self

    def clone(self) -> "Canvas":
        c = Canvas(self.dp, self.B)
        c.buf.copy_(self.buf)
        return c

    def result(self) -> torch.Tensor:
        p = self.plan
        out = torch.empty((self.B, p.H, p.W, 3), dtype=torch.float32, device=self.buf.device)
        _launch("dequantize", self.B * p.H * p.W * 15,
                lambda: nat.dequantize_canvas(self.buf.data_ptr(), out.data_ptr(), self.B, p.H, p.W, self.pitch,
                                              _stream_ptr()))
        self.launches += 1
        return out

    def result_u8(self) -> torch.Tensor:
        return self.buf[:, :, : self.plan.W * 3].reshape(self.B, self.plan.H, self.plan.W, 3)

    # K2 (tile_ops.py:96-155)
    def can_crop_image(self) -> bool:
        """The tensor-core crop can read the fp32 image itself (usdu_tile_crop_resize_f32)."""
        return self.path_crop == 2 and self.plan.W % 4 == 0

    def crop(self, tile_ids: Sequence[int], out: Optional[torch.Tensor] = None, image: Optional[torch.Tensor] = None):
        """-> (flat fp32 buffer, element offsets per tile).  Tile i is
        buffer[offs[i] : offs[i] + B*ph*pw*3].view(B, ph, pw, 3).
        image: crop the windows straight from this fp32 image [B,H,W,3] instead of the canvas (identical tiles as long
        as the canvas still is the quantised image there: a conflict-free partition, dist.StaticJob)."""
        tile_ids = tuple(int(t) for t in tile_ids)
        wl, offs, total, items, _ = self.dp.crop_list(tile_ids, self.B, self.path_crop)
        if image is not None:
            if not (self.can_crop_image() and wl.path == 2):
                raise nat.NativeError("crop from the fp32 image needs the tensor-core kernels and a canvas width that is a multiple of 4")
            _require_cuda(image, "image")
            if tuple(image.shape) != (self.B, self.plan.H, self.plan.W, 3) or image.dtype != torch.float32 or not image.is_contiguous():
                raise ValueError("crop: image must be contiguous float32 [B,H,W,3] of the plan's size")
            if out is None:
                out = torch.empty(total, dtype=torch.float32, device=self.buf.device)
            p = self.plan
            _launch("crop_resize", (wl.algo_bytes + 9 * sum(p.tiles[t].ew * p.tiles[t].eh for t in tile_ids)) * self.B,
                    lambda: nat.tile_crop_resize_f32(image.data_ptr(), self.B, p.H, p.W, self.dp.tabs.data_ptr(), items.data_ptr(),
                                                     items.shape[0], wl.patch_w, wl.patch_h, out.data_ptr(),
                                                     PATH_FLAGS[2] | (nat.FLAG_MMA_KS2 if wl.ks2 else 0), _stream_ptr()))
            self.launches += 1
            self.algo_bytes += wl.algo_bytes * self.B
            return out, offs
        if out is None:
            out = torch.empty(total, dtype=torch.float32, device=self.buf.device)
        elif out.numel() < total or out.dtype != torch.float32 or not out.is_cuda:
            raise ValueError("crop: `out` too small or wrong dtype/device")
        self.crop_jobs(wl, items, out)
        return out, offs

    def crop_jobs(self, wl: WorkList, items: torch.Tensor, out: torch.Tensor):
        """One crop launch over an explicit work list (the whole wave, or one part of a split wave)."""
        p = self.plan
        _launch("crop_resize", wl.algo_bytes * self.B,
                lambda: nat.tile_crop_resize(self.buf.data_ptr(), self.B, p.H, p.W, self.pitch,
                                             self.dp.tiles.data_ptr(), self.dp.tabs.data_ptr(), items.data_ptr(),
                                             items.shape[0], wl.patch_w, wl.patch_h, out.data_ptr(),
                                             PATH_FLAGS[wl.path] | (wl.block_rows << 8) | (wl.block_cols << 16) |
                                             (nat.FLAG_MMA_KS2 if wl.ks2 else 0), _stream_ptr()))
        self.launches += 1
        self.algo_bytes += wl.algo_bytes * self.B

    # K4 (tile_ops.py:310-349 after the truncating cast of single_gpu.py:60)
    def blend(self, tile_ids: Sequence[int], src: torch.Tensor, offs: np.ndarray,
              part: Optional[Tuple[int, int]] = None, canvas_ptr: Optional[int] = None):
        """Composite processed tiles into the canvas in the ORDER of `tile_ids`.
        src: flat fp32 (sampler output) or uint8 (already quantised) buffer.
        part = (i, n): this launch takes the i-th of n shares of the canvas blocks; canvas_ptr: device
        address of ANOTHER participant's canvas of the same geometry (peer memory) to composite into."""
        _require_cuda(src, "src")
        tile_ids = tuple(int(t) for t in tile_ids)
        if src.dtype not in (torch.float32, torch.uint8):
            raise ValueError(f"blend: src must be float32 or uint8, got {src.dtype}")
        src_u8 = src.dtype == torch.uint8
        wl, items, cover = self.dp.blend_list(tile_ids, offs, src_u8, self.path_blend, self.B, part)
        self.blend_jobs(wl, items, cover, src, canvas_ptr)

    def blend_jobs(self, wl: WorkList, items: torch.Tensor, cover: Optional[torch.Tensor], src: torch.Tensor,
                   canvas_ptr: Optional[int] = None):
        """One blend launch over an explicit work list (all blocks of the tiles, or one part of a split wave)."""
        if items.shape[0] == 0:
            return
        p = self.plan
        src = src.contiguous()
        src_u8 = src.dtype == torch.uint8
        n_grid = wl.n_launch if wl.n_launch >= 0 else items.shape[0]
        flags = PATH_FLAGS[wl.path] | (wl.block_rows << 8) | (wl.block_cols << 16) | (nat.FLAG_MMA_KS2 if wl.ks2 else 0)
        target = self.buf.data_ptr()
        if canvas_ptr is not None and canvas_ptr != target:
            target, flags = canvas_ptr, flags | nat.FLAG_REMOTE_CANVAS
        cover_ptr = cover.data_ptr() if cover is not None else 0
        _launch("blend", wl.algo_bytes * self.B,
                lambda: nat.tile_blend(target, self.B, p.H, p.W, self.pitch, self.dp.tiles.data_ptr(),
                                       self.dp.tabs.data_ptr(), self.dp.mask_pool.data_ptr(), items.data_ptr(),
                                       n_grid, cover_ptr, wl.patch_w, wl.patch_h, src.data_ptr(),
                                       src_u8, flags, _stream_ptr()))
        self.launches += 1
        self.algo_bytes += wl.algo_bytes * self.B


def tile_views(plan: Plan, tile_ids: Sequence[int], buf: torch.Tensor, offs: np.ndarray, B: int):
    """Group consecutive same-shape tiles of a packed buffer into [n, B, ph, pw, 3] views."""
    groups = []
    i = 0
    ids = list(tile_ids)
    while i < len(ids):
        t = plan.tiles[ids[i]]
        j = i
        while j + 1 < len(ids) and (plan.tiles[ids[j + 1]].pw, plan.tiles[ids[j + 1]].ph) == (t.pw, t.ph):
            j += 1
        n = j - i + 1
        sz = B * t.ph * t.pw * 3
        view = buf[int(offs[i]): int(offs[i]) + n * sz].view(n, B, t.ph, t.pw, 3)
        groups.append((ids[i:j + 1], view))
        i = j + 1
    return groups


def denoise_packed(plan: Plan, tile_ids: Sequence[int], buf: torch.Tensor, offs: np.ndarray, B: int,
                   denoiser: Denoiser) -> torch.Tensor:
    groups = tile_views(plan, tile_ids, buf, offs, B)
    if len(groups) == 1:   # uniform tiles: the sampler's output IS the packed buffer
        ids, view = groups[0]
        res = denoiser(view, [plan.tiles[i] for i in ids])
        if tuple(res.shape) != tuple(view.shape):
            raise ValueError(f"denoiser returned {tuple(res.shape)}, expected {tuple(view.shape)}")
        _require_cuda(res, "denoiser output")
        return reference_f32(res).contiguous().view(-1)
    out = torch.empty_like(buf)
    for ids, view in groups:
        res = denoiser(view, [plan.tiles[i] for i in ids])
        if tuple(res.shape) != tuple(view.shape):
            raise ValueError(f"denoiser returned {tuple(res.shape)}, expected {tuple(view.shape)}")
        _require_cuda(res, "denoiser output")
        o0 = int(offs[list(tile_ids).index(ids[0])])
        out[o0: o0 + view.numel()].view_as(view).copy_(reference_f32(res))
    return out


def _sorted_by_shape(plan: Plan, ids: Sequence[int]) -> List[int]:
    return sorted(ids, key=lambda i: (plan.tiles[i].ph, plan.tiles[i].pw, i))


def processing_order(plan: Plan, tile_ids: Sequence[int]) -> List[int]:
    """The order in which run_progressive handles `tile_ids`: wave by wave, same-shape tiles
    adjacent inside a wave (every rank can compute every other rank's order from the plan)."""
    return [t for w in plan.waves(tile_ids) for t in _sorted_by_shape(plan, w)]


def run_progressive(canvas: Canvas, order: Sequence[int], denoiser: Denoiser, keep_processed: bool = False,
                    payload: Optional[torch.Tensor] = None, where: Optional[dict] = None, skip: Sequence[str] = (),
                    crop_buf: Optional[torch.Tensor] = None):
    """Process `order` (tile ids) with the reference's progressive semantics on `canvas`
    (single_gpu.py:40-64 / static.py:242-280): wave by wave, each wave = crop kernel,
    one sampler call, blend kernel.  What a static-mode worker ships to the master (the
    truncated u8 tiles, worker_comms.py:30-33) is either returned as {tile id: u8 [B,ph,pw,3]}
    (keep_processed) or written straight into `payload` at `where[tile] = (rank, byte offset)`."""
    plan, B = canvas.plan, canvas.B
    shipped: Dict[int, torch.Tensor] = {}
    scratch = None
    waves = [_sorted_by_shape(plan, w) for w in plan.waves(order)]
    for wave in waves:
        if "crop" in skip and crop_buf is not None:    # the caller cropped this (single) wave itself: GraphedWaves.replay_from_image
            offs, total = plan.slot_offsets(wave, B)
            buf = crop_buf[:total]
        elif "crop" in skip:    # bench.py's differencing measurement: same graph minus one kernel kind
            offs, total = plan.slot_offsets(wave, B)
            if scratch is None or scratch.numel() < total:
                scratch = torch.zeros(total, dtype=torch.float32, device=canvas.buf.device)
            buf = scratch[:total]
        else:
            buf, offs = canvas.crop(wave)
        out = denoise_packed(plan, wave, buf, offs, B, denoiser)
        if "blend" not in skip:
            canvas.blend(wave, out, offs)
        if payload is not None:
            sizes = [B * plan.tiles[t].ph * plan.tiles[t].pw * 3 for t in wave]
            base = where[wave[0]][1]
            dense = all(sz % 16 == 0 for sz in sizes) and all(where[t][1] == base + int(offs[i]) for i, t in enumerate(wave))
            if dense:        # the wave occupies one contiguous span of the payload: pack in place
                nat.pack_tiles_u8(out.data_ptr(), payload[base:].data_ptr(), out.numel(), _stream_ptr())
                canvas.launches += 1
            else:
                q = torch.empty(out.numel(), dtype=torch.uint8, device=out.device)
                nat.pack_tiles_u8(out.data_ptr(), q.data_ptr(), out.numel(), _stream_ptr())
                canvas.launches += 1
                for i, tid in enumerate(wave):
                    payload[where[tid][1]: where[tid][1] + sizes[i]] = q[int(offs[i]): int(offs[i]) + sizes[i]]
        elif keep_processed:
            q = torch.empty(out.numel(), dtype=torch.uint8, device=out.device)
            nat.pack_tiles_u8(out.data_ptr(), q.data_ptr(), out.numel(), _stream_ptr())
            canvas.launches += 1
            for i, tid in enumerate(wave):
                t = plan.tiles[tid]
                n = B * t.ph * t.pw * 3
                shipped[tid] = q[int(offs[i]): int(offs[i]) + n].view(B, t.ph, t.pw, 3)
    return shipped


# split_crop (default: waves whose crop launches are split by what they really depend on, run_split) | waves (the plain
# level loop, run_progressive)
SCHEDULE = os.environ.get("USDU_SCHEDULE", "split_crop")
SCHEDULES = ("waves", "split_crop")
if SCHEDULE not in SCHEDULES:
    raise ValueError(f"USDU_SCHEDULE={SCHEDULE!r}: expected one of {', '.join(SCHEDULES)}")


# The canvas quantise / dequantise of a graphed 1-GPU job as row bands inside the wave graph (CastBands, run_split), beside
# the waves that do not touch those rows.  USDU_STREAM_OVERLAP=0 keeps the two eager whole-canvas passes around the graph.
# USDU_STREAM_CTAS: CTAs of a band beside the waves; USDU_STREAM_BANDS: bands per pass; USDU_STREAM_PRIORITY=1: the wave
# kernels outrank the bands in CTA dispatch (usdu_graph_instantiate).  Defaults from the sweep in DESIGN section 9.2.
STREAM_OVERLAP = os.environ.get("USDU_STREAM_OVERLAP", "1") == "1"
STREAM_CTAS = int(os.environ.get("USDU_STREAM_CTAS", "264"))
STREAM_BANDS = int(os.environ.get("USDU_STREAM_BANDS", "16"))
STREAM_PRIORITY = os.environ.get("USDU_STREAM_PRIORITY", "1") == "1"


class CastBands:
    """The quantise and dequantise passes of one graphed job, cut into row bands (Plan.stream_bands) that run on a
    streaming side stream of the wave graph: every quantise band is enqueued at the start and a stream waits for it just
    before the first crop that reads its rows; a dequantise band forks after the blend of the last wave that writes its
    rows.  The first quantise band and the last dequantise band have nothing beside them and run on the whole machine;
    the others use at most `max_ctas` CTAs.  The fp32 image and result addresses live in a device-side argument block
    (usdu_stream_args) that `set` rewrites before every replay, so one captured graph serves every caller's tensors."""

    def __init__(self, canvas: Canvas, order: Sequence[int], n_bands: int, max_ctas: int):
        # gated by the rows of the lists the graph launches: a taller early crop box reads rows the default lists do not
        lists = canvas.dp.split_lists(split_waves(canvas.plan, order), canvas.B, canvas.path_crop, canvas.path_blend)
        if lists is None:
            raise nat.NativeError("canvas cast bands need the split schedule's job-record work lists")
        levels = [([L["crop"][0]] + ([L["early"][0]] if L["early"] is not None else []), L["blend"][0]) for L in lists]
        self.q, self.d = canvas.plan.stream_bands(order, canvas.B, n_bands, levels=levels)
        dev = canvas.buf.device
        self.args = torch.zeros(nat.STREAM_ARGS_BYTES, dtype=torch.uint8, device=dev)
        self.stream = torch.cuda.Stream(device=dev)
        self.max_ctas = max_ctas
        self.full = max(nat.sm_count(), 1) * 128
        self._ev: List[torch.cuda.Event] = []
        self._waited: Dict[int, int] = {}

    @staticmethod
    def eligible(canvas: Canvas) -> bool:
        return canvas.plan.W % 4 == 0

    def set(self, image: torch.Tensor, out: torch.Tensor):
        nat.stream_args_set(self.args.data_ptr(), image.data_ptr(), out.data_ptr(), _stream_ptr())

    def start(self, canvas: Canvas, main: "torch.cuda.Stream"):
        """Fork the streaming stream off `main` and enqueue every quantise band on it."""
        p, s = canvas.plan, self.stream
        self._ev, self._waited = [], {}
        fork = torch.cuda.Event()
        fork.record(main)
        s.wait_event(fork)
        with torch.cuda.stream(s):
            for i, (y0, y1, _) in enumerate(self.q):
                nat.quantize_rows_streamed(self.args.data_ptr(), canvas.buf.data_ptr(), canvas.B, p.H, p.W, canvas.pitch, y0, y1,
                                           self.full if i == 0 else self.max_ctas, _stream_ptr())
                canvas.launches += 1
                e = torch.cuda.Event()
                e.record(s)
                self._ev.append(e)

    def need(self, k: int, stream: "torch.cuda.Stream"):
        """`stream` waits for every quantise band that wave k touches (the bands run in order: the last one suffices)."""
        j = max((i for i, b in enumerate(self.q) if b[2] <= k), default=-1)
        if j > self._waited.get(id(stream), -1):
            stream.wait_event(self._ev[j])
            self._waited[id(stream)] = j

    def after_blend(self, k: int, canvas: Canvas, main: "torch.cuda.Stream"):
        """Fork the dequantise bands whose rows no wave after k writes."""
        bands = [i for i, b in enumerate(self.d) if b[2] == k]
        if not bands:
            return
        p, s = canvas.plan, self.stream
        e = torch.cuda.Event()
        e.record(main)
        s.wait_event(e)
        with torch.cuda.stream(s):
            for i in bands:
                y0, y1, _ = self.d[i]
                nat.dequantize_rows_streamed(canvas.buf.data_ptr(), self.args.data_ptr(), canvas.B, p.H, p.W, canvas.pitch, y0, y1,
                                             self.full if i == len(self.d) - 1 else self.max_ctas, _stream_ptr())
                canvas.launches += 1

    def join(self, main: "torch.cuda.Stream"):
        e = torch.cuda.Event()
        e.record(self.stream)
        main.wait_event(e)


def use_split(canvas: Canvas, order: Sequence[int]) -> bool:
    """USDU_SCHEDULE=split_crop: level waves whose crop launches are split by what they really depend on."""
    return SCHEDULE == "split_crop" and canvas.path_crop >= 1 and canvas.path_blend >= 1 and len(canvas.plan.waves(order)) > 2


def split_waves(plan: Plan, order: Sequence[int]) -> List[List[int]]:
    """The dependency waves of `order` as run_split launches them: same-shape tiles adjacent."""
    return [_sorted_by_shape(plan, w) for w in plan.waves(order)]


def run_split(canvas: Canvas, order: Sequence[int], denoiser: Denoiser, s_early: "torch.cuda.Stream",
              casts: Optional[CastBands] = None) -> bool:
    """run_progressive(order) with every level's crop launch split by dependency (planner.split_lists); meant to be
    stream-captured.  single_gpu.py:40-64 orders a crop only after the blends that CHANGE pixels it reads:
    crop(k+1) = `late` jobs (their staged rectangle meets a feather support of wave k) + `early` jobs, which run on
    `s_early` beside sampler(k) / blend(k).  The chain per level shrinks to crop_late -> sampler -> blend (about a quarter
    of the crop jobs on cfg2).  A crop beside a blend only ever reads bytes whose value the blend leaves as it is.
    The late jobs run in short blocks (latency: they are on the chain), the early ones in tall blocks (fewer staged rows:
    they share the machine with blend(k)).
    False (nothing launched) when a wave has no job-record lists.
    casts: the canvas quantise / dequantise bands (CastBands) run inside the same graph: a crop waits for the quantise
    bands it reads, a dequantise band forks after the last blend that writes its rows."""
    plan, B = canvas.plan, canvas.B
    waves = split_waves(plan, order)
    lists = canvas.dp.split_lists(waves, B, canvas.path_crop, canvas.path_blend)
    if lists is None:
        return False
    dev = canvas.buf.device
    main = torch.cuda.current_stream(dev)
    bufs = [None] * len(waves)
    early_done = [None] * len(waves)
    bufs[0] = torch.empty(lists[0]["total"], dtype=torch.float32, device=dev)
    if casts is not None:
        casts.start(canvas, main)
    for k, wave in enumerate(waves):
        L = lists[k]
        buf = bufs[k]
        if casts is not None:
            casts.need(k, main)
        canvas.crop_jobs(L["crop"][0], L["crop"][1], buf)
        if early_done[k] is not None:
            main.wait_event(early_done[k])
        out = denoise_packed(plan, wave, buf, L["offs"], B, denoiser)
        if k + 1 < len(waves):                    # the crop jobs of wave k+1 that do not read what wave k changes
            N = lists[k + 1]
            bufs[k + 1] = torch.empty(N["total"], dtype=torch.float32, device=dev)
            if N["early"] is not None:
                fork = torch.cuda.Event()
                fork.record(main)
                s_early.wait_event(fork)
                if casts is not None:
                    casts.need(k + 1, s_early)
                with torch.cuda.stream(s_early):
                    canvas.crop_jobs(N["early"][0], N["early"][1], bufs[k + 1])
                    early_done[k + 1] = torch.cuda.Event()
                    early_done[k + 1].record(s_early)
        canvas.blend_jobs(L["blend"][0], L["blend"][1], None, out)
        if casts is not None:
            casts.after_blend(k, canvas, main)
        bufs[k] = None
    if casts is not None:
        casts.join(main)
    # (every launch on the side streams is already joined through its event; a stream that never joined the capture must
    # not be waited for)
    return True


class GraphedWaves:
    """The wave loop of a progressive job (crop -> sampler -> blend, x waves) captured once
    into a CUDA graph on a static canvas: one graph launch replaces ~5 kernel launches per
    wave, which removes the host enqueue gaps that dominate when the sampler is cheap.
    Only for samplers that declare `cuda_graph_safe` (pure device work, fixed shapes)."""

    _cache: "LruCache[GraphedWaves]" = LruCache(6)

    def __init__(self, dp: DevicePlan, B: int, denoiser: Denoiser, profile: Optional[KernelProfile],
                 order: Optional[Sequence[int]] = None, keep_processed: bool = False,
                 payload: Optional[torch.Tensor] = None, where: Optional[dict] = None, skip: Sequence[str] = (),
                 canvas_buf: Optional[torch.Tensor] = None, external_crop: bool = False, casts: bool = False):
        """casts: the graph also quantises the caller's image and dequantises the result (CastBands; replay_job) when
        the split_crop schedule runs; otherwise the caller fills the canvas and reads it back around the replay."""
        global PROFILE
        self.canvas = Canvas(dp, B, canvas_buf)
        self.denoiser = denoiser
        order = list(range(len(dp.plan.tiles))) if order is None else list(order)
        # external_crop: the tiles (ONE wave: a conflict-free share) are cropped by the caller from the fp32 image right
        # before every replay; the graph starts at the sampler
        self.crop_tiles, self.crop_buf = None, None
        if external_crop:
            waves = dp.plan.waves(order)
            if len(waves) != 1 or not self.canvas.can_crop_image():
                raise ValueError("external_crop needs a single wave and the tensor-core crop")
            self.crop_tiles = _sorted_by_shape(dp.plan, waves[0])
            self.crop_buf = torch.zeros(dp.plan.slot_offsets(self.crop_tiles, B)[1], dtype=torch.float32, device=dp.device)
            skip = tuple(set(skip) | {"crop"})
        self.shipped: Dict[int, torch.Tensor] = {}
        self.payload = payload        # caller-owned transport buffer the packed u8 tiles are written into
        self.canvas.buf.zero_()
        side = torch.cuda.Stream(device=dp.device)
        side.wait_stream(torch.cuda.current_stream(dp.device))
        saved = PROFILE
        PROFILE = None
        # split crops only for the whole job as it is (no per-kernel profile, no tile dictionary, no payload, nothing skipped:
        # bench.py's differencing and external_crop run the plain level loop)
        self.split = (bool(order) and profile is None and not keep_processed and payload is None and not skip
                      and use_split(self.canvas, order))
        s_early = torch.cuda.Stream(device=dp.device) if self.split else None
        self.casts = None
        if casts and STREAM_OVERLAP and self.split and canvas_buf is None and CastBands.eligible(self.canvas):
            self.casts = CastBands(self.canvas, order, STREAM_BANDS, STREAM_CTAS)

        def body(warm_up=False):
            if self.split and run_split(self.canvas, order, denoiser, s_early, None if warm_up else self.casts):
                return {}
            if self.casts is not None:
                raise nat.NativeError("canvas cast bands need the split schedule's job-record work lists")
            return run_progressive(self.canvas, order, denoiser, keep_processed, self.payload, where, skip, self.crop_buf)

        with torch.cuda.stream(side):                 # warm-up: fills every cache (work lists, noise); no casts (no image yet)
            body(warm_up=True)
        torch.cuda.current_stream(dp.device).wait_stream(side)
        torch.cuda.synchronize(dp.device)
        self.canvas.launches = 0
        self.canvas.algo_bytes = 0
        PROFILE = profile
        # with the cast bands the graph is instantiated here (usdu_graph_instantiate: node priorities), not by torch
        self.graph = torch.cuda.CUDAGraph(keep_graph=self.casts is not None)
        self.exec = None
        if profile is not None:
            profile.capturing = True
        try:
            with torch.cuda.graph(self.graph):
                self.shipped = body()
        finally:
            PROFILE = saved
            if profile is not None:
                profile.capturing = False
        if self.casts is not None:
            self.exec = nat.graph_instantiate(self.graph.raw_cuda_graph(), STREAM_PRIORITY)
        self.launches_per_replay = self.canvas.launches
        self.bytes_per_replay = self.canvas.algo_bytes

    def __del__(self):
        if getattr(self, "exec", None):
            nat.graph_exec_destroy(self.exec)
            self.exec = None

    @classmethod
    def get(cls, dp: DevicePlan, B: int, denoiser: Denoiser, profile: Optional[KernelProfile] = None,
            order: Optional[Sequence[int]] = None, keep_processed: bool = False,
            payload: Optional[torch.Tensor] = None, where: Optional[dict] = None, skip: Sequence[str] = (),
            canvas_buf: Optional[torch.Tensor] = None, external_crop: bool = False, casts: bool = False) -> "GraphedWaves":
        pkey = None if payload is None else (payload.data_ptr(), payload.numel())
        ckey = None if canvas_buf is None else canvas_buf.data_ptr()
        ckey_casts = (STREAM_OVERLAP, STREAM_CTAS, STREAM_BANDS, STREAM_PRIORITY) if casts else None
        key = (id(dp), B, getattr(denoiser, "graph_key", id(denoiser)), id(profile), FORCE_GENERIC, FORCE_NO_MMA, SCHEDULE,
               None if order is None else tuple(order), keep_processed, pkey, tuple(skip), ckey, external_crop, ckey_casts)
        return cls._cache.get_or_build(
            key, lambda: GraphedWaves(dp, B, denoiser, profile, order, keep_processed, payload, where, skip, canvas_buf,
                                      external_crop, casts), lambda gw: gw.canvas.dp is dp)

    def replay_job(self, image: torch.Tensor) -> torch.Tensor:
        """The whole job on the caller's fp32 image -> a new fp32 result: with cast bands one replay of the graph, which
        quantises, runs the wave loop and dequantises; otherwise Q0 (eager), the captured wave loop, the dequantise."""
        if self.casts is None:
            return self.replay(image).result()
        c, p = self.canvas, self.canvas.plan
        _require_cuda(image, "image")
        if tuple(image.shape) != (c.B, p.H, p.W, 3) or image.dtype != torch.float32:
            raise ValueError(f"image must be float32 [{c.B},{p.H},{p.W},3], got {image.dtype} {tuple(image.shape)}")
        image = image.contiguous()
        if image.data_ptr() % 16:                  # the vector loads of the streamed quantise
            image = image.clone()
        out = torch.empty((c.B, p.H, p.W, 3), dtype=torch.float32, device=c.buf.device)
        c.launches, c.algo_bytes = self.launches_per_replay, self.bytes_per_replay
        self.casts.set(image, out)
        nat.graph_launch(self.exec, _stream_ptr())
        return out

    def replay(self, image: torch.Tensor) -> Canvas:
        """Q0 from the caller's tensor (eager), then the captured wave loop."""
        if self.casts is not None:
            raise ValueError("this graph quantises its input itself: use replay_job")
        c = self.canvas
        c.launches, c.algo_bytes = self.launches_per_replay, self.bytes_per_replay
        c.load(image)
        self.graph.replay()
        return c

    def replay_from_image(self, image: torch.Tensor) -> Canvas:
        """external_crop: one eager crop launch straight from the caller's fp32 image (no quantised canvas at all), then
        the captured sampler + pack."""
        c = self.canvas
        c.launches, c.algo_bytes = self.launches_per_replay, self.bytes_per_replay
        c.crop(self.crop_tiles, out=self.crop_buf, image=image)
        self.graph.replay()
        return c

    def replay_resident(self) -> Canvas:
        """The captured wave loop on a canvas the caller has already filled with the quantised input."""
        c = self.canvas
        c.launches, c.algo_bytes = self.launches_per_replay, self.bytes_per_replay
        self.graph.replay()
        return c


def upscale_single(image: torch.Tensor, denoiser: Denoiser, tile_width: int, tile_height: int, padding: int,
                   mask_blur: int, force_uniform_tiles: bool = True, stats: Optional[dict] = None,
                   use_graph: Optional[bool] = None, _skip: Sequence[str] = ()) -> torch.Tensor:
    """One-GPU job on a CUDA image [B,H,W,3] fp32 -> fp32 (values k/255), exact
    progressive semantics of process_single_gpu."""
    check_batch(int(image.shape[0]))
    _require_cuda(image, "image")
    B, H, W, _ = image.shape
    plan = get_plan(W, H, tile_width, tile_height, padding, mask_blur, force_uniform_tiles)
    if use_graph is None:
        use_graph = bool(getattr(denoiser, "cuda_graph_safe", False)) and USE_CUDA_GRAPHS
    with torch.cuda.device(image.device):
        dp = DevicePlan.get(plan, image.device)
        if use_graph:
            gw = GraphedWaves.get(dp, B, denoiser, PROFILE, skip=_skip, casts=True)
            res = gw.replay_job(image)
            canvas = gw.canvas
        else:
            canvas = Canvas(dp, B).load(image)
            run_progressive(canvas, range(len(plan.tiles)), denoiser)
            res = canvas.result()
    if stats is not None:
        stats["gpu_launches"] = stats.get("gpu_launches", 0) + canvas.launches
        stats["algo_bytes"] = stats.get("algo_bytes", 0) + canvas.algo_bytes
        stats["tiles"] = len(plan.tiles)
        stats["waves"] = len(plan.waves())
    return res


class WorkerJob:
    """The device state of one static-mode worker of the reference's HTTP master for one job (static.py:191-314): the
    worker's own u8 canvas in HBM, and per tile id the master hands out a 1-tile step -- crop from this canvas, sampler,
    truncating u8 pack of the sampler output, blend into this canvas.  Each crop sees this worker's earlier blends and
    nothing else, as in static.py:242-280.  The packed tile is what the reference's worker PNG-encodes
    (`tensor_to_pil(processed_batch, b)`, worker_comms.py:30): the sampler output at processing size."""

    def __init__(self, image: torch.Tensor, denoiser: Denoiser, tile_width: int, tile_height: int, padding: int,
                 mask_blur: int, force_uniform_tiles: bool = True, device: Optional[torch.device] = None):
        self.device = image.device if image.is_cuda else (device or torch.device("cuda", torch.cuda.current_device()))
        x = reference_f32(image).contiguous()
        B, H, W, _ = x.shape
        self.plan = get_plan(W, H, tile_width, tile_height, padding, mask_blur, force_uniform_tiles)
        self.denoiser = denoiser
        # CUDA-event totals over step() and step_png()
        self.times = {"device_ms": 0.0, "encode_ms": 0.0, "d2h_ms": 0.0, "tiles": 0}
        with torch.cuda.device(self.device):
            if not x.is_cuda:                    # uploaded once; the canvas is all the job keeps
                x = (x if x.is_pinned() else x.pin_memory()).to(self.device, non_blocking=True)
            self.canvas = Canvas(DevicePlan.get(self.plan, self.device), B).load(x)
            torch.cuda.current_stream().synchronize()     # the fp32 upload may be freed now

    def step(self, tile_id: int) -> np.ndarray:
        """Process tile `tile_id` -> its u8 payload [B, ph, pw, 3] in page-locked host memory."""
        tile_id = int(tile_id)
        if not 0 <= tile_id < len(self.plan.tiles):
            raise ValueError(f"tile id {tile_id} is outside this job's {len(self.plan.tiles)} tiles")
        with torch.cuda.device(self.device):
            e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            e0.record()
            q = run_progressive(self.canvas, [tile_id], self.denoiser, keep_processed=True)[tile_id]
            e1.record()
            host = torch.empty(q.shape, dtype=torch.uint8, pin_memory=True)
            host.copy_(q, non_blocking=True)
            e2.record()
            e2.synchronize()
        self.times["device_ms"] += e0.elapsed_time(e1)
        self.times["d2h_ms"] += e1.elapsed_time(e2)
        self.times["tiles"] += 1
        return host.numpy()

    def step_png(self, tile_id: int):
        """Process tile `tile_id` -> its B frames as the PNG files encode_png writes, encoded on the device
        (http_worker.encode_png_gpu) on the same stream and brought back in one copy through page-locked memory.  For a
        tile shape whose layout check failed (http_worker.png_layout) -> step(tile_id)'s u8 tiles, for PIL."""
        from .http_worker import encode_png_gpu, png_layout
        tile_id = int(tile_id)
        if not 0 <= tile_id < len(self.plan.tiles):
            raise ValueError(f"tile id {tile_id} is outside this job's {len(self.plan.tiles)} tiles")
        t = self.plan.tiles[tile_id]
        layout = png_layout(t.ph, t.pw, self.device)
        if layout is None:
            return self.step(tile_id)
        B, n = self.canvas.B, layout.png_len
        with torch.cuda.device(self.device):
            e0, e1, e2, e3 = (torch.cuda.Event(enable_timing=True) for _ in range(4))
            e0.record()
            q = run_progressive(self.canvas, [tile_id], self.denoiser, keep_processed=True)[tile_id]
            e1.record()
            files = encode_png_gpu(q, layout, torch.empty(B * n, dtype=torch.uint8, device=self.device))
            e2.record()
            host = torch.empty(B * n, dtype=torch.uint8, pin_memory=True)
            host.copy_(files, non_blocking=True)
            e3.record()
            e3.synchronize()
        self.times["device_ms"] += e0.elapsed_time(e1)
        self.times["encode_ms"] += e1.elapsed_time(e2)
        self.times["d2h_ms"] += e2.elapsed_time(e3)
        self.times["tiles"] += 1
        data = host.numpy().tobytes()
        return [data[b * n:(b + 1) * n] for b in range(B)]

    def step_device(self, tile_id: int):
        """Process tile `tile_id` into this canvas only (the master of HTTP workers: its tiles never leave the device).
        Enqueued on the current stream, no host synchronisation."""
        tile_id = int(tile_id)
        if not 0 <= tile_id < len(self.plan.tiles):
            raise ValueError(f"tile id {tile_id} is outside this job's {len(self.plan.tiles)} tiles")
        with torch.cuda.device(self.device):
            run_progressive(self.canvas, [tile_id], self.denoiser)
        self.times["tiles"] += 1


# --------------------------------------------------------------------------------------
# host-tensor path: H2D, compute and D2H overlapped band by band
# --------------------------------------------------------------------------------------
def host_bands(plan: Plan, n_bands: int) -> List[dict]:
    """Bands of whole tile rows for the host pipeline.  Per band: `tiles` (row-major ids; processed in
    wave order inside the band), `in` = [lo, hi) image rows that have to be on the device before the band
    starts (everything up to its lowest crop window; consecutive bands continue where the previous one
    stopped, the last one takes the rest), `fin` = [lo, hi) canvas rows that are final once the band is
    done (no later band's feather support reaches them) and can travel back to the host."""
    rows = sorted({t.y for t in plan.tiles})
    n_bands = max(1, min(n_bands, len(rows)))
    cuts = [round(i * len(rows) / n_bands) for i in range(n_bands + 1)]
    bands = []
    fin_lo = in_lo = 0
    for k in range(n_bands):
        ys = set(rows[cuts[k]:cuts[k + 1]])
        tiles = [t.idx for t in plan.tiles if t.y in ys]
        later = [t for t in plan.tiles if t.y > max(ys)]
        in_hi = max(plan.tiles[i].y2 for i in tiles)
        fin_hi = min((t.y1 + plan.support(t)[1] for t in later), default=plan.H)
        fin_hi = max(fin_hi, fin_lo)
        bands.append({"tiles": tiles, "in": (in_lo, max(in_hi, in_lo)), "fin": (fin_lo, fin_hi)})
        in_lo, fin_lo = max(in_hi, in_lo), fin_hi
    bands[-1]["in"] = (bands[-1]["in"][0], plan.H)
    return bands


class HostPipeline:
    """One-GPU job for a HOST image (what ComfyUI hands a node), pipelined over bands of tile
    rows so that PCIe traffic in both directions overlaps with itself and with the kernels.

    The wavefront order used on a resident canvas needs the whole canvas before the first
    row is final (tile (0, last) runs in the same wave as tile (7, 0)), which would serialise
    H2D -> compute -> D2H.  Any topological order of the dependency DAG gives the same result,
    so here the tiles are processed band by band (each band = a few tile rows, wavefront order
    inside): band k needs only the image rows up to its lowest crop window, and once it is done
    every canvas row above the next band's first writable row is final and can travel back
    while later bands are still uploading.  Three streams: upload, compute, download."""

    _cache: "LruCache[HostPipeline]" = LruCache(3)

    def __init__(self, dp: DevicePlan, B: int, denoiser: Denoiser, n_bands: int):
        plan = dp.plan
        self.dp, self.B, self.denoiser = dp, B, denoiser
        dev = dp.device
        self.canvas = Canvas(dp, B)
        self.img = torch.empty((B, plan.H, plan.W, 3), dtype=torch.float32, device=dev)
        self.out = torch.empty((B, plan.H, plan.W, 3), dtype=torch.float32, device=dev)
        self.bands = host_bands(plan, n_bands)
        n_bands = len(self.bands)
        self.s_in, self.s_out = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
        self.graph_safe = bool(getattr(denoiser, "cuda_graph_safe", False)) and USE_CUDA_GRAPHS
        self.graphs = [None] * n_bands
        self.launches = 0

    @classmethod
    def get(cls, dp: DevicePlan, B: int, denoiser: Denoiser, n_bands: int) -> "HostPipeline":
        graph_safe = bool(getattr(denoiser, "cuda_graph_safe", False)) and USE_CUDA_GRAPHS
        # a captured pipeline belongs to one sampler configuration; an eager one serves any sampler
        key = (id(dp), B, getattr(denoiser, "graph_key", id(denoiser)) if graph_safe else "eager", n_bands, FORCE_GENERIC, FORCE_NO_MMA)
        hp = cls._cache.get_or_build(key, lambda: HostPipeline(dp, B, denoiser, n_bands), lambda hp: hp.dp is dp)
        if not hp.graph_safe:
            hp.denoiser = denoiser
        return hp

    def _rows(self, fn, y0: int, y1: int, src: torch.Tensor, dst: torch.Tensor, to_canvas: bool):
        """Quantise / dequantise canvas rows [y0, y1) of every frame (the kernels are row-wise)."""
        p, c = self.dp.plan, self.canvas
        if y1 <= y0:
            return
        for b in range(self.B):
            img_ptr = (src if to_canvas else dst)[b, y0].data_ptr()
            can_ptr = c.buf[b, y0].data_ptr()
            if to_canvas:
                nat.quantize_canvas(img_ptr, can_ptr, 1, y1 - y0, p.W, c.pitch, _stream_ptr())
            else:
                nat.dequantize_canvas(can_ptr, img_ptr, 1, y1 - y0, p.W, c.pitch, _stream_ptr())
            self.launches += 1

    def _band_compute(self, k: int):
        band = self.bands[k]
        if not self.graph_safe:
            run_progressive(self.canvas, band["tiles"], self.denoiser)
            return
        if self.graphs[k] is None:
            # capture on first use; the band has just been quantised, so the warm-up run is the real run
            # of this call, then the same work is captured for replays.  Warm-up must not change the
            # canvas twice: snapshot the rows the band can touch, run, restore, capture, replay.
            snap = self.canvas.buf.clone()
            run_progressive(self.canvas, band["tiles"], self.denoiser)
            torch.cuda.current_stream().synchronize()
            self.canvas.buf.copy_(snap)
            g = torch.cuda.CUDAGraph()
            cur = torch.cuda.current_stream()
            with torch.cuda.graph(g, stream=torch.cuda.Stream(device=self.dp.device)):
                run_progressive(self.canvas, band["tiles"], self.denoiser)
            cur.synchronize()
            self.canvas.buf.copy_(snap)
            del snap
            self.graphs[k] = g
        self.graphs[k].replay()

    def run(self, host_in: torch.Tensor, host_out: torch.Tensor, stage: Optional[torch.Tensor] = None) -> torch.Tensor:
        """host_in pinned: bands are uploaded straight from it.  host_in pageable (what ComfyUI
        usually hands over): pass a pinned `stage` buffer of the same shape -- each band is
        memcpy'd into it by the host right before its upload is enqueued, so the host copy of
        band k+1 overlaps the GPU's work on band k."""
        main = torch.cuda.current_stream(self.dp.device)
        self.canvas.launches = self.canvas.algo_bytes = 0
        self.launches = 0
        self.s_in.wait_stream(main)
        self.s_out.wait_stream(main)

        # Rows y0:y1 of a multi-frame batch are B separate contiguous spans: one async copy per frame
        # (a single strided copy_ would make torch stage the whole slab through pageable memory).
        def upload(band):
            y0, y1 = band["in"]
            src = host_in
            if stage is not None and y1 > y0:
                for b in range(self.B):
                    stage[b, y0:y1].copy_(host_in[b, y0:y1])
                src = stage
            with torch.cuda.stream(self.s_in):
                if y1 > y0:
                    for b in range(self.B):
                        self.img[b, y0:y1].copy_(src[b, y0:y1], non_blocking=True)
                e = torch.cuda.Event()
                e.record()
            return e

        ups = [upload(b) for b in self.bands] if stage is None else []
        for k, band in enumerate(self.bands):
            main.wait_event(ups[k] if stage is None else upload(band))
            self._rows(None, band["in"][0], band["in"][1], self.img, None, True)
            self._band_compute(k)
            f0, f1 = band["fin"]
            self._rows(None, f0, f1, None, self.out, False)
            e = torch.cuda.Event()
            e.record(main)
            with torch.cuda.stream(self.s_out):
                self.s_out.wait_event(e)
                if f1 > f0:
                    for b in range(self.B):
                        host_out[b, f0:f1].copy_(self.out[b, f0:f1], non_blocking=True)
        main.wait_stream(self.s_out)
        main.wait_stream(self.s_in)
        return host_out


class _PinnedPool:
    """Pinned result buffers, reused once the caller has dropped them.  A fresh 400 MB pinned
    allocation costs the time of many pipelined jobs (page locking), and torch's
    host allocator does not hand a block back quickly enough when the previous result is still
    referenced.  A buffer is recycled only if nothing but the pool references it: no other Python
    reference to the tensor object (views hold one through `_base`) and no other owner of its storage
    (numpy arrays made with `.numpy()` and views own the storage without referencing the tensor).
    Bounded: `keep` buffers per shape, `shapes` most recently used shapes (the rest goes back to torch's host allocator)."""

    def __init__(self, keep: int = 3, shapes: int = 4):
        self.bufs: "LruCache[list]" = LruCache(shapes)
        self.keep = keep

    def get(self, shape, dtype=torch.float32) -> torch.Tensor:
        key = (tuple(shape), dtype)
        lst = self.bufs.get_or_build(key, list)
        for i in range(len(lst)):
            if buffer_is_unreferenced(lst[i]):
                # a consumer may have queued an asynchronous copy out of the buffer on some stream and dropped the
                # tensor right away: let everything in flight on the device finish before the buffer is rewritten
                if torch.cuda.is_available():
                    torch.cuda.synchronize()
                return lst[i]
        if len(lst) >= self.keep:
            lst.pop(0)                               # still referenced elsewhere: just forget it
        t = torch.empty(tuple(shape), dtype=dtype, pin_memory=True)
        lst.append(t)
        return t


def buffer_is_unreferenced(t: torch.Tensor) -> bool:
    """True when nothing but the caller's container references tensor `t` or its storage: no other Python reference
    to the tensor object (views hold one through `_base`) and no other owner of the storage (numpy arrays made with
    `.numpy()` and views own the storage without referencing the tensor).  The storage count comes from a private torch
    entry point; when a torch build lacks it the answer is always False -- buffers are then never recycled, only
    replaced (slower, never unsafe)."""
    import sys
    use_count = getattr(torch._C, "_storage_Use_Count", None)
    if use_count is None:
        return False
    # the container + getrefcount's own argument (+ this function's parameter); the tensor + the temporary wrapper
    return sys.getrefcount(t) <= 3 and use_count(t.untyped_storage()._cdata) <= 2


PINNED_RESULTS = _PinnedPool()
PINNED_STAGING = _PinnedPool(keep=1)      # upload staging for pageable inputs (never handed out)
MAX_BANDS = 12


def upscale_host(host_image: torch.Tensor, denoiser: Denoiser, tile_width: int, tile_height: int, padding: int,
                 mask_blur: int, force_uniform_tiles: bool = True, device: Optional[torch.device] = None,
                 stats: Optional[dict] = None, n_bands: Optional[int] = None) -> torch.Tensor:
    """HOST tensor [B,H,W,3] fp32 -> HOST tensor (pinned), same result as upscale_single.
    n_bands: pipeline depth; default one band per tile row, at most MAX_BANDS (shorter fill/drain
    of the two PCIe streams; the extra small launches hide under the copies)."""
    if host_image.is_cuda:
        raise ValueError("upscale_host takes a host tensor; use upscale_single for device tensors")
    check_batch(int(host_image.shape[0]))
    device = device or torch.device("cuda", torch.cuda.current_device())
    x = reference_f32(host_image).contiguous()
    B, H, W, _ = x.shape
    plan = get_plan(W, H, tile_width, tile_height, padding, mask_blur, force_uniform_tiles)
    with torch.cuda.device(device):
        dp = DevicePlan.get(plan, device)
        if n_bands is None:
            n_bands = min(len({t.y for t in plan.tiles}), MAX_BANDS)
        hp = HostPipeline.get(dp, B, denoiser, n_bands)
        out = PINNED_RESULTS.get(x.shape)
        stage = None if x.is_pinned() else PINNED_STAGING.get(x.shape)
        try:
            hp.run(x, out, stage)
            torch.cuda.current_stream(device).synchronize()
        finally:
            if not hp.graph_safe:
                hp.denoiser = None      # do not keep the caller's MODEL / VAE alive in the cache
    if stats is not None:
        stats["gpu_launches"] = stats.get("gpu_launches", 0) + hp.canvas.launches + hp.launches
        stats["algo_bytes"] = stats.get("algo_bytes", 0) + hp.canvas.algo_bytes
        stats["tiles"], stats["bands"] = len(plan.tiles), len(hp.bands)
    return out


# --------------------------------------------------------------------------------------
# releasing the caches (POST /distributed/clear_memory, worker_routes.py)
# --------------------------------------------------------------------------------------
_jobs_lock = threading.Lock()       # guards the two below; every release of the caches happens under it
_jobs_running = 0
_release_pending = False


@contextlib.contextmanager
def job_scope():
    """The extent of one node run (UltimateSDUpscaleDistributed, DistributedCollector).  A release asked for while jobs
    run is done by the last of them to leave, so no cached canvas or graph is dropped while a job may still use it."""
    global _jobs_running
    with _jobs_lock:
        _jobs_running += 1
    try:
        yield
    finally:
        with _jobs_lock:
            _jobs_running -= 1
            if _jobs_running == 0 and _release_pending:
                _release_locked()


def release_device_caches():
    """Drop this package's device caches: the DevicePlan, GraphedWaves and HostPipeline entries, the pinned result and
    staging pools, the collector's text pool and dist's jobs and buffers (dist.release_caches).  A pool drops only its
    own reference: a result the caller still holds stays alive.  While a job runs the release is left to the last job
    to finish."""
    global _release_pending
    with _jobs_lock:
        if _jobs_running:
            _release_pending = True
        else:
            _release_locked()


def _release_locked():
    global _release_pending
    from . import dist
    from .nodes import collector
    _release_pending = False
    devices = {dp.device for dp in DevicePlan._cache.values()} | \
        {gw.canvas.dp.device for gw in GraphedWaves._cache.values()} | {hp.dp.device for hp in HostPipeline._cache.values()}
    for dev in devices:
        torch.cuda.synchronize(dev)             # nothing still in flight reads what is dropped
    for cache in (GraphedWaves._cache, HostPipeline._cache, DevicePlan._cache, PINNED_RESULTS.bufs, PINNED_STAGING.bufs):
        cache.clear()
    collector._text_pool = None
    dist.release_caches()
