"""Host-side planner of the USDU tile path: geometry, resample tables, feather-template
classes, dependency waves, rank partitions and the kernel work lists.

The geometry, the table pool, the feather-mask specs, the tile descriptors, the dependency
waves and the job records of the crop and blend kernels are built by libusdu_b200.so
(csrc/usdu_plan.cpp, the planner section of include/usdu_b200.h), so that a host without
Python drives the same plan; this module holds a plan handle and builds the schedules on top
of those records: rank partitions and split levels.

Everything here is integer bookkeeping that the reference recomputes per tile with
full-canvas PIL images; here it is computed once per job (and cached per geometry):

* tile grid ............ upscale/tile_ops.py:14-32 (round_to_multiple, calculate_tiles)
* crop window .......... upscale/tile_ops.py:51-82 / :108-138 with
                         utils/usdu_utils.py:49-112 (get_crop_region, fix_crop_region,
                         expand_crop)
* progressive order .... upscale/modes/single_gpu.py:40-64 (tile k sees tiles < k)
* static partition ..... upscale/modes/static.py:226-311 (pull queue) -> a fixed plan
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import _native as nat
from .lru import LruCache


@dataclass(frozen=True)
class Tile:
    idx: int
    x: int          # grid origin
    y: int
    x1: int         # crop window on the canvas
    y1: int
    x2: int
    y2: int
    pw: int         # processing size
    ph: int
    bx1: int        # bbox of the inclusive mask rectangle, clipped (exclusive right/bottom)
    by1: int
    bx2: int
    by2: int

    @property
    def ew(self) -> int:
        return self.x2 - self.x1

    @property
    def eh(self) -> int:
        return self.y2 - self.y1

    @property
    def region(self) -> Tuple[int, int, int, int]:
        return (self.x1, self.y1, self.x2, self.y2)


# --------------------------------------------------------------------------------------
# plan
# --------------------------------------------------------------------------------------
@dataclass
class WorkList:
    """Device work list for one kernel launch (numpy, uploaded by the engine)."""
    items: np.ndarray                 # int32 [n, words]
    cover: Optional[np.ndarray]       # int32 [m, COVER_WORDS] (blend only)
    patch_w: int
    patch_h: int
    algo_bytes: int                   # algorithmic HBM bytes of the launch per frame
    n_launch: int = -1                # grid size when it differs from len(items) (chained fast jobs)
    block_rows: int = 0               # block height the work list was built for (passed in `flags`)
    block_cols: int = 0               # block width (generic kernels only)
    rows: Optional[Tuple[int, int]] = None   # blend with part=(i, n): canvas rows [y0, y1) of this share (whole block rows)
    path: int = 0                     # 0 generic work items, 1 fast job records, 2 tensor-core job records
    ks2: bool = False                 # tensor-core records: some axis of the launch needs two k-steps (USDU_FLAG_MMA_KS2)


@dataclass
class Plan:
    W: int
    H: int
    tile_width: int
    tile_height: int
    padding: int
    mask_blur: int
    uniform: bool
    tw: int = 0
    th: int = 0
    tiles: List[Tile] = field(default_factory=list)
    tile_desc: np.ndarray = None          # int32 [T, TILE_WORDS]
    tabs: np.ndarray = None               # int32 pool
    mask_specs: np.ndarray = None         # int32 [n_cls, MASK_WORDS]
    mask_pool_bytes: int = 0
    mask_class: List[int] = field(default_factory=list)
    neighbors: List[List[int]] = field(default_factory=list)   # overlapping windows, any order
    fast: bool = True                     # every table has packed rows -> register-window kernels
    mma: bool = True                      # ... and tensor-core fragments (<= 2 k-steps), windows start on 4-px columns
    _tab_off: Dict[Tuple[int, int], int] = field(default_factory=dict)        # pool offset of the (n_in, n_out) table
    _tab_packed: Dict[Tuple[int, int], int] = field(default_factory=dict)     # pool index of its packed row 0
    _tab_frag: Dict[Tuple[int, int], int] = field(default_factory=dict)       # pool index of its fragment section
    _tab_ks: Dict[Tuple[int, int], int] = field(default_factory=dict)         # k-steps
    _tab_taps: Dict[Tuple[int, int], int] = field(default_factory=dict)       # staged taps of the integer-pipe kernels
    _tab_job_taps: Dict[Tuple[int, int], int] = field(default_factory=dict)   # taps the job records carry
    _mask_off: List[int] = field(default_factory=list)                        # per tile: its feather template
    _mask_pitch: List[int] = field(default_factory=list)
    _native: Optional[nat.NativePlan] = field(default=None, repr=False, compare=False)

    # ---- construction ---------------------------------------------------------------
    @staticmethod
    def build(W: int, H: int, tile_width: int, tile_height: int, padding: int, mask_blur: int,
              uniform: bool) -> "Plan":
        """The library's plan of one job geometry (usdu_plan_create); ValueError for what it rejects (a tile size
        that rounds to zero, feather templates of 2 GiB or more)."""
        p = Plan(W, H, tile_width, tile_height, padding, mask_blur, uniform)
        h = p._native = nat.NativePlan(W, H, tile_width, tile_height, padding, mask_blur, uniform)
        p.tw, p.th = int(h.info[nat.PI_TW]), int(h.info[nat.PI_TH])
        geo = h.tiles()
        p.tiles = [Tile(i, x, y, x1, y1, x1 + ew, y1 + eh, pw, ph, x, y, bx2, by2)
                   for i, (x, y, x1, y1, ew, eh, pw, ph, bx2, by2, _, _) in enumerate(geo.tolist())]
        p.mask_class = geo[:, 10].tolist()
        p.tile_desc = h.tile_desc()
        p.tabs = h.tables()
        p.mask_specs = h.mask_specs()
        p.mask_pool_bytes = int(h.info[nat.PI_MASK_POOL_BYTES])
        p._mask_off = p.tile_desc[:, nat.T_MASK_OFF].tolist()
        p._mask_pitch = p.tile_desc[:, nat.T_MASK_PITCH].tolist()
        p.fast, p.mma = bool(h.info[nat.PI_FAST]), bool(h.info[nat.PI_MMA])
        for n_in, n_out, off, packed, frag, ks, taps, job_taps in h.table_index().tolist():
            key = (n_in, n_out)
            p._tab_off[key], p._tab_packed[key], p._tab_taps[key], p._tab_job_taps[key] = off, packed, taps, job_taps
            if frag >= 0:
                p._tab_frag[key], p._tab_ks[key] = frag, ks
        p.neighbors = h.neighbors()
        return p

    def opaque_core(self, t: Tile) -> Tuple[int, int, int, int]:
        """Window-relative box inside which the feather alpha is exactly 255 (descriptor words T_FULL_*): the rectangle
        shrunk by the ramp, except on sides where the rectangle touches the canvas border."""
        return tuple(self.tile_desc[t.idx, nat.T_FULL_X0:nat.T_FULL_Y1 + 1].tolist())

    def support(self, t: Tile) -> Tuple[int, int, int, int]:
        """Window-relative bbox outside which the feather alpha is exactly 0 (descriptor words T_SUP_*)."""
        return tuple(self.tile_desc[t.idx, nat.T_SUP_X0:nat.T_SUP_Y1 + 1].tolist())

    # ---- schedules -------------------------------------------------------------------
    def waves(self, order: Optional[Sequence[int]] = None) -> List[List[int]]:
        """Level schedule of an ordered tile list under progressive semantics (usdu_plan_waves): tile k must
        see the blends of every earlier tile whose window intersects its own.  Tiles of
        one wave have pairwise disjoint windows, so they can be cropped, denoised and
        blended together; running the waves in sequence reproduces the sequential loop
        of upscale/modes/single_gpu.py:40-64 exactly."""
        order = list(range(len(self.tiles))) if order is None else [int(t) for t in order]
        level = self._native.waves(order).tolist()
        out: List[List[int]] = [[] for _ in range(max(level) + 1 if level else 0)]
        for t, lv in zip(order, level):
            out[lv].append(t)
        return out

    def conflict_free(self, assignment: Sequence[Sequence[int]]) -> bool:
        for tiles in assignment:
            s = set(tiles)
            for t in tiles:
                if any(n in s for n in self.neighbors[t]):
                    return False
        return True

    def partition(self, world: int) -> List[List[int]]:
        """Static tile -> rank plan replacing the reference's pull queue
        (upscale/modes/static.py:226-311).  Tries skewed colourings rank = (col + k*row)
        mod world that leave no rank with two window-overlapping tiles (then every crop
        comes from the original canvas and all ranks run fully in parallel); falls back
        to round-robin, which the engine executes as per-rank waves."""
        T = len(self.tiles)
        if world <= 1:
            return [list(range(T))]
        cols = math.ceil(self.W / self.tw)
        best = None
        for k in range(1, world):
            asg = [[] for _ in range(world)]
            for t in self.tiles:
                asg[((t.idx % cols) + k * (t.idx // cols)) % world].append(t.idx)
            if self.conflict_free(asg):
                spread = max(len(a) for a in asg) - min(len(a) for a in asg)
                if best is None or spread < best[0]:
                    best = (spread, asg)
        if best is not None:
            return best[1]
        asg = [[] for _ in range(world)]
        for t in self.tiles:
            asg[t.idx % world].append(t.idx)
        return asg

    # ---- kernel work lists (built by the library) ------------------------------------------
    def slot_offsets(self, tile_ids: Sequence[int], B: int) -> Tuple[np.ndarray, int]:
        """Element offsets of each tile's [B, ph, pw, 3] block in a packed buffer."""
        offs = np.zeros(len(tile_ids), dtype=np.int64)
        cur = 0
        for i, tid in enumerate(tile_ids):
            t = self.tiles[tid]
            offs[i] = cur
            cur += B * t.ph * t.pw * 3
        return offs, cur

    def kernel_path(self, use_fast=None) -> int:
        """Which kernels a work list is built for: 0 generic (any scale), 1 integer-pipe fast kernels, 2 tensor-core
        kernels.  None = the best this plan supports; True / False keep their round-1 meaning (1 / 0)."""
        path = 2 if use_fast is None else int(use_fast)
        if path >= 2 and not self.mma:
            path = 1
        if path >= 1 and not self.fast:
            path = 0
        return path

    @staticmethod
    def _request(use_fast) -> int:
        """Kernel family asked for: None = the best the plan supports; True / False keep their round-1 meaning (1 / 0)."""
        return 2 if use_fast is None else int(use_fast)

    @staticmethod
    def _launch_model() -> Tuple[int, int]:
        """(SMs of the current device or 0, forced tensor-core block height or 0): the block-height model's inputs."""
        return nat.sm_count(), int(os.environ.get("USDU_MMA_BH") or 0)   # experiments: force the tensor-core block height

    @staticmethod
    def _worklist(r: dict, blend: bool) -> WorkList:
        info = r["info"]
        path = int(info[nat.WL_PATH])
        return WorkList(r["items"], r["cover"] if blend and path == 0 else None, int(info[nat.WL_PATCH_W]),
                        int(info[nat.WL_PATCH_H]), int(info[nat.WL_ALGO_BYTES]), n_launch=int(info[nat.WL_N_LAUNCH]),
                        block_rows=int(info[nat.WL_BLOCK_ROWS]), block_cols=int(info[nat.WL_BLOCK_COLS]),
                        rows=(int(info[nat.WL_ROW0]), int(info[nat.WL_ROW1])) if info[nat.WL_ROW0] >= 0 else None,
                        path=path, ks2=bool(info[nat.WL_KS2]))

    def crop_worklist(self, tile_ids: Sequence[int], B: int, use_fast: Optional[bool] = None) -> Tuple[WorkList, np.ndarray, int]:
        """One crop launch over `tile_ids` (usdu_plan_crop_worklist) -> (work list, element offset of each tile's
        [B, ph, pw, 3] output in the packed buffer, total elements)."""
        r = self._native.crop_worklist(tile_ids, B, self._request(use_fast), *self._launch_model())
        return self._worklist(r, False), r["slots"], int(r["info"][nat.WL_TOTAL])

    def crop_split(self, wl: WorkList, prev_ids: Sequence[int]) -> np.ndarray:
        """late[j]: job j of a tensor-core / fast crop work list stages canvas pixels that some tile of `prev_ids` (the
        previous dependency wave) changes -- its staged rectangle meets that tile's feather support.  The other jobs read
        pixels whose VALUES the previous wave's blend does not touch (a blend rewrites whole blocks, but only pixels under
        a non-zero alpha change), so they may run before or beside it (single_gpu.py:40-64 orders only what overlaps)."""
        J = wl.items.reshape(-1, nat.JOB_WORDS).astype(np.int64)
        x0, y0 = J[:, nat.J_SRC_A], J[:, nat.J_SRC_B]
        x1, y1 = x0 + J[:, nat.J_LEAD] + J[:, nat.J_COLS], y0 + J[:, nat.J_ROWS]   # (integer-pipe records start `lead` pixels early)
        late = np.zeros(J.shape[0], dtype=bool)
        for tid in prev_ids:
            t = self.tiles[tid]
            sx0, sy0, sx1, sy1 = self.support(t)
            if sx1 > sx0 and sy1 > sy0:
                late |= (x0 < t.x1 + sx1) & (t.x1 + sx0 < x1) & (y0 < t.y1 + sy1) & (t.y1 + sy0 < y1)
        return late

    @staticmethod
    def sub_worklist(wl: WorkList, mask: np.ndarray) -> WorkList:
        """The jobs of an unchained job list (crop) selected by `mask`, same launch geometry."""
        import dataclasses
        J = wl.items.reshape(-1, nat.JOB_WORDS)
        keep = int(mask.sum())
        return dataclasses.replace(wl, items=np.ascontiguousarray(J[mask]), algo_bytes=int(wl.algo_bytes * keep / max(J.shape[0], 1)))

    def split_level(self, wave: Sequence[int], offs: np.ndarray, prev: Optional[Sequence[int]], B: int, path: int = 2):
        """Work lists of one dependency wave split by dependency on ONE crop geometry (split_lists sizes the two parts
        by role instead; this form is what tests/planner_model.py restates).
        -> (crop, offs, total, late mask or None, blend).
        crop jobs: `late` ones read pixels the previous wave `prev` changes, the rest may run beside the previous wave's
        sampler and blend."""
        cr, coffs, ctotal = self.crop_worklist(wave, B, path)
        late = self.crop_split(cr, prev) if (prev and cr.path >= 1) else None
        return cr, coffs, ctotal, late, self.blend_worklist(wave, offs, 4, path, B)

    def split_lists(self, wave: Sequence[int], offs: np.ndarray, prev: Optional[Sequence[int]], B: int, path: int = 2):
        """Work lists of one dependency wave as engine.run_split launches it (usdu_plan_split_worklists), each sized for
        its role: -> (chain crop, side crop or None, element offsets of the tiles' crop outputs, total elements, blend).
        The side crop holds the jobs that read no pixel the previous wave `prev` changes and runs beside prev's sampler
        and blend; the chain crop, in short blocks, holds the rest (every job of the first wave, or of a wave whose jobs
        all do).  Together they cover every crop output once.  path >= 1 (job records)."""
        late, early, blend = self._native.split_worklists(wave, offs, prev or [], B, path, self._launch_model()[0])
        late_wl, early_wl = self._worklist(late, False), self._worklist(early, False)
        chain, side = late_wl, early_wl
        if not len(late_wl.items):
            chain, side = early_wl, None
        elif not len(early_wl.items):
            side = None
        return chain, side, late["slots"], int(late["info"][nat.WL_TOTAL]), self._worklist(blend, True)

    CROP_BOX_ROWS = (0, 40, 48)           # rows of a crop's bulk-tensor box per kernel path (usdu_fast.cu / usdu_mma.cu kBoxR)

    def wave_rows(self, levels: Sequence[Tuple[Sequence[WorkList], WorkList]]):
        """Per dependency wave, the canvas rows its launches can touch.  levels[k] = (the crop work lists wave k launches,
        its blend work list), job records (path >= 1) -> (touch, write), bool [len(levels), H].  touch = rows a crop's TMA
        box can load (the whole box from its first staged row, plus the next row for the integer-pipe staging's 16-byte
        over-read) or a blend block loads; write = rows of whole blend blocks, which a blend stores back even where the
        mask leaves them unchanged."""
        touch = np.zeros((len(levels), self.H), dtype=bool)
        write = np.zeros((len(levels), self.H), dtype=bool)
        for k, (crops, bl) in enumerate(levels):
            if bl.path < 1 or any(cr.path < 1 for cr in crops):
                raise ValueError("wave_rows needs job-record work lists (path >= 1)")
            for cr in crops:
                J = cr.items.reshape(-1, nat.JOB_WORDS)
                box, slack = self.CROP_BOX_ROWS[cr.path], int(cr.path == 1)
                for y0, n in zip(J[:, nat.J_SRC_B].tolist(), J[:, nat.J_ROWS].tolist()):
                    touch[k, max(y0, 0):min(y0 + max(n, box) + slack, self.H)] = True
            J = bl.items.reshape(-1, nat.JOB_WORDS)
            for y0, n in zip(J[:, nat.J_DST_Y].tolist(), J[:, nat.J_ROWS_OUT].tolist()):
                write[k, max(y0, 0):min(y0 + max(n, bl.block_rows), self.H)] = True
            touch[k] |= write[k]
        return touch, write

    def stream_bands(self, order: Optional[Sequence[int]], B: int, n_bands: int, path_crop: int = 2, path_blend: int = 2,
                     levels: Optional[Sequence[Tuple[Sequence[WorkList], WorkList]]] = None):
        """Row bands of the canvas quantise and dequantise passes when they run beside the level waves of `order`
        (engine.run_split).  -> (quantise, dequantise), lists of (y0, y1, wave): each quantise band [y0, y1) is tagged
        with the FIRST wave that touches one of its rows (it must be complete before that wave's crops start), each
        dequantise band with the LAST wave that writes one of its rows (it may start once that wave's blend is done).
        Rows are those of every frame; each list covers [0, H) once, top to bottom.  The first quantise band is exactly
        the rows the first wave touches (from row 0) and the last dequantise band the rows from the last wave's first
        written row down; the rest of each pass is cut into n_bands - 1 bands of equal height.
        levels: the work lists the waves launch (see wave_rows); None = one crop and one blend list per wave of `order`
        as crop_worklist / blend_worklist build them."""
        if levels is None:
            levels = []
            for wave in self.waves(order):
                cr, offs, _ = self.crop_worklist(wave, B, path_crop)
                levels.append(([cr], self.blend_worklist(wave, offs, 4, path_blend, B)))
        touch, write = self.wave_rows(levels)
        n_waves = len(levels)
        H, n_bands = self.H, max(1, int(n_bands))
        lo = np.arange(n_waves)[:, None]
        first = np.where(touch, lo, n_waves).min(0)              # per row: first wave touching it
        last = np.where(write, lo, -1).max(0)                    # per row: last wave writing it
        if (last < 0).any():
            raise ValueError("stream_bands: some canvas row is written by no wave")

        def cut(y0, y1, n):
            n = max(1, min(n, y1 - y0))
            return [(y0 + (y1 - y0) * i // n, y0 + (y1 - y0) * (i + 1) // n) for i in range(n)]

        q_head = int(np.nonzero(touch[0])[0].max()) + 1
        q = [(0, q_head)] + (cut(q_head, H, n_bands - 1) if q_head < H and n_bands > 1 else [(q_head, H)] if q_head < H else [])
        d_tail = int(np.nonzero(write[-1])[0].min())
        d = (cut(0, d_tail, n_bands - 1) if d_tail > 0 and n_bands > 1 else [(0, d_tail)] if d_tail > 0 else []) + [(d_tail, H)]
        return ([(y0, y1, int(first[y0:y1].min())) for y0, y1 in q],
                [(y0, y1, int(last[y0:y1].max())) for y0, y1 in d])

    def blend_worklist(self, tile_ids: Sequence[int], offs: np.ndarray, src_bytes_per_elem: int = 4,
                       use_fast: Optional[bool] = None, B: int = 1, part: Optional[Tuple[int, int]] = None) -> WorkList:
        """Canvas blocks touched by the given tiles (usdu_plan_blend_worklist); each block lists its tiles in the
        given order (the order of `tile_ids` IS the blend order).  part = (i, n): only the blocks of the i-th of n
        horizontal slabs of the canvas (whole block rows, WorkList.rows = the slab's canvas rows; the n slabs tile
        the canvas) -- every block is owned by exactly one CTA, so n participants given the same tile list
        composite disjoint slabs (dist.upscale_static: each rank finishes its own slab of the final canvas)."""
        r = self._native.blend_worklist(tile_ids, offs, src_bytes_per_elem, B, self._request(use_fast), part, *self._launch_model())
        return self._worklist(r, True)


_PLAN_CACHE: LruCache[Plan] = LruCache(16)


def get_plan(W: int, H: int, tile_width: int, tile_height: int, padding: int, mask_blur: int, uniform: bool) -> Plan:
    key = (W, H, tile_width, tile_height, padding, mask_blur, bool(uniform))
    return _PLAN_CACHE.get_or_build(key, lambda: Plan.build(*key))

