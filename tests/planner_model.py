"""Test-only reference model of the host planner: the numpy builders the package used before the planner moved into
libusdu_b200.so (csrc/usdu_plan.cpp), kept unchanged so that tests/test_native_planner.py can check the library's
geometry, tables, descriptors, waves and work lists against them byte for byte.

Original module docstring:
Host-side planner of the USDU tile path: geometry, resample tables, feather-template
classes, dependency waves, rank partitions and the kernel work lists.

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

from __graft_entry__ import load_package

load_package()
from comfyui_distributed_b200 import _native as nat  # noqa: E402
from comfyui_distributed_b200.lru import LruCache  # noqa: E402


# --------------------------------------------------------------------------------------
# geometry
# --------------------------------------------------------------------------------------
def round_to_multiple(value: int, multiple: int = 8) -> int:
    # Python's round(): ties go to the even multiple, exactly as upscale/tile_ops.py:14-16
    return round(value / multiple) * multiple


def tile_origins(W: int, H: int, tw: int, th: int) -> List[Tuple[int, int]]:
    cols, rows = math.ceil(W / tw), math.ceil(H / th)
    return [(c * tw, r * th) for r in range(rows) for c in range(cols)]


def _grow(lo: int, hi: int, limit: int, target: int) -> Tuple[int, int]:
    """One axis of expand_crop (utils/usdu_utils.py:88-110): right/bottom by half the
    deficit, then left/top by what is still missing, then right/bottom again."""
    hi = min(hi + (target - (hi - lo)) // 2, limit)
    lo = max(lo - (target - (hi - lo)), 0)
    hi = min(hi + (target - (hi - lo)), limit)
    return lo, hi


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


def make_tile(idx: int, W: int, H: int, x: int, y: int, tw: int, th: int, padding: int, uniform: bool) -> Tile:
    # PIL draws the rectangle [x, y, x+tw, y+th] INCLUSIVE of its far corner; getbbox is
    # exclusive, hence the +1 (upscale/tile_ops.py:51-54, utils/usdu_utils.py:52).
    bx1, by1 = x, y
    bx2, by2 = min(x + tw + 1, W), min(y + th + 1, H)
    x1, y1 = max(bx1 - padding, 0), max(by1 - padding, 0)
    x2, y2 = min(bx2 + padding, W), min(by2 + padding, H)
    if x2 < W:
        x2 -= 1
    if y2 < H:
        y2 -= 1
    if uniform:
        pw, ph = round_to_multiple(tw + padding), round_to_multiple(th + padding)
        cw, ch = x2 - x1, y2 - y1
        crop_ratio = cw / ch if ch else 1.0
        proc_ratio = pw / ph if ph else 1.0
        if crop_ratio > proc_ratio:
            want_w, want_h = cw, (round(cw / proc_ratio) if proc_ratio else ch)
        else:
            want_w, want_h = round(ch * proc_ratio), ch
    else:
        pw = want_w = max(8, math.ceil((x2 - x1) / 8) * 8)
        ph = want_h = max(8, math.ceil((y2 - y1) / 8) * 8)
    x1, x2 = _grow(x1, x2, W, want_w)
    y1, y2 = _grow(y1, y2, H, want_h)
    return Tile(idx, x, y, x1, y1, x2, y2, pw, ph, bx1, by1, bx2, by2)


def _overlap(a: Tuple[int, int, int, int], b: Tuple[int, int, int, int]) -> bool:
    return a[0] < b[2] and b[0] < a[2] and a[1] < b[3] and b[1] < a[3]


# --------------------------------------------------------------------------------------
# tensor-core fragments of a resample table (csrc/usdu_mma.cu)
# --------------------------------------------------------------------------------------
MMA_M = 16                 # outputs per M-tile (mma.sync.m16n8k32)
MMA_K = 32                 # inputs per k-step
MMA_MAX_KSTEPS = 2


def build_mma_frags(tab: np.ndarray) -> Optional[np.ndarray]:
    """A resampling axis as a banded matrix product on the tensor cores: out[o] = sum_k A[o][k] * in[k0 + k] with the
    22-bit fixed-point coefficients of Pillow (tab = header + bounds + kk of usdu_build_resample_table) split into three
    8-bit limbs, coef = l2 * 65536 + l1 * 256 + l0 (l0, l1 unsigned, l2 signed), one u8 x u8 / s8 x u8 IMMA each with
    exact s32 accumulation.  Outputs are grouped in M-tiles of 16 (aligned in OUTPUT index space); M-tile mt reads the
    inputs k0[mt] .. k0[mt] + 32 * ksteps (k0 a multiple of 4: the kernels read them with 32-bit shared-memory loads).
    -> int32 words {n_mtiles, ksteps, 0, 0} then per M-tile {k0, 0, 0, 0, fragments}, fragments = for (kstep, limb)
    32 lanes x 4 registers in the A-operand layout of mma.m16n8k32 (lane = 4 g + t: a0 = A[g][4t..4t+3],
    a1 = A[g+8][4t..], a2 = A[g][16+4t..], a3 = A[g+8][16+4t..]), or None when an M-tile needs more than
    MMA_MAX_KSTEPS k-steps (extreme down-scales: those plans keep the integer-pipe kernels)."""
    n_in, n_out, ksize = int(tab[0]), int(tab[1]), int(tab[2])
    H = nat.TAB_HEADER
    bounds = tab[H:H + 2 * n_out].reshape(n_out, 2).astype(np.int64)
    kk = tab[H + 2 * n_out:H + 2 * n_out + n_out * ksize].reshape(n_out, ksize).astype(np.int64)
    first, cnt = bounds[:, 0], bounds[:, 1]
    n_mt = (n_out + MMA_M - 1) // MMA_M
    o_lo = np.arange(n_mt) * MMA_M
    o_hi = np.minimum(o_lo + MMA_M, n_out)
    k0 = first[o_lo] & ~3
    end = np.array([int((first[a:b] + cnt[a:b]).max()) for a, b in zip(o_lo, o_hi)])
    ksteps = int(max(1, ((end - k0 + MMA_K - 1) // MMA_K).max()))
    if ksteps > MMA_MAX_KSTEPS:
        return None
    K = MMA_K * ksteps
    A = np.zeros((n_mt * MMA_M, K), dtype=np.int64)              # row = output (padded), col = input - k0[mt]
    o = np.arange(n_out)
    for t in range(ksize):
        col = first + t - k0[o // MMA_M]
        ok = t < cnt
        A[o[ok], col[ok]] = kk[ok, t]
    if np.abs(A).max() >= 1 << 23:
        return None
    limbs = np.stack([A & 255, (A >> 8) & 255, (A >> 16) & 255], 0).astype(np.uint8)       # two's complement: l2 is the s8 limb
    L = limbs.reshape(3, n_mt, MMA_M, ksteps, MMA_K)              # [limb, mt, m, ks, k]
    g, t = np.arange(32) // 4, np.arange(32) % 4
    regs = []
    for (dm, dk) in ((0, 0), (8, 0), (0, 16), (8, 16)):           # a0 .. a3
        kidx = (4 * t + dk)[:, None] + np.arange(4)[None, :]     # [lane, byte]
        sel = L[:, :, (g + dm)[:, None], :, kidx]                 # advanced indexing -> [lane, byte, limb, mt, ks]
        regs.append(sel)
    R = np.stack(regs, 0)                                         # [reg, lane, byte, limb, mt, ks]
    R = np.transpose(R, (4, 5, 3, 1, 0, 2))                       # [mt, ks, limb, lane, reg, byte]
    words = np.ascontiguousarray(R).view(np.uint32).reshape(n_mt, -1).view(np.int32)          # [mt, ksteps * 3 * 128]
    # per M-tile: {k0, 0, 0, 0} then its fragments, so that a kernel that knows mt and ksteps (job record) addresses both
    # without first loading anything from the section (no dependent load before the fragment loads)
    per_mt = np.concatenate([np.stack([k0, np.zeros_like(k0), np.zeros_like(k0), np.zeros_like(k0)], 1).astype(np.int32), words], 1)
    head = np.array([n_mt, ksteps, 0, 0], np.int32)
    return np.ascontiguousarray(np.concatenate([head, per_mt.reshape(-1)]))


def mma_frag_k0(frags: np.ndarray) -> np.ndarray:
    """K-window starts per M-tile of a fragment section."""
    n_mt, ks = int(frags[0]), int(frags[1])
    return frags[4:].reshape(n_mt, 4 + ks * 384)[:, 0].astype(np.int64)


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
    _tab_frag: Dict[Tuple[int, int], int] = field(default_factory=dict)       # pool index of the fragment section
    _tab_k0: Dict[Tuple[int, int], np.ndarray] = field(default_factory=dict)  # K-window start per M-tile
    _tab_ks: Dict[Tuple[int, int], int] = field(default_factory=dict)         # k-steps
    _tab_end: Dict[Tuple[int, int], np.ndarray] = field(default_factory=dict) # first + count per output
    _tab_off: Dict[Tuple[int, int], int] = field(default_factory=dict)
    _tab_span: Dict[Tuple[int, int], np.ndarray] = field(default_factory=dict)
    _tab_packed: Dict[Tuple[int, int], int] = field(default_factory=dict)
    _tab_first: Dict[Tuple[int, int], np.ndarray] = field(default_factory=dict)
    _tab_taps: Dict[Tuple[int, int], int] = field(default_factory=dict)
    _tab_job_taps: Dict[Tuple[int, int], int] = field(default_factory=dict)
    _gblock: Optional[Tuple[int, int]] = None

    # ---- construction ---------------------------------------------------------------
    @staticmethod
    def build(W: int, H: int, tile_width: int, tile_height: int, padding: int, mask_blur: int,
              uniform: bool) -> "Plan":
        p = Plan(W, H, tile_width, tile_height, padding, mask_blur, uniform)
        p.tw, p.th = round_to_multiple(tile_width), round_to_multiple(tile_height)
        if p.tw <= 0 or p.th <= 0:
            raise ValueError(f"tile size rounds to zero: {tile_width}x{tile_height}")
        p.tiles = [make_tile(i, W, H, x, y, p.tw, p.th, padding, uniform)
                   for i, (x, y) in enumerate(tile_origins(W, H, p.tw, p.th))]
        p._build_tables()
        if any(t.x1 % 4 for t in p.tiles) or not p.fast:
            p.mma = False                  # the tensor-core kernels stage 4-pixel chunks at 4-pixel canvas columns
        p._build_masks()
        p._build_descriptors()
        p._build_neighbors()
        return p

    def _table(self, n_in: int, n_out: int) -> int:
        key = (n_in, n_out)
        if key not in self._tab_off:
            # an axis that keeps its size gets a one-tap identity table (Pillow skips the pass)
            tab = nat.build_identity_table(n_in) if n_in == n_out else nat.build_resample_table(n_in, n_out)
            if tab[4] == 0:
                self.fast = False
            off = 0 if self.tabs is None else int(self.tabs.shape[0])
            self.tabs = tab if self.tabs is None else np.concatenate([self.tabs, tab])
            self._tab_off[key] = off
            self._tab_packed[key] = off + int(tab[4])          # pool index of packed row 0 (fast kernels)
            taps = int(tab[6]) - 1 if tab[4] else int(tab[3])  # 7 or 15 staged taps per output on the fast path
            self._tab_taps[key] = taps
            # what the job records carry: the real maximum when it is below the 7-slot row (an up-scaling
            # LANCZOS axis uses exactly 6), so the kernels can skip the always-zero last slot
            self._tab_job_taps[key] = min(taps, max(int(tab[3]), 1)) if taps <= nat.FAST_TAPS else taps
            b = tab[nat.TAB_HEADER:nat.TAB_HEADER + 2 * n_out].reshape(n_out, 2)
            frags = build_mma_frags(tab) if self.mma else None
            if frags is None:
                self.mma = False
            else:
                foff = int(self.tabs.shape[0])                     # tables end on a multiple of 4 int32
                assert foff % 4 == 0
                self.tabs = np.concatenate([self.tabs, frags])
                pad = (-int(self.tabs.shape[0])) % 4
                if pad:
                    self.tabs = np.concatenate([self.tabs, np.zeros(pad, np.int32)])
                n_mt = int(frags[0])
                self._tab_frag[key], self._tab_ks[key] = foff, int(frags[1])
                self._tab_k0[key] = mma_frag_k0(frags)
                self._tab_end[key] = (b[:, 0] + b[:, 1]).astype(np.int64)
            self._tab_first[key] = b[:, 0].astype(np.int64)
            self._tab_span[key] = np.stack([b[:, 0], b[:, 0] + np.maximum(b[:, 1], taps)], 1)   # [lo, hi) per output
        return self._tab_off[key]

    def _build_tables(self):
        for t in self.tiles:
            self._table(t.ew, t.pw), self._table(t.eh, t.ph)
            self._table(t.pw, t.ew), self._table(t.ph, t.eh)

    def _ramp(self) -> int:
        """Pixels beyond the rectangle that the blurred mask can be non-zero (3 box
        passes of half-width rad+1 each)."""
        if self.mask_blur <= 0:
            return 0
        rad, _, _ = nat.box_blur_params(self.mask_blur)
        return 3 * (rad + 1)

    def _build_masks(self):
        ext = self._ramp()
        classes: Dict[tuple, int] = {}
        specs = []
        off = 0
        self.mask_class = []
        self._mask_off, self._mask_pitch = [], []
        for t in self.tiles:
            kh = (t.bx1 - t.x1, t.bx2 - t.x1, t.ew, min(t.x1, ext), min(self.W - t.x2, ext))
            kv = (t.by1 - t.y1, t.by2 - t.y1, t.eh, min(t.y1, ext), min(self.H - t.y2, ext))
            key = (kh, kv)
            if key not in classes:
                classes[key] = len(specs)
                pitch = (t.ew + 15) // 16 * 16
                specs.append([self.W, self.H, t.bx1, t.by1, t.bx2, t.by2, t.x1, t.y1, t.x2, t.y2,
                              self.mask_blur, off, pitch, 0, 0, 0])
                off += pitch * t.eh
                off = (off + 255) // 256 * 256
            c = classes[key]
            self.mask_class.append(c)
            self._mask_off.append(specs[c][11])
            self._mask_pitch.append(specs[c][12])
        self.mask_specs = np.asarray(specs, dtype=np.int32)
        self.mask_pool_bytes = max(off, 256)
        if self.mask_pool_bytes >= 2 ** 31:
            raise ValueError("feather templates exceed 2 GiB")

    def opaque_core(self, t: Tile) -> Tuple[int, int, int, int]:
        """Window-relative box inside which the feather alpha is exactly 255: the rectangle
        shrunk by the ramp, except on sides where the rectangle touches the canvas border
        (edge replication keeps the mask at 255 there)."""
        ext = self._ramp()
        fx0 = t.bx1 if t.bx1 == 0 else t.bx1 + ext
        fy0 = t.by1 if t.by1 == 0 else t.by1 + ext
        fx1 = t.bx2 if t.bx2 == self.W else t.bx2 - ext
        fy1 = t.by2 if t.by2 == self.H else t.by2 - ext
        fx0, fy0 = max(fx0, t.x1), max(fy0, t.y1)
        fx1, fy1 = min(fx1, t.x2), min(fy1, t.y2)
        if fx1 <= fx0 or fy1 <= fy0:
            return (0, 0, 0, 0)
        return (fx0 - t.x1, fy0 - t.y1, fx1 - t.x1, fy1 - t.y1)

    def support(self, t: Tile) -> Tuple[int, int, int, int]:
        """Window-relative bbox outside which the feather alpha is exactly 0."""
        ext = self._ramp()
        return (max(t.bx1 - ext, t.x1) - t.x1, max(t.by1 - ext, t.y1) - t.y1,
                min(t.bx2 + ext, t.x2) - t.x1, min(t.by2 + ext, t.y2) - t.y1)

    def _build_descriptors(self):
        d = np.zeros((len(self.tiles), nat.TILE_WORDS), dtype=np.int32)
        for t in self.tiles:
            r = d[t.idx]
            r[nat.T_X1], r[nat.T_Y1], r[nat.T_EW], r[nat.T_EH] = t.x1, t.y1, t.ew, t.eh
            r[nat.T_PW], r[nat.T_PH] = t.pw, t.ph
            r[nat.T_MASK_OFF], r[nat.T_MASK_PITCH] = self._mask_off[t.idx], self._mask_pitch[t.idx]
            r[nat.T_TAB_CROP_H], r[nat.T_TAB_CROP_V] = self._table(t.ew, t.pw), self._table(t.eh, t.ph)
            r[nat.T_TAB_BLEND_H], r[nat.T_TAB_BLEND_V] = self._table(t.pw, t.ew), self._table(t.ph, t.eh)
            r[nat.T_SUP_X0:nat.T_SUP_Y1 + 1] = self.support(t)
            r[nat.T_FULL_X0:nat.T_FULL_Y1 + 1] = self.opaque_core(t)
        self.tile_desc = d

    def _build_neighbors(self):
        """Tiles whose crop windows intersect (grid-bucketed, O(T * neighbours))."""
        T = len(self.tiles)
        self.neighbors = [[] for _ in range(T)]
        if T <= 1:
            return
        cell = max(max(t.ew for t in self.tiles), max(t.eh for t in self.tiles))
        buckets: Dict[Tuple[int, int], List[int]] = {}
        for t in self.tiles:
            for gx in range(t.x1 // cell, (t.x2 - 1) // cell + 1):
                for gy in range(t.y1 // cell, (t.y2 - 1) // cell + 1):
                    buckets.setdefault((gx, gy), []).append(t.idx)
        seen = set()
        for ids in buckets.values():
            for a in range(len(ids)):
                for b in range(a + 1, len(ids)):
                    i, j = ids[a], ids[b]
                    if (i, j) in seen:
                        continue
                    seen.add((i, j))
                    if _overlap(self.tiles[i].region, self.tiles[j].region):
                        self.neighbors[i].append(j)
                        self.neighbors[j].append(i)

    # ---- schedules -------------------------------------------------------------------
    def waves(self, order: Optional[Sequence[int]] = None) -> List[List[int]]:
        """Level schedule of an ordered tile list under progressive semantics: tile k must
        see the blends of every earlier tile whose window intersects its own.  Tiles of
        one wave have pairwise disjoint windows, so they can be cropped, denoised and
        blended together; running the waves in sequence reproduces the sequential loop
        of upscale/modes/single_gpu.py:40-64 exactly."""
        order = list(range(len(self.tiles))) if order is None else list(order)
        pos = {t: i for i, t in enumerate(order)}
        level: Dict[int, int] = {}
        out: List[List[int]] = []
        for t in order:
            lv = 0
            for n in self.neighbors[t]:
                if n in pos and pos[n] < pos[t]:
                    lv = max(lv, level[n] + 1)
            level[t] = lv
            while len(out) <= lv:
                out.append([])
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

    # ---- kernel work lists -----------------------------------------------------------
    def slot_offsets(self, tile_ids: Sequence[int], B: int) -> Tuple[np.ndarray, int]:
        """Element offsets of each tile's [B, ph, pw, 3] block in a packed buffer."""
        offs = np.zeros(len(tile_ids), dtype=np.int64)
        cur = 0
        for i, tid in enumerate(tile_ids):
            t = self.tiles[tid]
            offs[i] = cur
            cur += B * t.ph * t.pw * 3
        return offs, cur

    def _span_max(self, n_in: int, n_out: int, block: int, aligned: bool) -> int:
        """Largest input extent read by `block` consecutive outputs of an axis."""
        sp = self._tab_span[(n_in, n_out)]
        starts = np.arange(0, n_out, block) if aligned else np.arange(0, n_out)
        ends = np.minimum(starts + block, n_out) - 1
        return int((sp[ends, 1] - sp[starts, 0]).max())

    CTAS_PER_SM = 4            # resident CTAs of the fast kernels per SM
    DEFAULT_SMS = 132          # H100 SXM: the block shapes of plans made where no device can be queried

    @classmethod
    def resident_slots(cls) -> int:
        """Resident CTAs of the fast kernels on the current device (nat.sm_count(), the SM count the launchers see)."""
        return (nat.sm_count() or cls.DEFAULT_SMS) * cls.CTAS_PER_SM

    def block_shape(self, use_fast: bool, extents: Optional[Sequence[Tuple[int, int]]] = None, frames: int = 1,
                    mma: bool = False) -> Tuple[int, int]:
        """Block edge of a launch.  `extents` = (width, height) in pixels each tile covers in
        the launch's block space.  The block height is chosen by a simple wave model:
        cost(bh) = ceil(#CTAs / resident slots) * (bh + halo/fixed rows) -- short blocks give
        small (latency bound) launches more CTAs, and large launches avoid a nearly empty
        last wave."""
        if not use_fast:
            return self._generic_block
        bw = nat.FAST_BLOCK_W
        if not extents:
            return bw, nat.FAST_BLOCK_H
        best = None
        slots = self.resident_slots()
        forced = os.environ.get("USDU_MMA_BH") if mma else None            # experiments: force the tensor-core block height
        for bh in (((int(forced),) if forced else (16, 32)) if mma else (8, 12, 16, 20, 24, 28, 32)):   # M-tiles are 16 output rows
            n = sum(((w + bw - 1) // bw + 1) * ((h + bh - 1) // bh + 1) for w, h in extents) * frames   # +1: unaligned windows
            cost = math.ceil(n / max(slots, 1)) * (bh + 12)
            if best is None or cost < best[0] or (cost == best[0] and bh > best[1]):
                best = (cost, bh)
        return bw, best[1]

    @property
    def _generic_block(self) -> Tuple[int, int]:
        """Block of the generic kernels: 64 x 32 unless an extreme scale (a canvas much smaller
        than a tile) makes the input patch of such a block exceed shared memory; then halve."""
        if self._gblock is None:
            bw, bh = nat.BLOCK_W, nat.BLOCK_H
            while True:
                pw_ = max([self._span_max(a, b, bw, False) for (a, b) in self._tab_span] or [bw])
                ph_ = max([self._span_max(a, b, bh, False) for (a, b) in self._tab_span] or [bh])
                smem = nat.BLOCK_H * nat.BLOCK_W * 3 + ph_ * nat.BLOCK_W * 3 + ph_ * ((pw_ * 3 + 15) // 16 * 16)
                if smem <= 200 * 1024 or (bw <= 4 and bh <= 4):
                    break
                if pw_ * bh >= ph_ * bw and bw > 4 or bh <= 4:
                    bw //= 2
                else:
                    bh //= 2
            self._gblock = (bw, bh)
        return self._gblock

    def _crop_block_rows(self, t: Tile, use_fast: bool, bh_max: int) -> int:
        """Output rows per crop block (fast path: keep the staged input rows <= 40)."""
        if not use_fast:
            return self._generic_block[1]
        for bh in range(bh_max, 7, -1):
            if self._span_max(t.eh, t.ph, bh, True) <= 40:
                return bh
        return 8

    def kernel_path(self, use_fast=None) -> int:
        """Which kernels a work list is built for: 0 generic (any scale), 1 integer-pipe fast kernels, 2 tensor-core
        kernels.  None = the best this plan supports; True / False keep their round-1 meaning (1 / 0)."""
        path = 2 if use_fast is None else int(use_fast)
        if path >= 2 and not self.mma:
            path = 1
        if path >= 1 and not self.fast:
            path = 0
        return path

    def _mma_crop_rows(self, t: Tile, bh_max: int) -> int:
        """Output rows per tensor-core crop block: 32 unless the staged input rows would not fit the 48-row TMA box."""
        key = (t.eh, t.ph)
        for bh in ((32, 16) if bh_max >= 32 else (16,)):
            k0, end, ks = self._tab_k0[key], self._tab_end[key], self._tab_ks[key]
            worst = 0
            for oy0 in range(0, t.ph, bh):
                mv0, mv1 = oy0 // MMA_M, (min(oy0 + bh, t.ph) - 1) // MMA_M
                worst = max(worst, int(end[MMA_M * mv0:min(MMA_M * (mv1 + 1), t.ph)].max() - k0[mv0]))
            if worst <= 48:
                return bh
        return 16

    def crop_worklist(self, tile_ids: Sequence[int], B: int, use_fast: Optional[bool] = None) -> Tuple[WorkList, np.ndarray, int]:
        path = self.kernel_path(use_fast)
        use_fast = path >= 1
        offs, total = self.slot_offsets(tile_ids, B)
        rows = []
        pw_max = ph_max = 1
        nbytes = 0
        bw, bh_max = self.block_shape(use_fast, [(self.tiles[t].pw - nat.FAST_BLOCK_W, self.tiles[t].ph) for t in tile_ids], B,
                                      mma=path == 2)
        for i, tid in enumerate(tile_ids):
            t = self.tiles[tid]
            bh = self._mma_crop_rows(t, bh_max) if path == 2 else self._crop_block_rows(t, use_fast, bh_max)
            ox = np.arange(0, t.pw, bw, dtype=np.int64)
            oy = np.arange(0, t.ph, bh, dtype=np.int64)
            gx, gy = np.meshgrid(ox, oy)
            n = gx.size
            it = np.zeros((n, nat.CROP_ITEM_WORDS), dtype=np.int64)
            it[:, 0], it[:, 1], it[:, 2] = tid, gx.ravel(), gy.ravel()
            it[:, 3], it[:, 4], it[:, 5] = offs[i] & 0xFFFFFFFF, offs[i] >> 32, bh
            rows.append(it)
            pw_max = max(pw_max, self._span_max(t.ew, t.pw, bw, True))
            ph_max = max(ph_max, self._span_max(t.eh, t.ph, bh, True))
            nbytes += t.ew * t.eh * 3 + t.pw * t.ph * 3 * 4      # u8 window read + fp32 tile write
        items = np.concatenate(rows, 0) if rows else np.zeros((0, nat.CROP_ITEM_WORDS), dtype=np.int64)
        if path == 2 and items.shape[0]:
            items, pw_max, ph_max = self._crop_jobs_mma(items)
        elif use_fast and items.shape[0]:
            items = self._crop_jobs(items)
        items = items.astype(np.uint32).view(np.int32) if items.size else items.astype(np.int32)
        ks2 = bool(path == 2 and items.size and (items.reshape(-1, nat.JOB_WORDS)[:, [nat.J_TAPS_H, nat.J_TAPS_V]] > 1).any())
        return WorkList(np.ascontiguousarray(items), None, pw_max, ph_max, nbytes,
                        block_rows=0 if use_fast else bh_max, block_cols=0 if use_fast else bw, path=path, ks2=ks2), offs, total

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
        """Work lists of one dependency wave for the split schedule (engine.run_split).
        -> (crop, offs, total, late mask or None, blend).
        crop jobs: `late` ones read pixels the previous wave `prev` changes, the rest may run beside the previous wave's
        sampler and blend."""
        cr, coffs, ctotal = self.crop_worklist(wave, B, path)
        late = self.crop_split(cr, prev) if (prev and cr.path >= 1) else None
        return cr, coffs, ctotal, late, self.blend_worklist(wave, offs, 4, path, B)

    # ---- tensor-core job records ---------------------------------------------------------
    def _mma_axis(self, key: Tuple[int, int], base: np.ndarray, extent: np.ndarray):
        """One axis of the tensor-core job records.  base = output index of block column / row 0 (any alignment, may be
        negative), extent = block size along the axis.  -> (frag pool index, k-steps, staged start s0 (input index,
        multiple of 4), staged count, K-window need = inputs from s0 the last M-tile's window reaches)."""
        k0, end, ks, n_out = self._tab_k0[key], self._tab_end[key], self._tab_ks[key], key[1]
        n_in = key[0]
        lo = np.clip(base, 0, n_out - 1)
        hi = np.clip(base + extent, 1, n_out)                       # exclusive
        m0, m1 = lo // MMA_M, (hi - 1) // MMA_M
        s0 = k0[m0]
        cmax = np.maximum.accumulate(end)                          # first + count is non-decreasing in practice; be safe
        last = np.minimum(MMA_M * (m1 + 1), n_out) - 1
        stop = np.minimum(cmax[last], n_in)
        count = np.maximum(stop - s0, 1)
        need = k0[m1] + MMA_K * ks - s0
        return self._tab_frag[key], ks, s0, count, need

    def _crop_jobs_mma(self, items: np.ndarray):
        """Generic crop items [tile, ox0, oy0, off_lo, off_hi, bh] -> tensor-core job records (USDU_FLAG_MMA)."""
        n = items.shape[0]
        J = np.zeros((n, nat.JOB_WORDS), dtype=np.int64)
        tid, ox0, oy0, bh = items[:, 0], items[:, 1], items[:, 2], items[:, 5]
        geo = np.array([[t.x1, t.y1, t.ew, t.eh, t.pw, t.ph] for t in self.tiles], dtype=np.int64)[tid]
        x1, y1, ew, eh, pw, ph = geo.T
        sx0 = np.zeros(n, np.int64); cols = np.zeros(n, np.int64); need_w = np.zeros(n, np.int64)
        sy0 = np.zeros(n, np.int64); rws = np.zeros(n, np.int64); need_h = np.zeros(n, np.int64)
        for key in {(int(a), int(b)) for a, b in zip(ew, pw)}:
            m = (ew == key[0]) & (pw == key[1])
            J[m, nat.J_ROWS_H], J[m, nat.J_TAPS_H], sx0[m], cols[m], need_w[m] = self._mma_axis(key, ox0[m], np.full(int(m.sum()), nat.FAST_BLOCK_W))
        for key in {(int(a), int(b)) for a, b in zip(eh, ph)}:
            m = (eh == key[0]) & (ph == key[1])
            J[m, nat.J_ROWS_V], J[m, nat.J_TAPS_V], sy0[m], rws[m], need_h[m] = self._mma_axis(key, oy0[m], bh[m])
        cols = (cols + 3) & ~3
        J[:, nat.J_SRC_A], J[:, nat.J_SRC_B], J[:, nat.J_LEAD] = x1 + sx0, y1 + sy0, 0
        J[:, nat.J_COLS], J[:, nat.J_ROWS], J[:, nat.J_IX0], J[:, nat.J_IY0] = cols, rws, sx0, sy0
        J[:, nat.J_OX_BASE], J[:, nat.J_N_OUT_H] = ox0, pw
        J[:, nat.J_OY_BASE], J[:, nat.J_N_OUT_V] = oy0, ph
        J[:, nat.J_DST_X], J[:, nat.J_DST_Y] = ox0, oy0
        J[:, nat.J_OFF_LO], J[:, nat.J_OFF_HI] = items[:, 3], items[:, 4]
        J[:, nat.J_ROWS_OUT] = np.minimum(bh, ph - oy0)
        J[:, nat.J_COLS_OUT] = np.minimum(nat.FAST_BLOCK_W, pw - ox0)
        J[:, nat.J_PITCH] = pw * 3
        frame = ph * pw * 3
        J[:, nat.J_FRAME_LO], J[:, nat.J_FRAME_HI] = frame & 0xFFFFFFFF, frame >> 32
        J[:, nat.J_NEXT] = -1
        J[:, nat.J_CY1] = bh                                        # block height (rows per CTA)
        pw_ = int(max(cols.max(), need_w.max()))
        return J, pw_, self._mma_patch_h(rws, need_h, pw_)

    @staticmethod
    def _mma_patch_h(rws: np.ndarray, need_h: np.ndarray, patch_w: int = 0) -> int:
        """patch_h word of a tensor-core launch: plane rows in bits 0..15 -- the staged rows up to a multiple of 8 (the
        horizontal pass runs 16 rows per step and finishes with an 8-row step when <= 8 rows are left) --, rows of the
        intermediate the kernel ALLOCATES in bits 16..31.  The horizontal pass writes plane_rows rows of it; the K window of
        the last vertical M-tile may reach further (need_h), but only with zero coefficients, and the kernels lay the byte
        planes out right BEHIND the intermediate, so those reads land in the planes: the allocation stops at the written
        rows whenever the overrun fits there (it always does for one-k-step axes)."""
        plane_rows = int((rws.max() + 7) // 8 * 8)
        need = int((max(plane_rows, int(need_h.max())) + 3) // 4 * 4)
        overrun_bytes = (need - plane_rows) // 4 * 440 * 4
        planes_bytes = 3 * plane_rows * ((patch_w + 31) // 32 * 32 + 16)
        mid_rows = plane_rows if overrun_bytes <= planes_bytes else need
        return plane_rows | (mid_rows << 16)

    def _first(self, key: Tuple[int, int], idx: np.ndarray) -> np.ndarray:
        f = self._tab_first[key]
        return f[np.clip(idx, 0, f.shape[0] - 1)]

    def _crop_jobs(self, items: np.ndarray) -> np.ndarray:
        """Generic crop items [tile, ox0, oy0, off_lo, off_hi, bh] -> fast job records."""
        n = items.shape[0]
        J = np.zeros((n, nat.JOB_WORDS), dtype=np.int64)
        tid, ox0, oy0, bh = items[:, 0], items[:, 1], items[:, 2], items[:, 5]
        geo = np.array([[t.x1, t.y1, t.ew, t.eh, t.pw, t.ph] for t in self.tiles], dtype=np.int64)[tid]
        x1, y1, ew, eh, pw, ph = geo.T
        ix0 = np.zeros(n, np.int64); ix1 = np.zeros(n, np.int64); iy0 = np.zeros(n, np.int64); iy1 = np.zeros(n, np.int64)
        rows_h = np.zeros(n, np.int64); rows_v = np.zeros(n, np.int64)
        taps_h = np.zeros(n, np.int64); taps_v = np.zeros(n, np.int64)
        for key in {(int(a), int(b)) for a, b in zip(ew, pw)}:
            m = (ew == key[0]) & (pw == key[1])
            ix0[m] = self._first(key, ox0[m])
            ix1[m] = np.minimum(self._first(key, ox0[m] + nat.FAST_BLOCK_W - 1) + self._tab_taps[key], key[0])
            rows_h[m], taps_h[m] = self._tab_packed[key], self._tab_job_taps[key]
        for key in {(int(a), int(b)) for a, b in zip(eh, ph)}:
            m = (eh == key[0]) & (ph == key[1])
            iy0[m] = self._first(key, oy0[m])
            iy1[m] = np.minimum(self._first(key, oy0[m] + bh[m] - 1) + self._tab_taps[key], key[0])
            rows_v[m], taps_v[m] = self._tab_packed[key], self._tab_job_taps[key]
        J[:, nat.J_TAPS_H], J[:, nat.J_TAPS_V] = taps_h, taps_v
        px_abs = x1 + ix0
        lead = px_abs & 3
        J[:, nat.J_SRC_A], J[:, nat.J_SRC_B], J[:, nat.J_LEAD] = px_abs - lead, y1 + iy0, lead
        J[:, nat.J_COLS], J[:, nat.J_ROWS], J[:, nat.J_IX0], J[:, nat.J_IY0] = ix1 - ix0, iy1 - iy0, ix0, iy0
        J[:, nat.J_ROWS_H], J[:, nat.J_OX_BASE], J[:, nat.J_N_OUT_H] = rows_h, ox0, pw
        J[:, nat.J_ROWS_V], J[:, nat.J_OY_BASE], J[:, nat.J_N_OUT_V] = rows_v, oy0, ph
        J[:, nat.J_DST_X], J[:, nat.J_DST_Y] = ox0, oy0
        J[:, nat.J_OFF_LO], J[:, nat.J_OFF_HI] = items[:, 3], items[:, 4]
        J[:, nat.J_ROWS_OUT] = np.minimum(bh, ph - oy0)
        J[:, nat.J_COLS_OUT] = np.minimum(nat.FAST_BLOCK_W, pw - ox0)
        J[:, nat.J_PITCH] = pw * 3
        frame = ph * pw * 3
        J[:, nat.J_FRAME_LO], J[:, nat.J_FRAME_HI] = frame & 0xFFFFFFFF, frame >> 32
        J[:, nat.J_NEXT] = -1
        return J

    def blend_worklist(self, tile_ids: Sequence[int], offs: np.ndarray, src_bytes_per_elem: int = 4,
                       use_fast: Optional[bool] = None, B: int = 1, part: Optional[Tuple[int, int]] = None) -> WorkList:
        """Canvas blocks touched by the given tiles; each block lists its tiles in the
        given order (the order of `tile_ids` IS the blend order).  part = (i, n): only the blocks of the i-th of n
        horizontal slabs of the canvas (whole block rows, WorkList.rows = the slab's canvas rows; the n slabs tile
        the canvas) -- every block is owned by exactly one CTA, so n participants given the same tile list
        composite disjoint slabs (dist.upscale_static: each rank finishes its own slab of the final canvas)."""
        path = self.kernel_path(use_fast)
        use_fast = path >= 1
        ext = []
        for t in tile_ids:
            sx0, sy0, sx1, sy1 = self.support(self.tiles[t])
            ext.append((sx1 - sx0, sy1 - sy0))
        bw, bh = self.block_shape(use_fast, ext, B, mma=path == 2)
        nbx = (self.W + bw - 1) // bw
        nby = (self.H + bh - 1) // bh
        rows = None
        if part is not None:
            i, n = part
            lo_b, hi_b = (nby * i) // n, (nby * (i + 1)) // n
            rows = (min(lo_b * bh, self.H), min(hi_b * bh, self.H))
        keys, tids, seq = [], [], []
        pw_max = ph_max = 1
        nbytes = 0
        for s, tid in enumerate(tile_ids):
            t = self.tiles[tid]
            sx0, sy0, sx1, sy1 = self.support(t)
            if sx1 <= sx0 or sy1 <= sy0:
                continue
            X0, Y0, X1, Y1 = t.x1 + sx0, t.y1 + sy0, t.x1 + sx1, t.y1 + sy1
            gx = np.arange(X0 // bw, (X1 - 1) // bw + 1, dtype=np.int64)
            gy = np.arange(Y0 // bh, (Y1 - 1) // bh + 1, dtype=np.int64)
            if part is not None:
                gy = gy[(gy >= lo_b) & (gy < hi_b)]
                if gy.size == 0:
                    continue
            k = (gy[:, None] * nbx + gx[None, :]).ravel()
            keys.append(k)
            tids.append(np.full(k.size, tid, dtype=np.int64))
            seq.append(np.full(k.size, s, dtype=np.int64))
            pw_max = max(pw_max, self._span_max(t.pw, t.ew, bw, False))
            ph_max = max(ph_max, self._span_max(t.ph, t.eh, bh, False))
            frac = 1.0 if part is None else gy.size * bh / max(Y1 - Y0, 1)
            nbytes += int(min(frac, 1.0) * (t.pw * t.ph * 3 * src_bytes_per_elem + 2 * (sx1 - sx0) * (sy1 - sy0) * 3))
        if not keys:
            return WorkList(np.zeros((0, nat.JOB_WORDS if use_fast else nat.BLEND_ITEM_WORDS), np.int32),
                            None if use_fast else np.zeros((0, nat.COVER_WORDS), np.int32), pw_max, ph_max, 0,
                            n_launch=0, block_rows=bh, block_cols=0 if use_fast else bw, rows=rows, path=path)
        keys, tids, seq = np.concatenate(keys), np.concatenate(tids), np.concatenate(seq)
        order = np.lexsort((seq, keys))             # by block, then by position in tile_ids
        keys, tids, seq = keys[order], tids[order], seq[order]
        first = np.flatnonzero(np.r_[True, keys[1:] != keys[:-1]])
        counts = np.diff(np.r_[first, keys.size])
        items = np.zeros((first.size, nat.BLEND_ITEM_WORDS), dtype=np.int64)
        items[:, 0] = (keys[first] % nbx) * bw
        items[:, 1] = (keys[first] // nbx) * bh
        items[:, 2] = first
        items[:, 3] = counts
        if use_fast:
            jobs = self._blend_jobs(keys, tids, np.asarray(offs, dtype=np.int64)[seq], first, nbx, bw, bh, path == 2)
            if path == 2:
                jobs, pw_max, ph_max = jobs
            ks2 = bool(path == 2 and (jobs[:, [nat.J_TAPS_H, nat.J_TAPS_V]] > 1).any())
            return WorkList(np.ascontiguousarray(jobs.astype(np.uint32).view(np.int32)), None, pw_max, ph_max, nbytes,
                            n_launch=int(first.size), block_rows=bh, rows=rows, path=path, ks2=ks2)
        cover = np.zeros((keys.size, nat.COVER_WORDS), dtype=np.int64)
        o = np.asarray(offs, dtype=np.int64)[seq]
        cover[:, 0], cover[:, 1], cover[:, 2] = tids, o & 0xFFFFFFFF, o >> 32
        return WorkList(np.ascontiguousarray(items.astype(np.uint32).view(np.int32)),
                        np.ascontiguousarray(cover.astype(np.uint32).view(np.int32)), pw_max, ph_max, nbytes,
                        block_rows=bh, block_cols=bw, rows=rows)


    def _blend_jobs(self, keys, tids, src_off, first, nbx, bw, bh, mma: bool = False):
        """(block, tile) pairs sorted by (block, blend order) -> fast job records; the first
        record of every block comes first (they form the grid), the rest is chained by NEXT.
        mma: tensor-core flavour of the records (-> records, patch_w, patch_h word)."""
        n = keys.size
        bx0, by0 = (keys % nbx) * bw, (keys // nbx) * bh
        geo = np.array([[t.x1, t.y1, t.ew, t.eh, t.pw, t.ph] for t in self.tiles], dtype=np.int64)[tids]
        x1, y1, ew, eh, pw, ph = geo.T
        desc = self.tile_desc.astype(np.int64)[tids]
        ox_base, oy_base = bx0 - x1, by0 - y1
        ix0 = np.zeros(n, np.int64); ix1 = np.zeros(n, np.int64); iy0 = np.zeros(n, np.int64); iy1 = np.zeros(n, np.int64)
        rows_h = np.zeros(n, np.int64); rows_v = np.zeros(n, np.int64)
        taps_h = np.zeros(n, np.int64); taps_v = np.zeros(n, np.int64)
        need_w = np.zeros(n, np.int64); need_h = np.zeros(n, np.int64)
        for key in {(int(a), int(b)) for a, b in zip(pw, ew)}:
            m = (pw == key[0]) & (ew == key[1])
            if mma:
                rows_h[m], taps_h[m], ix0[m], cnt, need_w[m] = self._mma_axis(key, ox_base[m], np.full(int(m.sum()), bw))
                ix1[m] = ix0[m] + ((cnt + 3) & ~3)
                continue
            ix0[m] = self._first(key, ox_base[m])
            ix1[m] = np.minimum(self._first(key, ox_base[m] + bw - 1) + self._tab_taps[key], key[0])
            rows_h[m], taps_h[m] = self._tab_packed[key], self._tab_job_taps[key]
        for key in {(int(a), int(b)) for a, b in zip(ph, eh)}:
            m = (ph == key[0]) & (eh == key[1])
            if mma:
                rows_v[m], taps_v[m], iy0[m], cnt, need_h[m] = self._mma_axis(key, oy_base[m], np.full(int(m.sum()), bh))
                iy1[m] = iy0[m] + cnt
                continue
            iy0[m] = self._first(key, oy_base[m])
            iy1[m] = np.minimum(self._first(key, oy_base[m] + bh - 1) + self._tab_taps[key], key[0])
            rows_v[m], taps_v[m] = self._tab_packed[key], self._tab_job_taps[key]
        lead = np.zeros(n, np.int64) if mma else ix0 & 3
        J = np.zeros((n, nat.JOB_WORDS), dtype=np.int64)
        J[:, nat.J_TAPS_H], J[:, nat.J_TAPS_V] = taps_h, taps_v
        src = src_off + (iy0 * pw + ix0 - lead) * 3
        J[:, nat.J_SRC_A], J[:, nat.J_SRC_B], J[:, nat.J_LEAD] = src & 0xFFFFFFFF, src >> 32, lead
        J[:, nat.J_COLS], J[:, nat.J_ROWS], J[:, nat.J_IX0], J[:, nat.J_IY0] = ix1 - ix0, iy1 - iy0, ix0, iy0
        J[:, nat.J_ROWS_H], J[:, nat.J_OX_BASE], J[:, nat.J_N_OUT_H] = rows_h, ox_base, ew
        J[:, nat.J_ROWS_V], J[:, nat.J_OY_BASE], J[:, nat.J_N_OUT_V] = rows_v, oy_base, eh
        J[:, nat.J_DST_X], J[:, nat.J_DST_Y] = bx0, by0
        mpitch = desc[:, nat.T_MASK_PITCH]
        moff = (desc[:, nat.T_MASK_OFF] & 0xFFFFFFFF) + oy_base * mpitch + ox_base          # may be negative
        J[:, nat.J_OFF_LO], J[:, nat.J_OFF_HI] = moff & 0xFFFFFFFF, moff >> 32
        cw, chh = np.minimum(bw, self.W - bx0), np.minimum(bh, self.H - by0)
        X0 = np.maximum(bx0, x1 + desc[:, nat.T_SUP_X0]); X1 = np.minimum(bx0 + cw, x1 + desc[:, nat.T_SUP_X1])
        Y0 = np.maximum(by0, y1 + desc[:, nat.T_SUP_Y0]); Y1 = np.minimum(by0 + chh, y1 + desc[:, nat.T_SUP_Y1])
        J[:, nat.J_CX0], J[:, nat.J_CX1], J[:, nat.J_CY0], J[:, nat.J_CY1] = X0 - bx0, X1 - bx0, Y0 - by0, Y1 - by0
        J[:, nat.J_ROWS_OUT] = Y1 - by0
        opaque = ((cw == bw) & (chh == bh) & (bx0 >= x1 + desc[:, nat.T_FULL_X0]) & (bx0 + bw <= x1 + desc[:, nat.T_FULL_X1]) &
                  (by0 >= y1 + desc[:, nat.T_FULL_Y0]) & (by0 + bh <= y1 + desc[:, nat.T_FULL_Y1]))
        J[:, nat.J_FLAGS] = opaque.astype(np.int64)
        J[:, nat.J_MPITCH], J[:, nat.J_PITCH] = mpitch, pw * 3
        frame = ph * pw * 3
        J[:, nat.J_FRAME_LO], J[:, nat.J_FRAME_HI] = frame & 0xFFFFFFFF, frame >> 32
        # record order: heads (one per block) first, then the rest; chain through NEXT
        is_head = np.zeros(n, bool)
        is_head[first] = True
        pos = np.empty(n, np.int64)
        pos[is_head] = np.arange(first.size)
        pos[~is_head] = first.size + np.arange(n - first.size)
        nxt = np.full(n, -1, np.int64)
        same = np.r_[keys[1:] == keys[:-1], False]
        nxt[same] = pos[1:][same[:-1]]
        J[:, nat.J_NEXT] = nxt
        out = np.zeros_like(J)
        out[pos] = J
        if mma:
            pw_ = int(max((ix1 - ix0).max(), need_w.max()))
            return out, pw_, self._mma_patch_h(iy1 - iy0, need_h, pw_)
        return out


_PLAN_CACHE: LruCache[Plan] = LruCache(16)


def get_plan(W: int, H: int, tile_width: int, tile_height: int, padding: int, mask_blur: int, uniform: bool) -> Plan:
    key = (W, H, tile_width, tile_height, padding, mask_blur, bool(uniform))
    return _PLAN_CACHE.get_or_build(key, lambda: Plan.build(*key))
