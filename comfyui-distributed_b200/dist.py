"""Multi-GPU plumbing: one process per GPU, torch.distributed (NCCL over NVLink 4 /
NVSwitch; gloo in the CPU tests).  Replaces the reference's HTTP + PNG transport:

* upscale/worker_comms.py:16-108  (PNG multipart POST of processed tiles)  and
  upscale/result_collector.py:36-182 (master drain loop)   -> u8 tiles stay in their owner's HBM (symmetric
                                                              memory); the blend kernels of all ranks read them
                                                              over NVLink and composite shares of the master's
                                                              canvas in place (fallback: all_gather of u8 tiles)
* upscale/worker_comms.py:124-188 (HTTP pull of tile ids)  -> static plan (planner.partition)
* nodes/collector.py:84-119 + api/job_routes.py:273-343 (base64 PNG per image)
                                                           -> all_gather of u8 images

Semantics kept (SURVEY.md section 8e, `replay_static`): every participant starts from the
quantised input, crops from ITS OWN progressive canvas, and the result is the master's
canvas with every worker tile blended on top in ascending tile id
(upscale/modes/static.py:521-553).  Workers return their input unchanged (:314).
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as td

from .casts import reference_f32
from .lru import LruCache


def dist_info(group=None) -> Tuple[int, int]:
    if td.is_available() and td.is_initialized():
        return td.get_rank(group), td.get_world_size(group)
    return 0, 1


def _parse_worker_index(worker_id: str) -> Optional[int]:
    """An injected worker id as the reference reads it: "worker_N" or a plain integer N; None when it does not parse
    (nodes/utilities.py:60-75)."""
    try:
        return int(worker_id.split("_")[1]) if worker_id.startswith("worker_") else int(worker_id)
    except (ValueError, IndexError):
        return None


def participant(is_worker: bool = False, worker_id: str = "", group=None) -> Optional[int]:
    """Which participant of a distributed prompt this process is: None for the master, k for worker k (0-based, the
    numbering of the reference's orchestrator, which injects "worker_k" for the k-th enabled worker,
    prompt_transform.py:327).  The per-participant utility nodes (DistributedSeed, DistributedValue) key off it.

    * No process group (world size 1): the hidden inputs decide, as in the reference -- is_worker=False is the master,
      is_worker=True is the worker that worker_id names; a worker_id that does not parse falls back to the master.
    * World size > 1 (SPMD, one rank per GPU): the rank decides, as for UltimateSDUpscaleDistributed.  Rank 0 is the
      master; rank r >= 1 is worker r - 1 unless an injected worker_id parses, and then that worker.  Without hidden
      inputs worker k is rank k + 1, the rank order DistributedCollector gathers in; with the orchestrator's ids it is
      the position in enabled_worker_ids, the order the collector uses then."""
    rank, world = dist_info(group)
    if world == 1:
        return _parse_worker_index(worker_id) if is_worker else None
    if rank == 0:
        return None
    k = _parse_worker_index(worker_id)
    return rank - 1 if k is None else k


# --------------------------------------------------------------------------------------
# transport (device agnostic: NCCL on CUDA tensors, gloo on CPU tensors in the tests)
# --------------------------------------------------------------------------------------
def all_gather_bytes(payload: torch.Tensor, group=None, sizes: Optional[Sequence[int]] = None) -> Tuple[torch.Tensor, List[int]]:
    """All-gather variable-length u8 payloads.  Returns (buffer [world, cap], sizes).
    One padded all_gather_into_tensor, preceded by a size exchange (int64 all_gather) only
    when the caller cannot supply `sizes` (the tile paths know them from the plan)."""
    assert payload.dtype == torch.uint8 and payload.dim() == 1
    rank, world = dist_info(group)
    if world == 1:
        return payload.view(1, -1), [payload.numel()]
    if sizes is None:
        n = torch.tensor([payload.numel()], dtype=torch.int64, device=payload.device)
        got = torch.empty(world, dtype=torch.int64, device=payload.device)
        td.all_gather_into_tensor(got, n, group=group)
        sizes = got.tolist()
    sizes = [int(s) for s in sizes]
    cap = max(max(sizes), 1)
    cap = (cap + 15) // 16 * 16
    send = payload
    if payload.numel() != cap:
        send = torch.zeros(cap, dtype=torch.uint8, device=payload.device)
        send[: payload.numel()] = payload
    out = torch.empty((world, cap), dtype=torch.uint8, device=payload.device)
    td.all_gather_into_tensor(out.view(-1), send, group=group)
    return out, sizes


def tile_payload_layout(plan, assignment: Sequence[Sequence[int]], B: int):
    """Byte offset of every tile's u8 [B,ph,pw,3] block inside its owner's payload, in
    the owner's processing order.  -> ({tile: (rank, offset)}, payload bytes per rank)"""
    where: Dict[int, Tuple[int, int]] = {}
    sizes = []
    for r, tiles in enumerate(assignment):
        cur = 0
        for tid in tiles:
            t = plan.tiles[tid]
            where[tid] = (r, cur)
            cur += B * t.ph * t.pw * 3
            cur = (cur + 15) // 16 * 16
        sizes.append(cur)
    return where, sizes


# --------------------------------------------------------------------------------------
# peer transport: the master's blend kernel pulls worker tiles straight out of the workers'
# HBM over NVLink (no gather step, no staging copy; the transfer overlaps the blend math CTA
# by CTA).  The payload buffers are symmetric allocations (same size on every rank) whose
# device addresses are exchanged once by torch's symmetric-memory rendezvous; inside one
# unified virtual address space a tile of rank r is simply  own_base + (ptr[r] - ptr[own]) +
# offset, which the blend kernel's 64-bit source offsets already express.
# --------------------------------------------------------------------------------------
USE_PEER_BLEND = os.environ.get("USDU_PEER_BLEND", "1") != "0"
# ... and, with it, the final composite is SHARDED BY CANVAS SLAB: every rank owns one horizontal slab of the final
# canvas (whole block rows), quantises it from the input, composites every tile that reaches into it -- the master's
# tiles in the master's order, then all worker tiles in ascending id, the order of static.py:521-553 inside every
# block -- into its LOCAL HBM (bulk-tensor loads and stores never leave the device; only the u8 tiles are read from
# their owners over NVLink), and the master gathers the N finished slabs with peer LOADS while it dequantises them
# into the result.  (Round 1 let every rank store its blocks into the master's canvas: N-1 ranks storing into one
# HBM with a system-scope fence per CTA made N = 8 slower than N = 2.)
USE_SHARED_FINAL_BLEND = os.environ.get("USDU_SHARED_FINAL_BLEND", "1") != "0"


def peer_offsets(order: Sequence[int], where: Dict[int, Tuple[int, int]], ptrs: Sequence[int], own_rank: int) -> np.ndarray:
    """Byte offset, relative to this rank's payload base, of every tile of `order` inside its
    owner's payload buffer (ptrs[r] = device address of rank r's buffer as mapped HERE)."""
    base = int(ptrs[own_rank])
    return np.array([int(ptrs[where[t][0]]) - base + where[t][1] for t in order], dtype=np.int64)


class PeerPayload:
    """Symmetric u8 buffer + rendezvous handle, cached per (tag, bytes, device, group)."""

    _cache: "LruCache[Optional[PeerPayload]]" = LruCache(8)
    _warned = False

    def __init__(self, nbytes: int, device, group):
        import torch.distributed._symmetric_memory as symm
        self.buf = symm.empty(nbytes, dtype=torch.uint8, device=device)
        self.hdl = symm.rendezvous(self.buf, group if group is not None else td.group.WORLD)
        self.ptrs = [int(p) for p in self.hdl.buffer_ptrs]
        self.buf.zero_()

    def barrier(self, channel: int = 0):
        """Stream-ordered barrier over all ranks (signal pads in peer memory, system-scope
        release/acquire): kernels enqueued before it on any rank are complete and visible to
        kernels enqueued after it on every rank."""
        self.hdl.barrier(channel=channel, timeout_ms=20000)

    def peer_view(self, rank: int, shape, dtype=torch.uint8) -> torch.Tensor:
        """Rank `rank`'s buffer as a tensor mapped into this process (NVLink peer memory)."""
        return self.hdl.get_buffer(rank, tuple(shape), dtype)

    @classmethod
    def get(cls, nbytes: int, device, group, tag: str = "payload") -> Optional["PeerPayload"]:
        """Collective.  Returns None on EVERY rank if any rank cannot set the buffer up (no
        NVLink/P2P, symmetric memory unsupported) -- the caller then uses the NCCL all-gather."""
        if not (USE_PEER_BLEND and td.is_initialized() and td.get_backend(group) == "nccl"):
            return None
        key = (tag, int(nbytes), str(device), id(group))
        if key in cls._cache:
            return cls._cache.get(key)
        obj, ok = None, 1
        try:
            obj = PeerPayload(int(nbytes), device, group)
        except Exception as e:     # noqa: BLE001 -- any failure means "transport not available here"
            ok = 0
            cls.last_error = repr(e)
        flag = torch.tensor([ok], dtype=torch.int32, device=device)
        td.all_reduce(flag, op=td.ReduceOp.MIN, group=group)
        if int(flag.item()) == 0:
            obj = None
            if not cls._warned:        # once: a mis-set box must not lose the NVLink transport silently
                cls._warned = True
                import warnings
                warnings.warn("comfyui-distributed_b200: symmetric-memory peer transport unavailable "
                              f"({cls.last_error or 'a peer rank failed'}); falling back to NCCL all_gather of the tiles",
                              RuntimeWarning, stacklevel=2)
        return cls._cache.put(key, obj)

    last_error: Optional[str] = None


def final_blend_order(assignment: Sequence[Sequence[int]]) -> List[int]:
    """Tile ids of all NON-master participants in the order the master composites them
    (ascending tile id, upscale/modes/static.py:521-526)."""
    return sorted(t for r, tiles in enumerate(assignment) if r != 0 for t in tiles)


# --------------------------------------------------------------------------------------
# static mode, SPMD
# --------------------------------------------------------------------------------------
class StaticJob:
    """Everything one rank needs for static-mode jobs of one geometry: the plan and its partition, the symmetric
    buffers (u8 tile payload, working canvas, final canvas), the captured per-rank wave graph and the slab of the
    final canvas this rank composites.  Cached: a second job of the same shape only replays."""

    _cache: "LruCache[StaticJob]" = LruCache(4)

    def __init__(self, plan, B: int, device, group, denoiser, assignment, graphed: bool):
        from . import engine as _eng
        from .engine import Canvas, DevicePlan
        self.plan, self.B, self.device, self.group = plan, B, device, group
        self.rank, self.world = dist_info(group)
        world = self.world
        self.asg = [list(a) for a in (assignment if assignment is not None else plan.partition(world))]
        if len(self.asg) != world:
            raise ValueError(f"assignment has {len(self.asg)} participants, world size is {world}")
        self.dp = DevicePlan.get(plan, device)
        self.conflict_free = plan.conflict_free(self.asg)
        # payload layout follows every rank's processing order (wave by wave), so a wave's packed u8 tiles land in
        # one contiguous span
        proc = [_eng.processing_order(plan, a) for a in self.asg]
        self.where, sizes = tile_payload_layout(plan, proc, B)
        self.sizes = [max(sz, 16) for sz in sizes]
        pitch = Canvas.pitch_of(plan.W)
        self.canvas_bytes = B * plan.H * pitch          # (symmetric allocations below are rounded up: slack behind the last row)
        self.peer = PeerPayload.get((max(self.sizes) + 255) // 256 * 256, device, group) if world > 1 else None
        self.work = self.final = None
        if self.peer is not None and USE_SHARED_FINAL_BLEND:
            self.work = PeerPayload.get(self.canvas_bytes + 256, device, group, tag="work")
            self.final = PeerPayload.get(self.canvas_bytes + 256, device, group, tag="final")
        self.sharded = self.final is not None and self.work is not None
        if world > 1:
            self.payload = (self.peer.buf[: self.sizes[self.rank]] if self.peer is not None
                            else _payload_buffer(self.sizes[self.rank], device))
        else:
            self.payload = None
        self.work_buf = self.work.buf[: self.canvas_bytes].view(B, plan.H, pitch) if self.sharded else None
        # the composite order of the final canvas: the master's tiles as the master processed them, then every
        # worker tile in ascending id (static.py:521-553)
        self.final_order = list(self.asg[0]) + final_blend_order(self.asg)
        self.graphed = graphed and len(self.asg[self.rank]) > 0
        # with a conflict-free partition no crop of this rank ever sees one of its own blends and, when the final
        # canvas is composited slab by slab from the payloads, nobody reads this rank's working canvas: skip them
        self.skip = ("blend",) if (self.sharded and self.conflict_free) else ()
        # ... and then its crops can read the fp32 image directly: the whole-canvas quantise (a pass over the whole canvas
        # in every rank's step, never sharded) disappears from the device-resident path
        self.from_image = bool(self.skip) and Canvas(self.dp, B, self.work_buf).can_crop_image() and len(self.asg[self.rank]) > 0
        self.gw = None
        if self.graphed:
            self.gw = _eng.GraphedWaves.get(self.dp, B, denoiser, _eng.PROFILE, order=self.asg[self.rank], payload=self.payload,
                                            where=self.where, canvas_buf=self.work_buf, skip=self.skip, external_crop=self.from_image)
        self.final_canvas = None
        self.rows = None
        if self.sharded:
            self.final_canvas = Canvas(self.dp, B, self.final.buf[: self.canvas_bytes].view(B, plan.H, pitch))
            offs = peer_offsets(self.final_order, self.where, self.peer.ptrs, self.rank)
            wl = self.dp.blend_list(tuple(self.final_order), offs, True, self.final_canvas.path_blend, B, (self.rank, world))[0]
            self.final_offs = offs
            bh = max(wl.block_rows, 1)
            nby = (plan.H + bh - 1) // bh
            self.rows = [(min((nby * q) // world * bh, plan.H), min((nby * (q + 1)) // world * bh, plan.H)) for q in range(world)]
            assert self.rows[self.rank] == tuple(wl.rows), (self.rows, wl.rows)

    @classmethod
    def get(cls, plan, B, device, group, denoiser, assignment, graphed: bool) -> "StaticJob":
        from . import engine as _eng
        akey = None if assignment is None else tuple(tuple(a) for a in assignment)
        key = (id(plan), B, str(device), id(group), getattr(denoiser, "graph_key", id(denoiser)) if graphed else "eager",
               akey, graphed, _eng.FORCE_GENERIC, _eng.FORCE_NO_MMA, USE_PEER_BLEND, USE_SHARED_FINAL_BLEND)
        return cls._cache.get_or_build(key, lambda: StaticJob(plan, B, device, group, denoiser, assignment, graphed),
                                       lambda job: job.plan is plan)

    # ---- phases -----------------------------------------------------------------------------
    def run_tiles(self, image: Optional[torch.Tensor], denoiser, resident: bool = False):
        """Phase A: this rank's tiles (crop -> sampler -> local blend -> u8 pack into the payload).  resident: the
        working canvas already holds the quantised input (host path: gathered slabs)."""
        from .engine import Canvas, run_progressive, _sorted_by_shape
        if self.gw is not None:
            if resident:                         # (host path: the working canvas holds the gathered u8 slabs; crop from it)
                if self.from_image:
                    c = self.gw.canvas
                    c.launches, c.algo_bytes = self.gw.launches_per_replay, self.gw.bytes_per_replay
                    c.crop(self.gw.crop_tiles, out=self.gw.crop_buf)
                    self.gw.graph.replay()
                    return c
                return self.gw.replay_resident()
            return self.gw.replay_from_image(image) if self.from_image else self.gw.replay(image)
        canvas = Canvas(self.dp, self.B, self.work_buf)
        if self.from_image and not resident:
            tiles = _sorted_by_shape(self.plan, self.plan.waves(self.asg[self.rank])[0])
            buf, _ = canvas.crop(tiles, image=image)
            run_progressive(canvas, self.asg[self.rank], denoiser, payload=self.payload, where=self.where,
                            skip=tuple(set(self.skip) | {"crop"}), crop_buf=buf)
            return canvas
        if not resident:
            canvas.load(image)
        run_progressive(canvas, self.asg[self.rank], denoiser, payload=self.payload, where=self.where, skip=self.skip)
        return canvas

    def composite_slab(self, image_ptr: int):
        """Phase B: this rank's slab of the final canvas = quantised input rows + every tile, in the reference's order.
        image_ptr: address of row 0 of frame 0 of the fp32 input as THIS process sees it (a slab upload passes an
        address offset so that its first row lands on the slab's first row)."""
        from . import _native as nat
        from .engine import _stream_ptr
        p, c = self.plan, self.final_canvas
        y0, y1 = self.rows[self.rank]
        if y1 > y0:
            nat.quantize_rows(image_ptr, c.buf.data_ptr(), self.B, p.H, p.W, c.pitch, y0, y1, _stream_ptr())
            c.launches += 1
        c.blend(self.final_order, self.peer.buf, self.final_offs, part=(self.rank, self.world))

    def gather_result(self, out: torch.Tensor):
        """Phase C on the producing rank: dequantise the N finished slabs straight out of their owners' HBM."""
        from . import _native as nat
        from .engine import _stream_ptr
        p, c = self.plan, self.final_canvas
        live = [q for q in range(self.world) if self.rows[q][1] > self.rows[q][0]]
        bounds = [0] + [self.rows[q][1] for q in live]
        bounds[-1] = p.H
        nat.gather_dequantize([self.final.ptrs[q] for q in live], bounds, out.data_ptr(), self.B, p.H, p.W, c.pitch, _stream_ptr())
        c.launches += 1


def upscale_static(image: torch.Tensor, denoiser, tile_width: int, tile_height: int, padding: int,
                   mask_blur: int, force_uniform_tiles: bool = True, group=None,
                   assignment: Optional[Sequence[Sequence[int]]] = None, all_ranks_result: bool = False,
                   stats: Optional[dict] = None) -> torch.Tensor:
    """Every rank calls this with the same (replicated) CUDA image, like the reference's
    workers which each re-execute the upstream graph (SURVEY.md 3.1).  Rank 0 returns the
    blended canvas; other ranks return `image` unchanged unless all_ranks_result."""
    from . import engine as _eng
    from .engine import Canvas, _require_cuda
    from .planner import get_plan

    _require_cuda(image, "image")
    rank, world = dist_info(group)
    B, H, W, _ = image.shape
    plan = get_plan(W, H, tile_width, tile_height, padding, mask_blur, force_uniform_tiles)
    image = image.contiguous()
    with torch.cuda.device(image.device):
        graphed = bool(getattr(denoiser, "cuda_graph_safe", False)) and _eng.USE_CUDA_GRAPHS
        job = StaticJob.get(plan, B, image.device, group, denoiser, assignment, graphed)
        asg, where, peer = job.asg, job.where, job.peer
        produce = rank == 0 or all_ranks_result
        if job.sharded:
            marks = [] if (stats is not None and stats.get("time_phases")) else None

            def mark(name):                              # per-rank phase times (bench.py reports the max over ranks)
                if marks is not None:
                    e = torch.cuda.Event(enable_timing=True)
                    e.record()
                    marks.append((name, e))

            mark("start")
            canvas = job.run_tiles(image, denoiser)
            mark("tiles (quantise + crop/sampler/blend waves + pack)")
            peer.barrier(0)                              # every payload is complete and visible
            mark("barrier 0")
            job.final_canvas.launches = job.final_canvas.algo_bytes = 0
            job.composite_slab(image.data_ptr())
            mark("composite own slab of the final canvas")
            peer.barrier(1)                              # every slab is final; nobody refills a payload that is being read
            mark("barrier 1")
            res = image
            if produce:
                res = torch.empty((B, H, W, 3), dtype=torch.float32, device=image.device)
                job.gather_result(res)
            mark("gather + dequantise the slabs (producing rank)")
            if marks is not None:
                torch.cuda.current_stream().synchronize()
                stats["phase_ms"] = {marks[i][0]: marks[i - 1][1].elapsed_time(marks[i][1]) for i in range(1, len(marks))}
            launches = canvas.launches + job.final_canvas.launches
            algo = canvas.algo_bytes + job.final_canvas.algo_bytes
        else:
            base = None
            if job.gw is not None and not all_ranks_result:
                canvas = job.gw.replay(image)
            else:
                canvas = Canvas(job.dp, B).load(image)
                base = canvas.clone() if (all_ranks_result and rank != 0) else None
                _eng.run_progressive(canvas, asg[rank], denoiser, payload=job.payload, where=where)
            if world > 1:
                target, order = canvas, final_blend_order(asg)
                if produce and rank != 0:
                    # rebuild the master's canvas: base + master tiles in the master's order
                    target, order = base, list(asg[0]) + order
                if peer is not None:
                    peer.barrier(0)                          # every payload is complete and visible
                    if produce:
                        target.blend(order, peer.buf, peer_offsets(order, where, peer.ptrs, rank))
                    peer.barrier(1)                          # nobody refills its payload while it is being read
                else:
                    gathered, _ = all_gather_bytes(job.payload, group, sizes=job.sizes)
                    cap = gathered.shape[1]
                    if produce:
                        offs = np.array([where[t][0] * cap + where[t][1] for t in order], dtype=np.int64)
                        target.blend(order, gathered.view(-1), offs)
                if produce:
                    canvas = target
            res = canvas.result() if produce else image
            launches, algo = canvas.launches, canvas.algo_bytes
    if stats is not None:
        stats["gpu_launches"] = stats.get("gpu_launches", 0) + launches
        stats["algo_bytes"] = stats.get("algo_bytes", 0) + algo
        stats["tiles"] = len(plan.tiles)
        stats["tiles_this_rank"] = len(asg[rank])
        stats["conflict_free"] = job.conflict_free
        stats["transport"] = "single" if world == 1 else ("nvlink peer loads" if peer is not None else "nccl all_gather")
        stats["final_blend"] = ("master" if not job.sharded else
                                f"sharded: each of {world} ranks composites its slab of the final canvas locally, the master gathers the slabs")
    return res


# --------------------------------------------------------------------------------------
# static mode on HOST tensors: every rank moves 1/N of the image over ITS OWN PCIe link
# --------------------------------------------------------------------------------------
class _near_gpu_cpus:
    """Context: run on the CPUs next to this process's current GPU (NVML's affinity mask) -- used for first-touch page
    placement only; silently a no-op when NVML or sched_setaffinity is unavailable."""

    def __enter__(self):
        self.saved = None
        try:
            import pynvml
            pynvml.nvmlInit()
            uuid = torch.cuda.get_device_properties(torch.cuda.current_device()).uuid
            h = pynvml.nvmlDeviceGetHandleByUUID(("GPU-" + str(uuid)).encode())
            n_words = (os.cpu_count() + 63) // 64
            mask = pynvml.nvmlDeviceGetCpuAffinity(h, n_words)
            cpus = {64 * i + b for i, w in enumerate(mask) for b in range(64) if (int(w) >> b) & 1}
            if cpus:
                self.saved = os.sched_getaffinity(0)
                os.sched_setaffinity(0, cpus & self.saved or cpus)
        except Exception:        # noqa: BLE001 -- placement is an optimisation
            self.saved = None
        return self

    def __exit__(self, *exc):
        if self.saved is not None:
            try:
                os.sched_setaffinity(0, self.saved)
            except Exception:    # noqa: BLE001
                pass
        return False


class SharedHost:
    """Result buffers in POSIX shared memory, page-locked (cudaHostRegister) in every rank's process, plus a small
    control block for host-side hand-shakes.  The reference's workers each hold the whole canvas and the master alone
    returns the result (upscale/modes/static.py:209-212, :556-564); here every rank downloads its slab of the final
    canvas into the master's result tensor directly, so no result byte crosses NVLink or the master's PCIe link.

    Life time of the memory: a buffer's file is unlinked as soon as every rank has mapped it (a crashed job leaves nothing
    in /dev/shm); at most MAX_MAPPED buffers stay mapped and page-locked -- when a new one is needed beyond that, rank 0
    names the least recently used buffer its consumer has dropped and every rank unmaps it in the same hand-shake."""

    _inst: Dict[int, "SharedHost"] = {}
    CTRL_WORDS = 64 + 64          # [0] job id published by rank 0, [1] buffer index of that job, [2], [3] buffer (numel, index)
    #                               every rank unmaps first ([3] < 0: none), [64 + r] last job rank r finished
    MAX_MAPPED = 6

    def __init__(self, group):
        import atexit
        import uuid
        self.group = group
        self.rank, self.world = dist_info(group)
        tok = [f"{os.getpid()}_{uuid.uuid4().hex[:10]}" if self.rank == 0 else None]
        td.broadcast_object_list(tok, src=td.get_global_rank(group, 0) if group is not None else 0, group=group)
        self.uid = tok[0]
        self.paths: List[str] = []
        self.pin = torch.cuda.is_available()                # (the gloo tests drive the hand-shakes without a device)
        path = self._path("ctrl")
        if self.rank == 0:
            np.zeros(self.CTRL_WORDS, dtype=np.int64).tofile(path)
            self.paths.append(path)
        atexit.register(self.close)
        td.barrier(group=group)
        self.ctrl = np.memmap(path, dtype=np.int64, mode="r+", shape=(self.CTRL_WORDS,))
        td.barrier(group=group)
        self._unlink(path)                                  # the mappings keep the memory alive
        self.job = 0
        self.bufs: Dict[int, List[Optional[torch.Tensor]]] = {}     # numel -> mapped + registered tensors by index
        self.last_use: Dict[Tuple[int, int], int] = {}               # (numel, index) -> job

    @classmethod
    def get(cls, group) -> "SharedHost":
        key = id(group)
        if key not in cls._inst:
            cls._inst[key] = SharedHost(group)
        return cls._inst[key]

    def _path(self, name: str) -> str:
        return f"/dev/shm/usdu_b200_{self.uid}_{name}"

    def _unlink(self, path: str):
        if self.rank == 0:
            try:
                os.unlink(path)
            except OSError:
                pass
            if path in self.paths:
                self.paths.remove(path)

    def close(self):
        for p in list(self.paths):
            self._unlink(p)

    def mapped(self) -> int:
        return sum(1 for lst in self.bufs.values() for i in range(len(lst)) if lst[i] is not None)

    def _map(self, numel: int, k: int, touch: Optional[Tuple[int, int]] = None) -> torch.Tensor:
        """Buffer k of `numel` floats: mapped and page-locked on first use (once: page locking is slow), COLLECTIVELY (every
        rank maps a new buffer in the same job, see begin()).  touch = (a, b): element range this rank will write -- it
        is first-touched here."""
        lst = self.bufs.setdefault(numel, [])
        while len(lst) <= k:
            lst.append(None)
        if lst[k] is None:
            path = self._path(f"{numel}_{k}")
            t = torch.from_file(path, shared=True, size=numel, dtype=torch.float32)
            if touch is not None:
                # First touch decides which NUMA node a page of the shared buffer lives on.  Every rank touches the rows IT
                # will download into, on a CPU next to its GPU: otherwise all pages sit next to rank 0 and the GPUs of the
                # other socket write across the inter-socket link, several times slower than writes to local memory.
                a, b = touch
                with _near_gpu_cpus():
                    t.view(-1)[a:b].zero_()
            td.barrier(group=self.group)                    # everybody has the file open and mapped
            self._unlink(path)
            if self.pin:
                err = torch.cuda.cudart().cudaHostRegister(t.data_ptr(), numel * 4, 0)
                if int(err) != 0:
                    raise RuntimeError(f"cudaHostRegister of the shared result buffer failed: {err}")
            lst[k] = t
        return lst[k]

    def _unmap(self, numel: int, k: int):
        """Drop buffer (numel, k): nothing on this rank references it any more (rank 0 checked its consumer; the other
        ranks only ever hold it inside one call, and synchronised their copies before finish())."""
        lst = self.bufs.get(numel, [])
        if k < len(lst) and lst[k] is not None:
            if self.pin:
                torch.cuda.cudart().cudaHostUnregister(lst[k].data_ptr())
            lst[k] = None                                   # the last reference: the mapping goes with the storage
        self.last_use.pop((numel, k), None)

    def _pick_victim(self) -> Tuple[int, int]:
        """Rank 0: the least recently used mapped buffer nobody references, or (0, -1)."""
        from .engine import buffer_is_unreferenced
        for (numel, k), _ in sorted(self.last_use.items(), key=lambda kv: kv[1]):
            if self.bufs[numel][k] is not None and buffer_is_unreferenced(self.bufs[numel][k]):
                return numel, k
        return 0, -1

    def _wait(self, idx: int, value: int, what: str):
        import time
        t0 = time.perf_counter()
        while int(self.ctrl[idx]) < value:
            if time.perf_counter() - t0 > 120.0:
                raise RuntimeError(f"shared-host hand-shake timed out waiting for {what}")

    def begin(self, shape, touch: Optional[Tuple[int, int]] = None) -> torch.Tensor:
        """Collective (host side only): the result tensor of the next job, the same physical pages on every rank.
        Rank 0 picks a buffer nobody references any more (engine.buffer_is_unreferenced) or maps a new one.
        touch: flat element range of the result this rank writes (NUMA placement of a new buffer, see _map)."""
        from .engine import buffer_is_unreferenced
        numel = int(np.prod(shape))
        self.job += 1
        if self.rank == 0:
            lst = self.bufs.setdefault(numel, [])
            k = -1                             # (index loops: a loop variable bound to the tensor would count as a reference)
            for i in range(len(lst)):
                if lst[i] is not None and buffer_is_unreferenced(lst[i]):
                    k = i
                    break
            victim = (0, -1)
            if k >= 0:
                if self.pin:
                    torch.cuda.synchronize()   # copies a consumer may have queued out of a recycled buffer
            else:                              # a new buffer: create the file, then publish, then map it together with the others
                k = next((i for i in range(len(lst)) if lst[i] is None), len(lst))
                if self.mapped() >= self.MAX_MAPPED:
                    victim = self._pick_victim()
                with open(self._path(f"{numel}_{k}"), "wb") as f:
                    f.truncate(numel * 4)
                self.paths.append(self._path(f"{numel}_{k}"))
            self.ctrl[1] = k
            self.ctrl[2], self.ctrl[3] = victim
            self.ctrl[0] = self.job
        else:
            self._wait(0, self.job, "the master to publish the job")
            k = int(self.ctrl[1])
            victim = (int(self.ctrl[2]), int(self.ctrl[3]))
        if victim[1] >= 0:
            self._unmap(*victim)
        buf = self._map(numel, k, touch)
        self.last_use[(numel, k)] = self.job
        return buf.view(tuple(shape))

    def finish(self):
        """This rank's part of the result has landed (call after synchronising the copy stream); rank 0 returns once
        every rank's part has."""
        self.ctrl[64 + self.rank] = self.job
        if self.rank == 0:
            for r in range(self.world):
                self._wait(64 + r, self.job, f"rank {r}'s slab")


def upscale_static_host(host_image: torch.Tensor, denoiser, tile_width: int, tile_height: int, padding: int, mask_blur: int,
                        force_uniform_tiles: bool = True, group=None, device: Optional[torch.device] = None,
                        stats: Optional[dict] = None) -> Optional[torch.Tensor]:
    """Static mode for HOST images (what ComfyUI hands the node; every rank holds the same image because every rank
    re-executed the upstream graph, SURVEY.md 3.1).  Rank r uploads only slab r -- 1/N of the rows, over its own PCIe
    link -- and quantises it; the u8 slabs are exchanged over NVLink (a quarter of the fp32 bytes); the tiles run as in
    upscale_static; every rank composites its slab of the final canvas, dequantises it and downloads it into ONE result
    tensor in page-locked shared memory.  Returns that tensor on rank 0 and None on the other ranks; falls back to
    upload-everything + upscale_static when the NVLink peer transport is unavailable (returns NotImplemented)."""
    from . import _native as nat
    from . import engine as _eng
    from .engine import _stream_ptr
    from .planner import get_plan

    rank, world = dist_info(group)
    device = device or torch.device("cuda", torch.cuda.current_device())
    x = reference_f32(host_image).contiguous()
    B, H, W, _ = x.shape
    plan = get_plan(W, H, tile_width, tile_height, padding, mask_blur, force_uniform_tiles)
    with torch.cuda.device(device):
        graphed = bool(getattr(denoiser, "cuda_graph_safe", False)) and _eng.USE_CUDA_GRAPHS
        job = StaticJob.get(plan, B, device, group, denoiser, None, graphed)
        if not job.sharded:
            return NotImplemented
        import time as _time
        timing = stats is not None and bool(stats.get("time_phases"))
        marks, cpu = [], {}

        def mark(name):                                # GPU-side phase boundaries on this rank's stream
            if timing:
                e = torch.cuda.Event(enable_timing=True)
                e.record()
                marks.append((name, e))

        t_cpu = _time.perf_counter()
        shared = SharedHost.get(group)
        ya, yb = job.rows[rank]
        out = shared.begin((B, H, W, 3), touch=(ya * W * 3, yb * W * 3) if B == 1 else None)
        cpu["begin (host hand-shake: result buffer of this job)"] = (_time.perf_counter() - t_cpu) * 1e3
        y0, y1 = job.rows[rank]
        n = y1 - y0
        max_rows = max(b - a for a, b in job.rows)
        if getattr(job, "slab", None) is None:
            job.slab = torch.empty((B, max(max_rows, 1), W, 3), dtype=torch.float32, device=device)
            job.stage = None
        slab, work, fin = job.slab, job.work_buf, job.final_canvas
        pitch, row_bytes = fin.pitch, W * 3 * 4
        src = x
        if n > 0 and not x.is_pinned():            # pageable input: only this rank's slab goes through a pinned staging buffer
            if job.stage is None:
                job.stage = torch.empty((B, max(max_rows, 1), W, 3), dtype=torch.float32, pin_memory=True)
            job.stage[:, :n].copy_(x[:, y0:y1])
            src = None
        mark("start")
        for b in range(B):                             # H2D of the slab, one contiguous span per frame
            if n > 0:
                slab[b, :n].copy_(job.stage[b, :n] if src is None else x[b, y0:y1], non_blocking=True)
                # `slab[b]` holds rows y0..y1 of frame b: hand the kernel the address its row 0 would have
                nat.quantize_rows(slab[b].data_ptr() - y0 * row_bytes, work[b].data_ptr(), 1, H, W, pitch, y0, y1, _stream_ptr())
        mark("upload + quantise own slab")
        job.peer.barrier(0)                            # every slab of the quantised input is in its owner's working canvas
        mark("barrier (slabs quantised)")
        live = [q for q in range(world) if job.rows[q][1] > job.rows[q][0]]      # all-gather of the u8 slabs: peer loads over NVLink
        bounds = [0] + [job.rows[q][1] for q in live]
        bounds[-1] = H
        nat.gather_canvas([job.work.ptrs[q] for q in live], bounds, work.data_ptr(), B, H, W, pitch, _stream_ptr())
        mark("all-gather of the u8 slabs over NVLink")
        job.peer.barrier(1)                            # nobody blends into a working canvas that is still being read
        mark("barrier (gathered)")
        canvas = job.run_tiles(None, denoiser, resident=True)
        mark("tiles")
        job.peer.barrier(0)                            # every payload is complete and visible
        mark("barrier (payloads)")
        fin.launches = fin.algo_bytes = 0
        for b in range(B):
            if n > 0:
                nat.quantize_rows(slab[b].data_ptr() - y0 * row_bytes, fin.buf[b].data_ptr(), 1, H, W, pitch, y0, y1, _stream_ptr())
        fin.blend(job.final_order, job.peer.buf, job.final_offs, part=(rank, world))
        mark("composite own slab")
        job.peer.barrier(1)                            # nobody refills a payload that is still being read
        mark("barrier (composited)")
        for b in range(B):
            if n > 0:
                nat.dequantize_rows(fin.buf[b].data_ptr(), slab[b].data_ptr() - y0 * row_bytes, 1, H, W, pitch, y0, y1, _stream_ptr())
                out[b, y0:y1].copy_(slab[b, :n], non_blocking=True)
        mark("dequantise + download own slab")
        t_cpu = _time.perf_counter()
        torch.cuda.current_stream(device).synchronize()
        cpu["stream synchronize"] = (_time.perf_counter() - t_cpu) * 1e3
        t_cpu = _time.perf_counter()
        shared.finish()
        cpu["finish (host hand-shake: all slabs landed)"] = (_time.perf_counter() - t_cpu) * 1e3
        if timing:
            stats["phase_ms"] = {marks[i][0]: marks[i - 1][1].elapsed_time(marks[i][1]) for i in range(1, len(marks))}
            stats["phase_ms"].update({"cpu: " + k: v for k, v in cpu.items()})
    if stats is not None:
        stats["gpu_launches"] = stats.get("gpu_launches", 0) + canvas.launches + fin.launches + 3 * B
        stats["algo_bytes"] = stats.get("algo_bytes", 0) + canvas.algo_bytes + fin.algo_bytes
        stats["tiles"], stats["tiles_this_rank"] = len(plan.tiles), len(job.asg[rank])
        stats["conflict_free"] = job.conflict_free
        stats["transport"] = "nvlink peer loads"
        stats["host_path"] = f"slab {rank}: rows {y0}-{y1} of {H} up and down over this rank's PCIe link"
    return out if rank == 0 else None


_PAYLOADS: "LruCache[torch.Tensor]" = LruCache(8)


def _payload_buffer(nbytes: int, device) -> torch.Tensor:
    """Reused send buffer of the NCCL transport (stable address: it is baked into the wave graph)."""
    key = (int(nbytes), str(device))
    return _PAYLOADS.get_or_build(key, lambda: torch.zeros(int(nbytes), dtype=torch.uint8, device=device))


def release_caches():
    """Drop the cached peer buffers, static and exact jobs and send buffers (engine.release_device_caches) -- unless a
    process group of more than one rank is initialised: those entries are created collectively, and one rank dropping
    them alone would desynchronise the ranks."""
    if dist_info()[1] > 1:
        return
    for cache in (StaticJob._cache, ExactJob._cache, PeerPayload._cache, _PAYLOADS):
        cache.clear()


class ExactJob:
    """Per-geometry state of `semantics="exact"` jobs: for every dependency wave the round-robin shares, the payload
    layout, the send buffer and the gathered buffer (all sizes follow from the plan: no size exchange, no host sync,
    nothing allocated per job)."""

    _cache: "LruCache[ExactJob]" = LruCache(4)

    def __init__(self, plan, B: int, device, group):
        from .engine import _sorted_by_shape
        self.plan, self.B = plan, B
        rank, world = dist_info(group)
        self.waves = []
        for wave in plan.waves():
            wave = _sorted_by_shape(plan, wave)
            shares = [wave[r::world] for r in range(world)]
            where, sizes = tile_payload_layout(plan, shares, B)
            cap = (max(max(sizes), 16) + 15) // 16 * 16
            offs_all = np.array([where[t][0] * cap + where[t][1] for t in wave], dtype=np.int64)
            send = torch.zeros(cap, dtype=torch.uint8, device=device)
            recv = torch.empty(world * cap, dtype=torch.uint8, device=device) if world > 1 else send
            self.waves.append((wave, shares[rank], where, offs_all, send, recv))

    @classmethod
    def get(cls, plan, B, device, group) -> "ExactJob":
        key = (id(plan), B, str(device), id(group))
        return cls._cache.get_or_build(key, lambda: ExactJob(plan, B, device, group), lambda job: job.plan is plan)


def upscale_exact(image: torch.Tensor, denoiser, tile_width: int, tile_height: int, padding: int, mask_blur: int,
                  force_uniform_tiles: bool = True, group=None, stats: Optional[dict] = None) -> torch.Tensor:
    """`semantics="exact"` (SURVEY.md 8f rank 2): N ranks cooperatively execute the SINGLE-GPU
    progressive job, so the result is bit-identical to process_single_gpu at any world size
    (the reference's static mode is not -- SURVEY.md 8c).  Every rank keeps a full canvas;
    the tiles of each dependency wave are split round-robin, each rank crops + samples its
    share and packs the truncated u8 tiles straight into its send buffer, one all_gather_into_tensor
    per wave exchanges them, and every rank blends the whole wave (replicated blend keeps all canvases
    identical).  Every rank returns the result."""
    from . import _native as nat
    from .engine import Canvas, DevicePlan, _require_cuda, _stream_ptr, denoise_packed
    from .planner import get_plan

    _require_cuda(image, "image")
    rank, world = dist_info(group)
    B, H, W, _ = image.shape
    plan = get_plan(W, H, tile_width, tile_height, padding, mask_blur, force_uniform_tiles)
    with torch.cuda.device(image.device):
        dp = DevicePlan.get(plan, image.device)
        job = ExactJob.get(plan, B, image.device, group)
        canvas = Canvas(dp, B).load(image.contiguous())
        for wave, mine, where, offs_all, send, recv in job.waves:
            if mine:
                buf, offs = canvas.crop(mine)
                out = denoise_packed(plan, mine, buf, offs, B, denoiser)
                sizes = [B * plan.tiles[t].ph * plan.tiles[t].pw * 3 for t in mine]
                base = where[mine[0]][1]
                if all(sz % 16 == 0 for sz in sizes) and all(where[t][1] == base + int(offs[i]) for i, t in enumerate(mine)):
                    nat.pack_tiles_u8(out.data_ptr(), send[base:].data_ptr(), out.numel(), _stream_ptr())     # one dense span
                else:
                    q = torch.empty(out.numel(), dtype=torch.uint8, device=out.device)
                    nat.pack_tiles_u8(out.data_ptr(), q.data_ptr(), out.numel(), _stream_ptr())
                    for i, tid in enumerate(mine):
                        send[where[tid][1]: where[tid][1] + sizes[i]] = q[int(offs[i]): int(offs[i]) + sizes[i]]
                canvas.launches += 1
            if world > 1:
                td.all_gather_into_tensor(recv, send, group=group)
            canvas.blend(wave, recv, offs_all)
        res = canvas.result()
    if stats is not None:
        stats["gpu_launches"] = stats.get("gpu_launches", 0) + canvas.launches
        stats["algo_bytes"] = stats.get("algo_bytes", 0) + canvas.algo_bytes
        stats["tiles"], stats["waves"] = len(plan.tiles), len(job.waves)
        stats["transport"] = "single" if world == 1 else "nccl all_gather_into_tensor per wave (sizes from the plan)"
    return res


# --------------------------------------------------------------------------------------
# collector
# --------------------------------------------------------------------------------------
def collector_order(world: int, enabled_worker_ids: Sequence[str], worker_id_of_rank: Sequence[str]) -> List[int]:
    """Rank order of the collected batch: master (rank 0) first, then workers in the order of
    `enabled_worker_ids` with repeated ids dropped (the node de-duplicates the list before it assembles,
    nodes/collector.py:245-253; the assembly loop itself, :193-223, would repeat them), then
    unexpected ids sorted."""
    order = [0]
    rank_of = {str(w): r for r, w in enumerate(worker_id_of_rank) if r != 0}
    seen = set()
    for w in [str(x) for x in enabled_worker_ids]:
        if w in seen:
            continue
        seen.add(w)
        if w in rank_of:
            order.append(rank_of[w])
    for w in sorted(rank_of):
        if w not in seen:
            order.append(rank_of[w])
    return order


def gather_to_root(payload: torch.Tensor, extra: dict, group=None):
    """Collector transport: ONLY rank 0 consumes the batches, so the u8 images travel to rank 0 and nowhere else -- one
    gather_object of the small per-rank records ({"shape": ..., **extra}: worker id, audio) and one receive per worker
    with its exact size (nodes/collector.py:84-119 + api/job_routes.py:273-343 POST every image to the master).
    -> (u8 tensors [B_r, H, W, C] by rank, records by rank) on rank 0, (None, None) elsewhere."""
    rank, world = dist_info(group)
    record = {"shape": [int(v) for v in payload.shape], **extra}
    if world == 1:
        return [payload], [record]
    root = td.get_global_rank(group, 0) if group is not None else 0
    records = [None] * world if rank == 0 else None
    td.gather_object(record, records, dst=root, group=group)
    flat = payload.contiguous().view(-1)
    if rank != 0:
        if flat.numel():
            for w in td.batch_isend_irecv([td.P2POp(td.isend, flat, root, group)]):
                w.wait()
        return None, None
    parts, ops = [payload], []
    for r in range(1, world):
        shape = records[r]["shape"]
        buf = torch.empty(int(np.prod(shape)), dtype=torch.uint8, device=payload.device)
        if buf.numel():
            src = td.get_global_rank(group, r) if group is not None else r
            ops.append(td.P2POp(td.irecv, buf, src, group))
        parts.append(buf.view(shape))
    if ops:
        for w in td.batch_isend_irecv(ops):       # one batched group of receives (no per-op serialisation on NCCL)
            w.wait()
    return parts, records


def gather_image_payloads(payload: torch.Tensor, shape: Sequence[int], group=None):
    """All-gather one u8 image batch per rank; shapes may differ in the batch dimension.
    -> list of u8 tensors [B_r, H, W, C] indexed by rank."""
    rank, world = dist_info(group)
    meta = torch.tensor(list(shape), dtype=torch.int64, device=payload.device)
    metas = torch.empty((world, 4), dtype=torch.int64, device=payload.device)
    if world == 1:
        metas[0] = meta
    else:
        td.all_gather_into_tensor(metas.view(-1), meta, group=group)
    buf, _ = all_gather_bytes(payload.reshape(-1), group)
    out = []
    for r in range(world):
        b, h, w, c = [int(v) for v in metas[r].tolist()]
        out.append(buf[r, : b * h * w * c].view(b, h, w, c))
    return out
