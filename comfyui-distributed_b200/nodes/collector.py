"""DistributedCollector -- same node signature as the reference's nodes/collector.py:24-56.

The reference's workers PNG+base64-encode every image and POST it to the master
(collector.py:84-119 -> api/job_routes.py:273-343); here every rank contributes its batch
to one NCCL all-gather of u8 images and rank 0 assembles the result in the reference's
order: master's images first (kept at full fp32 precision, collector.py:276), then each
enabled worker's images (which went through the truncating u8 cast, collector.py:95-98),
then unexpected workers sorted by id (collector.py:193-236).  Audio stays in Python.

Started by the reference's orchestrator as an HTTP worker (no torch.distributed peers), the node sends its images to
the reference's master as that worker does: one job_complete POST per image with a level-0 PNG in base64
(http_worker.send_collector_batch).  The cast, the PNG layout and the base64 text are computed on the GPU
(usdu_png_base64_u8); only the finished text goes to the host.

As the master of HTTP workers (no torch.distributed peers, enabled workers, and this process serving the reference's
job_complete route, http_collector.py), the node collects their images as the reference's master does
(collector.py:238-469): each worker's PNGs are decoded on the GPU as they arrive, and one launch writes every worker
frame, as k / 255, into the result after the master's own frames.
"""
from __future__ import annotations

import json

import torch

from .. import dist as usdu_dist
from .. import http_collector, http_worker
from ..casts import reference_f32
from ..engine import job_scope

PNG_TEXT_BUDGET = 64 << 20    # pinned host bytes for one group of frames' base64 text (at least one frame)
PNG_MAX_GROUP = 65535         # frames of one usdu_png_base64_u8 launch (one per grid.y index)


def _native_pack(images: torch.Tensor) -> torch.Tensor:
    """IMAGE [B,H,W,C] (any device) -> u8 CUDA tensor, the reference's trunc(255*x) on the GPU."""
    from .. import _native as nat
    dev = images.device if images.is_cuda else torch.device("cuda", torch.cuda.current_device())
    x = reference_f32(images).contiguous()
    if not x.is_cuda:
        x = (x if x.is_pinned() else x.pin_memory()).to(dev, non_blocking=True)
    q = torch.empty(x.shape, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        nat.pack_tiles_u8(x.data_ptr(), q.data_ptr(), x.numel(), torch.cuda.current_stream().cuda_stream)
    return q


def _native_unpack(q: torch.Tensor) -> torch.Tensor:
    from .. import _native as nat
    out = torch.empty(q.shape, dtype=torch.float32, device=q.device)
    q = q.contiguous()
    with torch.cuda.device(q.device):
        nat.unpack_tiles_f32(q.data_ptr(), out.data_ptr(), q.numel(), torch.cuda.current_stream().cuda_stream)
    return out


_text_pool = None


def _native_png_b64(q: torch.Tensor):
    """u8 CUDA frames [B,H,W,C] -> each frame's base64 PNG text in batch order (usdu_png_base64_u8).  Frames are encoded
    in groups of at most PNG_MAX_GROUP frames whose text fits PNG_TEXT_BUDGET; a group's text is copied to pinned host
    memory once.  Each item is a memoryview into that buffer, valid until the next item is requested."""
    global _text_pool
    from .. import _native as nat
    from ..engine import _PinnedPool
    B, H, W, C = (int(v) for v in q.shape)
    if B == 0:
        return
    _, text_len, staging_len = nat.png_sizes(H, W, C)
    group = max(1, min(B, PNG_TEXT_BUDGET // text_len, PNG_MAX_GROUP))
    q = q.contiguous()
    if _text_pool is None:
        _text_pool = _PinnedPool(keep=1, shapes=2)
    host = _text_pool.get((group * text_len,), torch.uint8)
    with torch.cuda.device(q.device):
        stream = torch.cuda.current_stream()
        staging = torch.empty(group * staging_len, dtype=torch.uint8, device=q.device)
        text = torch.empty(group * text_len, dtype=torch.uint8, device=q.device)
        view = memoryview(host.numpy())
        for b0 in range(0, B, group):
            n = min(group, B - b0)
            nat.png_base64_u8(q[b0].data_ptr(), n, H, W, C, staging.data_ptr(), text.data_ptr(), stream.cuda_stream)
            host[:n * text_len].copy_(text[:n * text_len], non_blocking=True)
            stream.synchronize()
            for i in range(n):
                yield view[i * text_len:(i + 1) * text_len]


def send_to_master(images: torch.Tensor, audio, multi_job_id: str, master_url: str, worker_id: str,
                   pack=_native_pack, encode=_native_png_b64, post_times=None) -> int:
    """The reference worker's send_batch_to_master (collector.py:84-119): B = 0 sends nothing; a frame PIL cannot write
    as PNG (C other than 2, 3 or 4) raises TypeError before any request, as Image.fromarray does.  -> images sent."""
    B = int(images.shape[0]) if images.ndim >= 1 else 0
    if B == 0:
        return 0
    if images.ndim != 4 or images.shape[-1] not in (2, 3, 4):
        raise TypeError(f"DistributedCollector: cannot send frames of shape {tuple(images.shape[1:])} as PNG "
                        "(2, 3 or 4 channels)")
    return http_worker.send_collector_batch(master_url, multi_job_id, worker_id, B, encode(pack(images)), audio,
                                            post_times)


def collect_images(images: torch.Tensor, enabled_worker_ids, worker_id: str, delegate_only: bool = False,
                   group=None, pack=_native_pack, unpack=_native_unpack, audio=None):
    """SPMD collective behind the node: the u8 batches and the small per-rank records (worker id, audio) travel to
    rank 0 only (dist.gather_to_root).  Returns (combined CPU batch, rank order, audio pieces by rank) on rank 0 and
    (None, None, None) on the other ranks."""
    rank, world = usdu_dist.dist_info(group)
    q = pack(images)
    parts, records = usdu_dist.gather_to_root(q, {"worker_id": str(worker_id), "audio": audio}, group)
    if rank != 0:
        return None, None, None
    ids = [rec["worker_id"] for rec in records]
    order = usdu_dist.collector_order(world, enabled_worker_ids, ids)
    out = []
    for r in order:
        if r == 0:
            if not delegate_only:
                out.append(images.detach().to("cpu", torch.float32).contiguous())
        elif parts[r].numel() > 0:
            out.append(unpack(parts[r]).cpu())
    if not out:
        raise ValueError("No image data collected from master or workers")
    return torch.cat(out, dim=0).contiguous(), order, [rec["audio"] for rec in records]


def combine_audio(pieces, empty_audio):
    """collector.py:121-174 -- concatenate waveforms along the sample axis, master first."""
    waves, rate = [], 44100
    for a in pieces:
        if a is None:
            continue
        w = a.get("waveform")
        if w is not None and w.numel() > 0:
            if not waves or rate == 44100:
                rate = a.get("sample_rate", 44100)
            waves.append(w)
    if not waves:
        return empty_audio
    try:
        return {"waveform": torch.cat(waves, dim=-1), "sample_rate": rate}
    except Exception:
        return empty_audio


class DistributedCollectorNode:
    EMPTY_AUDIO = {"waveform": torch.zeros(1, 2, 1), "sample_rate": 44100}
    # the HTTP worker's cast (IMAGE -> u8 frames) and encoder (u8 frames -> base64 PNG texts)
    pack = staticmethod(_native_pack)
    encode = staticmethod(_native_png_b64)
    # the HTTP master's decode and assembly (None: http_collector.GpuFrames on the master's device)
    frames = None

    @classmethod
    def INPUT_TYPES(s):
        return {
            "required": {
                "images": ("IMAGE",),
                "load_balance": ("BOOLEAN", {
                    "default": False,
                    "tooltip": "Run this workflow on one least-busy participant (master included when participating).",
                }),
            },
            "optional": {"audio": ("AUDIO",)},
            "hidden": {
                "multi_job_id": ("STRING", {"default": ""}),
                "is_worker": ("BOOLEAN", {"default": False}),
                "master_url": ("STRING", {"default": ""}),
                "enabled_worker_ids": ("STRING", {"default": "[]"}),
                "worker_batch_size": ("INT", {"default": 1, "min": 1, "max": 1024}),
                "worker_id": ("STRING", {"default": ""}),
                "pass_through": ("BOOLEAN", {"default": False}),
                "delegate_only": ("BOOLEAN", {"default": False}),
            },
        }

    RETURN_TYPES = ("IMAGE", "AUDIO")
    RETURN_NAMES = ("images", "audio")
    FUNCTION = "run"
    CATEGORY = "image"

    @job_scope()
    def run(self, images, load_balance=False, audio=None, multi_job_id="", is_worker=False, master_url="",
            enabled_worker_ids="[]", worker_batch_size=1, worker_id="", pass_through=False, delegate_only=False):
        empty_audio = {"waveform": torch.zeros(1, 2, 1), "sample_rate": 44100}
        if not multi_job_id or pass_through:
            return (images, audio if audio is not None else empty_audio)
        rank, world = usdu_dist.dist_info()
        enabled = [str(w) for w in json.loads(enabled_worker_ids)]
        if world == 1:
            if is_worker:   # an HTTP worker of the reference's orchestrator: send to its master (collector.py:239-243)
                send_to_master(images, audio, multi_job_id, master_url, worker_id, pack=self.pack, encode=self.encode)
                return (images, audio if audio is not None else self.EMPTY_AUDIO)
            if enabled and http_collector.serving():
                # this process serves job_complete: collect the HTTP workers' images (collector.py:244-469)
                master = http_collector.HttpCollectorMaster(multi_job_id, enabled, frames=self.frames)
                try:
                    return master.run(images, audio, bool(delegate_only))
                finally:
                    self.last_stats = master.stats
            return (images, audio if audio is not None else empty_audio)   # no participants (collector.py:255-256)
        wid = worker_id if (worker_id or rank == 0) else f"rank{rank}"
        if not enabled:  # SPMD launch without the reference's orchestrator: every rank is enabled
            enabled = [f"rank{r}" for r in range(1, world)]
        combined, order, audios = collect_images(images, enabled, wid, delegate_only=delegate_only, audio=audio)
        if rank != 0:
            return (images, audio if audio is not None else self.EMPTY_AUDIO)
        pieces = [audios[r] for r in order if not (r == 0 and delegate_only)]
        return (combined, combine_audio(pieces, empty_audio))
