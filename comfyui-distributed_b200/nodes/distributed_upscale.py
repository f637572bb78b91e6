"""UltimateSDUpscaleDistributed -- same ComfyUI node signature as the reference's
nodes/distributed_upscale.py:46-279, running the tile path on the H100 kernels.

What changes behind the signature:
* pixels never touch PIL or the CPU (except the PNG tiles an HTTP worker posts, below): the canvas lives in HBM as u8,
  crop / feather / blend are sm_90a kernels (engine.py);
* "workers" are torch.distributed ranks (one process per GPU, NCCL); the hidden inputs
  injected by the reference's orchestrator (multi_job_id, is_worker, master_url,
  enabled_worker_ids, worker_id, tile_indices, dynamic_threshold) are accepted and
  validated the same way, but the role comes from the rank (rank 0 = master);
* the tile pull-queue becomes a static plan (planner.partition);
* started by the reference's orchestrator as a worker (no torch.distributed peers), the node is a static-mode worker of
  the reference's HTTP master: tiles are pulled and posted back as PNGs (http_worker.py), each computed on this GPU
  against the worker's own u8 canvas (engine.WorkerJob);
* `semantics` (class / instance attribute, default from USDU_SEMANTICS, not a widget -- the signature stays the
  reference's): "static" = the reference's multi-worker result for that plan (upscale/modes/static.py); "exact" = the
  N ranks cooperatively compute the reference's SINGLE-GPU result (single_gpu.py:8-72), bit-identical at any world size
  (dist.upscale_exact, SURVEY.md 8f rank 2).
"""
from __future__ import annotations

import json
import os

import torch

from .. import dist as usdu_dist
from .. import http_master
from ..casts import reference_f32
from ..denoise import ComfySampler
from ..engine import WorkerJob, check_batch, job_scope, upscale_host, upscale_single
from ..http_worker import HttpStaticWorker

try:  # ComfyUI supplies these lists; outside ComfyUI keep the signature importable
    import comfy.samplers as _cs
    _SAMPLERS, _SCHEDULERS = _cs.KSampler.SAMPLERS, _cs.KSampler.SCHEDULERS
except Exception:  # pragma: no cover - exercised only inside ComfyUI
    _SAMPLERS = ["euler", "euler_ancestral", "heun", "dpm_2", "dpmpp_2m", "dpmpp_2m_sde", "dpmpp_sde", "ddim", "uni_pc"]
    _SCHEDULERS = ["normal", "karras", "exponential", "sgm_uniform", "simple", "ddim_uniform", "beta"]


class UltimateSDUpscaleDistributed:
    @classmethod
    def INPUT_TYPES(s):
        return {
            "required": {
                "upscaled_image": ("IMAGE",),
                "model": ("MODEL",),
                "positive": ("CONDITIONING",),
                "negative": ("CONDITIONING",),
                "vae": ("VAE",),
                "seed": ("INT", {"default": 0, "min": 0, "max": 0xffffffffffffffff}),
                "steps": ("INT", {"default": 20, "min": 1, "max": 10000}),
                "cfg": ("FLOAT", {"default": 8.0, "min": 0.0, "max": 100.0}),
                "sampler_name": (_SAMPLERS,),
                "scheduler": (_SCHEDULERS,),
                "denoise": ("FLOAT", {"default": 0.5, "min": 0.0, "max": 1.0, "step": 0.01}),
                "tile_width": ("INT", {"default": 512, "min": 64, "max": 2048, "step": 8}),
                "tile_height": ("INT", {"default": 512, "min": 64, "max": 2048, "step": 8}),
                "padding": ("INT", {"default": 32, "min": 0, "max": 256, "step": 8}),
                "mask_blur": ("INT", {"default": 8, "min": 0, "max": 256}),
                "force_uniform_tiles": ("BOOLEAN", {"default": True}),
                "tiled_decode": ("BOOLEAN", {"default": False}),
            },
            "hidden": {
                "multi_job_id": ("STRING", {"default": ""}),
                "is_worker": ("BOOLEAN", {"default": False}),
                "master_url": ("STRING", {"default": ""}),
                "enabled_worker_ids": ("STRING", {"default": "[]"}),
                "worker_id": ("STRING", {"default": ""}),
                "tile_indices": ("STRING", {"default": ""}),
                "dynamic_threshold": ("INT", {"default": 8, "min": 1, "max": 64}),
            },
        }

    RETURN_TYPES = ("IMAGE",)
    FUNCTION = "run"
    CATEGORY = "image/upscaling"
    semantics = os.environ.get("USDU_SEMANTICS", "static")       # multi-GPU jobs: "static" | "exact" (see module docstring)

    @classmethod
    def IS_CHANGED(cls, **kwargs):
        return float("nan")

    # -- sampler selection ------------------------------------------------------------
    @staticmethod
    def _make_denoiser(model, positive, negative, vae, seed, steps, cfg, sampler_name, scheduler, denoise,
                       tiled_decode, image_size):
        """A MODEL object that knows how to denoise device tiles itself (test doubles, the
        synthetic sampler) provides `as_usdu_denoiser`; anything else is a ComfyUI MODEL."""
        if hasattr(model, "as_usdu_denoiser"):
            return model.as_usdu_denoiser(positive=positive, negative=negative, vae=vae, seed=seed, steps=steps,
                                          cfg=cfg, sampler_name=sampler_name, scheduler=scheduler, denoise=denoise,
                                          tiled_decode=tiled_decode, image_size=image_size)
        from ..conditioning import make_cond_cropper
        return ComfySampler(model, positive, negative, vae, seed, steps, cfg, sampler_name, scheduler, denoise,
                            tiled_decode=tiled_decode, image_size=image_size, cond_cropper=make_cond_cropper())

    @job_scope()
    def run(self, upscaled_image, model, positive, negative, vae, seed, steps, cfg, sampler_name, scheduler,
            denoise, tile_width, tile_height, padding, mask_blur, force_uniform_tiles, tiled_decode,
            multi_job_id="", is_worker=False, master_url="", enabled_worker_ids="[]", worker_id="",
            tile_indices="", dynamic_threshold=8):
        rank, world = usdu_dist.dist_info()
        distributed = bool(multi_job_id) and world > 1
        worker = (rank != 0) if distributed else bool(is_worker)
        try:
            batch_size = int(getattr(upscaled_image, "shape", [1])[0])
        except Exception:
            batch_size = 1
        # 4n+1 rule, master only (nodes/distributed_upscale.py:131-142)
        if not worker and batch_size != 1 and (batch_size % 4 != 1):
            raise ValueError(
                f"Batch size {batch_size} is not of the form 4n+1. "
                "This node requires batch sizes of 1 or 4n+1 (1, 5, 9, 13, ...). "
                "Please adjust the batch size.")
        check_batch(batch_size)              # both roles: one frame per grid.y index of the tile launches
        if multi_job_id:
            json.loads(enabled_worker_ids)   # raw parse like :175/:227 -> JSONDecodeError propagates

        src_device = upscaled_image.device
        dev = src_device if upscaled_image.is_cuda else torch.device("cuda", torch.cuda.current_device())
        self.last_stats = {"time_phases": True} if getattr(self, "time_phases", False) else {}
        if multi_job_id and is_worker and world == 1:
            # The reference's HTTP orchestrator started this process as a worker (static.py:191-314): pull tile ids from
            # its master, process each on this GPU against this worker's own canvas, post the PNG tiles back, and hand
            # the input through (static.py:314).
            _, H, W, _ = upscaled_image.shape
            denoiser = self._make_denoiser(model, positive, negative, vae, seed, steps, cfg, sampler_name, scheduler,
                                           denoise, tiled_decode, (W, H))
            job = WorkerJob(upscaled_image, denoiser, tile_width, tile_height, padding, mask_blur, force_uniform_tiles,
                            device=dev)
            worker = HttpStaticWorker(master_url, multi_job_id, worker_id, padding,
                                      [(t.x1, t.y1, t.ew, t.eh) for t in job.plan.tiles], job.canvas.B)
            worker.run(job.step_png)
            self.last_stats.update(pulled=list(worker.pulled), chunks=worker.chunks)
            return (upscaled_image,)
        if multi_job_id and not is_worker and world == 1 and json.loads(enabled_worker_ids) and http_master.serving():
            # This process serves the reference's USDU routes (http_master.py): be the static-mode master of the HTTP
            # workers (static.py:371-570) -- own tiles from the shared queue on this GPU, worker PNG tiles decoded on
            # the GPU as they arrive, one composite at the end.
            _, H, W, _ = upscaled_image.shape
            denoiser = self._make_denoiser(model, positive, negative, vae, seed, steps, cfg, sampler_name, scheduler,
                                           denoise, tiled_decode, (W, H))
            job = WorkerJob(upscaled_image, denoiser, tile_width, tile_height, padding, mask_blur, force_uniform_tiles,
                            device=dev)
            master = http_master.HttpStaticMaster(job, multi_job_id, [str(w) for w in json.loads(enabled_worker_ids)])
            out = master.run()
            self.last_stats.update(master.stats, assignment=master.assignment())
            if not upscaled_image.is_cuda:
                pinned = torch.empty(out.shape, dtype=out.dtype, pin_memory=True)
                pinned.copy_(out, non_blocking=True)
                torch.cuda.current_stream(dev).synchronize()
                out = pinned
            return (out,)
        if self.semantics not in ("static", "exact"):
            raise ValueError(f"semantics must be 'static' or 'exact', got {self.semantics!r}")
        exact = distributed and self.semantics == "exact"
        if not upscaled_image.is_cuda and not distributed:
            # ComfyUI IMAGE tensors live on the host: upload, kernels and download overlap band by band
            _, H, W, _ = upscaled_image.shape
            denoiser = self._make_denoiser(model, positive, negative, vae, seed, steps, cfg, sampler_name, scheduler,
                                           denoise, tiled_decode, (W, H))
            return (upscale_host(upscaled_image, denoiser, tile_width, tile_height, padding, mask_blur,
                                 force_uniform_tiles, device=dev, stats=self.last_stats),)
        if distributed and not exact and not upscaled_image.is_cuda:
            # every rank moves only its slab of the image over its own PCIe link (dist.upscale_static_host)
            _, H, W, _ = upscaled_image.shape
            denoiser = self._make_denoiser(model, positive, negative, vae, seed, steps, cfg, sampler_name, scheduler,
                                           denoise, tiled_decode, (W, H))
            out = usdu_dist.upscale_static_host(upscaled_image, denoiser, tile_width, tile_height, padding, mask_blur,
                                                force_uniform_tiles, device=dev, stats=self.last_stats)
            if out is not NotImplemented:
                return (upscaled_image,) if worker else (out,)
        if upscaled_image.is_cuda:
            image = reference_f32(upscaled_image)
        else:
            # ComfyUI IMAGE tensors live on the host: stage through pinned memory
            host = reference_f32(upscaled_image).contiguous()
            host = host if host.is_pinned() else host.pin_memory()
            image = host.to(dev, non_blocking=True)
        _, H, W, _ = image.shape
        denoiser = self._make_denoiser(model, positive, negative, vae, seed, steps, cfg, sampler_name, scheduler,
                                       denoise, tiled_decode, (W, H))
        if distributed:
            run = usdu_dist.upscale_exact if exact else usdu_dist.upscale_static
            out = run(image, denoiser, tile_width, tile_height, padding, mask_blur, force_uniform_tiles, stats=self.last_stats)
            if worker:
                return (upscaled_image,)           # workers return their input (static.py:314)
        else:
            out = upscale_single(image, denoiser, tile_width, tile_height, padding, mask_blur,
                                 force_uniform_tiles, stats=self.last_stats)
        if not upscaled_image.is_cuda:
            pinned = torch.empty(out.shape, dtype=out.dtype, pin_memory=True)
            pinned.copy_(out, non_blocking=True)
            torch.cuda.current_stream(dev).synchronize()
            out = pinned
        return (out,)


NODE_CLASS_MAPPINGS = {"UltimateSDUpscaleDistributed": UltimateSDUpscaleDistributed}
NODE_DISPLAY_NAME_MAPPINGS = {"UltimateSDUpscaleDistributed": "Ultimate SD Upscale Distributed (No Upscale)"}
