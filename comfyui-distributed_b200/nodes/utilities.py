"""The reference's utility nodes (nodes/utilities.py:23-354), with the same signatures.

* ImageBatchDivider / AudioBatchDivider: split an IMAGE batch, or an AUDIO waveform along its sample axis, into up to
  10 contiguous, near-equal chunks.  Zero-copy views on whatever device the data lives on -- the natural partners of
  DistributedCollector's gathered batch and audio.
* DistributedSeed / DistributedValue: one seed or value per participant, so that N ranks running the same prompt
  render N different images.  Who is which participant comes from dist.participant (the rank under torch.distributed,
  the orchestrator's hidden inputs otherwise).
* DistributedModelName: shows its input as text in the UI and in the saved workflow.
* DistributedEmptyImage: an empty [0, H, W, C] IMAGE for a master that delegates all the work.
No pixel work happens here: nothing in this module calls the CUDA library."""
from __future__ import annotations

import json

import torch

from .. import dist as usdu_dist

MAX_PARTS = 10


def chunk_bounds(total_items: int, n_splits: int):
    """Contiguous [start, end) bounds; the first `total % n` chunks get one extra item."""
    n = max(1, int(n_splits))
    total = max(0, int(total_items))
    base, extra = divmod(total, n)
    out, start = [], 0
    for i in range(n):
        end = start + base + (1 if i < extra else 0)
        out.append((start, end))
        start = end
    return out


class _Wildcard(str):
    """ComfyUI's link validation compares types with `!=`; a type that is never unequal connects to
    anything (the reference's AnyType, nodes/utilities.py:79-83)."""

    def __ne__(self, other) -> bool:
        return False


class _AnyTuple(tuple):
    """ComfyUI indexes RETURN_TYPES per connected output: every index answers with the wildcard type,
    like the reference's ByPassTypeTuple (nodes/utilities.py:226-233); iteration still yields the
    declared entries."""

    def __getitem__(self, index):
        item = super().__getitem__(0 if isinstance(index, int) and index > 0 else index)
        return _Wildcard("*") if isinstance(item, str) else item


class DistributedSeed:
    """The master gets `seed`, worker k gets `seed + k + 1`.  Under SPMD without hidden inputs that is `seed + rank`."""

    @classmethod
    def INPUT_TYPES(cls):
        return {
            "required": {
                "seed": ("INT", {"default": 1125899906842, "min": 0, "max": 1125899906842624, "forceInput": False}),
            },
            "hidden": {
                "is_worker": ("BOOLEAN", {"default": False}),
                "worker_id": ("STRING", {"default": ""}),
            },
        }

    RETURN_TYPES = ("INT",)
    RETURN_NAMES = ("seed",)
    FUNCTION = "distribute"
    CATEGORY = "utils"

    def distribute(self, seed, is_worker=False, worker_id=""):
        k = usdu_dist.participant(is_worker, worker_id)
        return (seed if k is None else seed + k + 1,)


def _coerce(value, value_type):
    """A DistributedValue entry as the type its map declares under "_type" (anything but INT / FLOAT stays as is)."""
    if value_type == "INT":
        return int(float(value))
    if value_type == "FLOAT":
        return float(value)
    return value


class DistributedValue:
    """The master gets `default_value`; worker k gets entry `str(k + 1)` of the JSON map `worker_values`, or
    `default_value` when that entry is missing or empty.  A map entry "_type" of "INT" or "FLOAT" converts the result;
    an entry that is not a number then also gives the default, and the default itself stays a string when it is not
    one.  Malformed JSON or a map that is not an object counts as an empty map."""

    @classmethod
    def INPUT_TYPES(cls):
        return {
            "required": {
                "default_value": ("STRING", {"default": ""}),
                "worker_values": ("STRING", {"default": "{}"}),
            },
            "hidden": {
                "is_worker": ("BOOLEAN", {"default": False}),
                "worker_id": ("STRING", {"default": ""}),
            },
        }

    RETURN_TYPES = (_Wildcard("*"),)
    RETURN_NAMES = ("value",)
    FUNCTION = "distribute"
    CATEGORY = "utils"

    def distribute(self, default_value, worker_values="{}", is_worker=False, worker_id=""):
        values = worker_values
        if isinstance(worker_values, str):
            try:
                values = json.loads(worker_values)
            except json.JSONDecodeError:
                values = {}
        if not isinstance(values, dict):
            values = {}
        value_type = values.get("_type", "STRING")
        try:
            default = _coerce(default_value, value_type)
        except (TypeError, ValueError):
            default = default_value
        k = usdu_dist.participant(is_worker, worker_id)
        if k is not None:
            raw = values.get(str(k + 1), "")
            if raw:
                try:
                    return (_coerce(raw, value_type),)
                except ValueError:
                    pass
        return (default,)


class DistributedModelName:
    """Passes its input through as text and shows it: in the UI, and as the node's widget value in the workflow that
    ComfyUI saves with the outputs."""

    @classmethod
    def INPUT_TYPES(cls):
        return {
            "required": {
                "text": ("STRING", {"default": ""}),
            },
            "hidden": {
                "unique_id": "UNIQUE_ID",
                "extra_pnginfo": "EXTRA_PNGINFO",
            },
        }

    RETURN_TYPES = (_Wildcard("*"),)
    RETURN_NAMES = ("output",)
    FUNCTION = "log_input"
    OUTPUT_NODE = True
    CATEGORY = "utils"

    @staticmethod
    def _as_text(value) -> str:
        if isinstance(value, str):
            return value
        if isinstance(value, (int, float, bool)):
            return str(value)
        try:
            return json.dumps(value, indent=4)
        except Exception:      # noqa: BLE001 -- anything json cannot encode is shown as its str()
            return str(value)

    @staticmethod
    def _show_in_workflow(extra_pnginfo, unique_id, texts):
        if not extra_pnginfo:
            return
        info = extra_pnginfo[0] if isinstance(extra_pnginfo, list) else extra_pnginfo
        if not isinstance(info, dict) or "workflow" not in info:
            return
        if isinstance(unique_id, list) and unique_id:
            node_id = str(unique_id[0])
        else:
            node_id = None if unique_id is None else str(unique_id)
        if not node_id:
            return
        node = next((n for n in info["workflow"]["nodes"] if str(n.get("id")) == node_id), None)
        if node:
            node["widgets_values"] = [texts]

    def log_input(self, text, unique_id=None, extra_pnginfo=None):
        texts = [self._as_text(v) for v in text] if isinstance(text, list) else [self._as_text(text)]
        self._show_in_workflow(extra_pnginfo, unique_id, texts)
        return {"ui": {"text": texts}, "result": (texts[0] if len(texts) == 1 else texts,)}


class ImageBatchDivider:
    @classmethod
    def INPUT_TYPES(s):
        return {"required": {
            "images": ("IMAGE",),
            "divide_by": ("INT", {"default": 2, "min": 1, "max": MAX_PARTS, "step": 1, "display": "number",
                                  "tooltip": "Number of parts to divide the batch into"}),
        }}

    RETURN_TYPES = _AnyTuple(("IMAGE",))
    RETURN_NAMES = _AnyTuple(tuple(f"batch_{i + 1}" for i in range(MAX_PARTS)))
    FUNCTION = "divide_batch"
    OUTPUT_NODE = True
    CATEGORY = "image"

    def divide_batch(self, images, divide_by):
        parts = max(1, min(int(divide_by), MAX_PARTS))
        empty = images[:0]
        outs = [images[a:b] if b > a else empty for a, b in chunk_bounds(images.shape[0], parts)]
        outs += [empty] * (MAX_PARTS - len(outs))
        return tuple(outs[:MAX_PARTS])


class AudioBatchDivider:
    """Splits an AUDIO waveform [..., samples] along its last axis.  A missing or empty waveform gives 10 one-sample
    silent stereo clips at the input's sample rate."""

    @classmethod
    def INPUT_TYPES(s):
        return {"required": {
            "audio": ("AUDIO",),
            "divide_by": ("INT", {"default": 2, "min": 1, "max": MAX_PARTS, "step": 1, "display": "number",
                                  "tooltip": "Number of parts to divide the audio into"}),
        }}

    RETURN_TYPES = _AnyTuple(("AUDIO",))
    RETURN_NAMES = _AnyTuple(tuple(f"audio_{i + 1}" for i in range(MAX_PARTS)))
    FUNCTION = "divide_audio"
    OUTPUT_NODE = True
    CATEGORY = "audio"

    def divide_audio(self, audio, divide_by):
        waveform = audio.get("waveform")
        rate = audio.get("sample_rate", 44100)
        if waveform is None or waveform.numel() == 0:
            return ({"waveform": torch.zeros(1, 2, 1), "sample_rate": rate},) * MAX_PARTS
        parts = max(1, min(int(divide_by), MAX_PARTS))
        empty = waveform[..., :0]
        outs = [{"waveform": waveform[..., a:b] if b > a else empty, "sample_rate": rate}
                for a, b in chunk_bounds(waveform.shape[-1], parts)]
        outs += [{"waveform": empty, "sample_rate": rate}] * (MAX_PARTS - len(outs))
        return tuple(outs)


class DistributedEmptyImage:
    """An IMAGE batch of 0 frames, float32 on the host: what a master that delegates all the work hands downstream."""

    @classmethod
    def INPUT_TYPES(cls):
        return {
            "required": {
                "height": ("INT", {"default": 64, "min": 1, "max": 4096, "step": 1}),
                "width": ("INT", {"default": 64, "min": 1, "max": 4096, "step": 1}),
                "channels": ("INT", {"default": 3, "min": 1, "max": 4, "step": 1}),
            }
        }

    RETURN_TYPES = ("IMAGE",)
    FUNCTION = "create"
    CATEGORY = "image"

    def create(self, height, width, channels):
        return (torch.zeros((0, height, width, channels), dtype=torch.float32),)
