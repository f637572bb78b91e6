"""Record the reference's utility nodes (TEST INFRASTRUCTURE; recording needs the reference tree, the build container
only): the signatures of DistributedSeed, DistributedValue, DistributedModelName, AudioBatchDivider and
DistributedEmptyImage, the display names the reference registers, what the REAL classes (nodes/utilities.py, loaded
through ref_collector with nodes/__init__.py) return for a fixed table of inputs at world size 1, and which of the
reference's node types its shipped workflows use, with their widget values.
`python oracle/ref_utility_nodes.py` writes tests/golden/utility_nodes.json.

The input table, the input builders and the output encoding live here and are imported by
tests/test_utility_nodes.py, which runs this package's classes through `record` and compares with the file."""
from __future__ import annotations

import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
GOLDEN = os.path.join(os.path.dirname(HERE), "tests", "golden")

NODES = ("DistributedSeed", "DistributedValue", "DistributedModelName", "AudioBatchDivider", "DistributedEmptyImage")
WORKFLOWS = ("distributed-txt2img.json", "distributed-upscale-video.json", "distributed-upscale.json",
             "distributed-wan-2.2_14b_t2v.json", "distributed-wan.json")

ROLES = ((False, ""), (True, "worker_0"), (True, "worker_1"), (True, "worker_7"), (True, "3"), (True, "w1"), (True, ""))
SEEDS = (0, 1125899906842, 1125899906842624)
VALUE_MAPS = ("{}", '{"1":"a","2":"b"}', '{"_type":"INT","1":"3.7"}', '{"_type":"FLOAT","2":"x"}', "[1]", "{not json")
VALUE_DEFAULTS = ("7", "")
_WORKFLOW_INFO = {"workflow": {"nodes": [{"id": 5, "type": "DistributedModelName", "widgets_values": [""]},
                                         {"id": 6, "type": "Note", "widgets_values": ["keep"]}]}}


def cases() -> dict:
    """The input table: {node: [JSON-able inputs of one call]}.  Tensors are described, `build` makes them."""
    roles = [{"is_worker": w, "worker_id": i} for w, i in ROLES]
    audio = [{"waveform_shape": [1, 2, 10], "sample_rate": 48000, "divide_by": d} for d in (1, 3, 10, 12)]
    audio += [{"waveform_shape": [1, 2, 0], "divide_by": 2},                       # no sample_rate key: 44100
              {"waveform_shape": None, "sample_rate": 22050, "divide_by": 2}]
    info = _WORKFLOW_INFO
    return {
        "DistributedSeed": [{"seed": s, **r} for s in SEEDS for r in roles],
        "DistributedValue": [{"default_value": d, "worker_values": m, **r}
                             for d in VALUE_DEFAULTS for m in VALUE_MAPS for r in roles],
        "DistributedModelName": [
            {"text": "sdxl_base.safetensors", "unique_id": "5", "extra_pnginfo": info},
            {"text": ["a.safetensors", 3, {"k": [1, 2]}], "unique_id": ["5"], "extra_pnginfo": [info]},
            {"text": ["only.safetensors"], "unique_id": "6", "extra_pnginfo": info},
            {"text": 42, "unique_id": 5, "extra_pnginfo": info},
            {"text": 42, "unique_id": None, "extra_pnginfo": info},
        ],
        "AudioBatchDivider": audio,
        "DistributedEmptyImage": [{"height": h, "width": w, "channels": c}
                                  for h, w, c in ((64, 64, 3), (1, 1, 1), (4096, 17, 4))],
    }


def build(node: str, inputs: dict) -> dict:
    """Keyword arguments of the node's entry method for one row of the table (fresh objects on every call)."""
    kw = json.loads(json.dumps(inputs))
    if node == "AudioBatchDivider":
        shape = kw.pop("waveform_shape")
        wave = None if shape is None else torch.arange(int(torch.tensor(shape).prod()), dtype=torch.float32).view(shape)
        audio = {"waveform": wave}
        if "sample_rate" in kw:
            audio["sample_rate"] = kw.pop("sample_rate")
        kw["audio"] = audio
    return kw


def _encode_audio(out: dict, source) -> dict:
    w = out["waveform"]
    view = source is not None and w.untyped_storage().data_ptr() == source.untyped_storage().data_ptr()
    return {"shape": list(w.shape), "dtype": str(w.dtype), "sample_rate": out["sample_rate"], "sum": float(w.sum()),
            "bounds": [w.storage_offset(), w.storage_offset() + int(w.shape[-1])] if view else None}


def run(cls, node: str, inputs: dict):
    """Call the node's entry method on one row of the table -> a JSON-able record of what it returned."""
    kw = build(node, inputs)
    try:
        res = getattr(cls(), cls.FUNCTION)(**kw)
    except Exception as e:      # noqa: BLE001 -- an exception is part of the behaviour
        return {"raises": type(e).__name__}
    if node == "DistributedValue":
        return [{"value": v, "type": type(v).__name__} for v in res]
    if node == "DistributedModelName":
        return {"returned": json.loads(json.dumps(res)), "extra_pnginfo": kw["extra_pnginfo"]}
    if node == "AudioBatchDivider":
        return [_encode_audio(o, kw["audio"]["waveform"]) for o in res]
    if node == "DistributedEmptyImage":
        return [{"shape": list(t.shape), "dtype": str(t.dtype), "device": str(t.device)} for t in res]
    return list(res)


def record(classes: dict) -> dict:
    """{node: [{"inputs": row, "output": run(...)}]} for every row of the table."""
    return {node: [{"inputs": row, "output": run(classes[node], node, row)} for row in rows]
            for node, rows in cases().items()}


def workflow_inventory(root: str, types) -> dict:
    """{workflow file: [{"type", "widgets_values"}]} of every node of a reference type in the shipped workflows."""
    out = {}
    for name in WORKFLOWS:
        with open(os.path.join(root, "workflows", name)) as f:
            wf = json.load(f)
        out[name] = [{"type": n["type"], "widgets_values": n.get("widgets_values")}
                     for n in wf["nodes"] if n.get("type") in types]
    return out


def reference_record() -> dict:
    import ref_collector
    import ref_signatures
    ref_collector.load()                       # stub packages the reference's nodes/ imports resolve against
    util = ref_collector._load("nodes.utilities", "nodes/utilities.py")
    reg = ref_collector._load("nodes.__init__", "nodes/__init__.py")
    with open(os.path.join(GOLDEN, "node_signatures.json")) as f:     # the upscale node registers itself elsewhere
        upscale = json.load(f)["nodes"]["upscale_mappings"]
    display = {**reg.NODE_DISPLAY_NAME_MAPPINGS, **upscale["NODE_DISPLAY_NAME_MAPPINGS"]}
    keys = sorted(set(reg.NODE_CLASS_MAPPINGS) | set(upscale["NODE_CLASS_MAPPINGS"]))
    classes = {n: getattr(util, n) for n in NODES}
    return {"signatures": {n: ref_signatures.describe(classes[n]) for n in NODES},
            "node_keys": keys, "display_names": {k: display[k] for k in keys},
            "outputs": record(classes),
            "workflows": workflow_inventory(ref_collector.REF_ROOT, set(keys))}


if __name__ == "__main__":
    rec = reference_record()
    path = os.path.join(GOLDEN, "utility_nodes.json")
    with open(path, "w") as f:
        json.dump({"generator": "oracle/ref_utility_nodes.py", "reference": "a91f9fb", **rec}, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", path, {k: len(v) for k, v in rec["outputs"].items()})
