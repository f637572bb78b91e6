"""The reference's utility nodes (DistributedSeed, DistributedValue, DistributedModelName, AudioBatchDivider,
DistributedEmptyImage): the reference's signatures and display names, the outputs its REAL classes gave for a fixed
input table at world size 1 (tests/golden/utility_nodes.json, written by oracle/ref_utility_nodes.py), every node type
the reference's shipped workflows use is registered, and under torch.distributed (gloo, 3 ranks) seeds and values are
per participant, in the order DistributedCollector gathers."""
import functools
import json
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as td
import torch.multiprocessing as mp

import ref_signatures
import ref_utility_nodes as rec
import usdu_oracle as orc
from __graft_entry__ import load_package

load_package()
import comfyui_distributed_b200 as pkg  # noqa: E402
from comfyui_distributed_b200 import dist as udist  # noqa: E402

GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "utility_nodes.json")))
SEED = 1125899906842


@pytest.mark.parametrize("name", rec.NODES)
def test_node_signature_equals_reference(name):
    got, want = ref_signatures.describe(pkg.NODE_CLASS_MAPPINGS[name]), GOLD["signatures"][name]
    assert got["input_order"] == want["input_order"]                 # widget order is positional in saved workflows
    assert json.loads(json.dumps(got["input_types"])) == want["input_types"]
    for key in ("return_types", "return_types_beyond_end", "return_names", "function", "category", "output_node",
                "params", "is_changed_nan"):
        assert json.loads(json.dumps(got[key])) == want[key], key


def test_all_reference_node_keys_registered_with_its_display_names():
    assert len(GOLD["node_keys"]) == 8
    assert set(GOLD["node_keys"]) <= set(pkg.NODE_CLASS_MAPPINGS)
    for key in GOLD["node_keys"]:
        assert pkg.NODE_DISPLAY_NAME_MAPPINGS[key] == GOLD["display_names"][key], key


def test_wildcard_outputs_connect_to_any_type():
    for name in ("DistributedValue", "DistributedModelName"):
        rt = pkg.NODE_CLASS_MAPPINGS[name].RETURN_TYPES
        assert not (rt[0] != "STRING") and not (rt[0] != "INT")
    rt = pkg.NODE_CLASS_MAPPINGS["AudioBatchDivider"].RETURN_TYPES
    assert tuple(rt) == ("AUDIO",) and not (rt[9] != "AUDIO")


@pytest.mark.parametrize("name", rec.NODES)
def test_outputs_equal_reference_at_world_size_1(name):
    assert udist.dist_info() == (0, 1)
    want = GOLD["outputs"][name]
    assert [c["inputs"] for c in want] == json.loads(json.dumps(rec.cases()[name]))
    for case in want:
        got = rec.run(pkg.NODE_CLASS_MAPPINGS[name], name, case["inputs"])
        assert json.loads(json.dumps(got)) == case["output"], case["inputs"]


def test_divider_and_empty_image_do_not_copy():
    wave = torch.rand(1, 2, 10)
    outs = pkg.NODE_CLASS_MAPPINGS["AudioBatchDivider"]().divide_audio({"waveform": wave, "sample_rate": 8000}, 3)
    assert all(o["waveform"].untyped_storage().data_ptr() == wave.untyped_storage().data_ptr() for o in outs)
    assert torch.equal(torch.cat([o["waveform"] for o in outs], dim=-1), wave)
    (img,) = pkg.NODE_CLASS_MAPPINGS["DistributedEmptyImage"]().create(32, 48, 3)
    assert img.shape == (0, 32, 48, 3) and img.dtype == torch.float32 and img.device.type == "cpu"


def test_shipped_workflow_node_types_are_registered():
    types = {n["type"] for nodes in GOLD["workflows"].values() for n in nodes}
    assert "DistributedSeed" in types
    assert types <= set(pkg.NODE_CLASS_MAPPINGS)
    seed_cls = pkg.NODE_CLASS_MAPPINGS["DistributedSeed"]
    opts = seed_cls.INPUT_TYPES()["required"]["seed"][1]
    for nodes in GOLD["workflows"].values():
        for n in nodes:
            if n["type"] == "DistributedSeed":               # the saved seed widget loads and passes through on the master
                seed = n["widgets_values"][0]
                assert opts["min"] <= seed <= opts["max"]
                assert seed_cls().distribute(seed) == (seed,)


# ---- 3 processes, gloo ------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _run(fn, world, *args):
    mp.spawn(_entry, args=(world, _free_port(), fn, args), nprocs=world, join=True)


def _entry(rank, world, port, fn, args):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    load_package()
    td.init_process_group("gloo", rank=rank, world_size=world)
    try:
        fn(rank, world, *args)
    finally:
        td.destroy_process_group()


def _w_seeds_and_values(rank, world):
    from comfyui_distributed_b200 import dist as udist
    from comfyui_distributed_b200.nodes import DistributedSeed, DistributedValue
    seed, value = DistributedSeed(), DistributedValue()
    assert udist.participant() == (None if rank == 0 else rank - 1)
    # no hidden inputs (plain SPMD launch): worker k is rank k + 1, so every rank gets seed + rank
    assert seed.distribute(SEED) == (SEED + rank,)
    assert seed.distribute(SEED, is_worker=True, worker_id="w1") == (SEED + rank,)      # an id that does not parse
    assert value.distribute("m", '{"1": "a", "2": "b"}') == ("m", "a", "b")[rank:rank + 1]
    (v,) = value.distribute("0", '{"_type": "INT", "1": "11.5", "2": "22"}')
    assert v == (0, 11, 22)[rank] and type(v) is int
    # the orchestrator's ids win over the rank (here rank r >= 1 is handed worker_{world-1-r})
    k = world - 1 - rank
    hidden = {"is_worker": rank != 0, "worker_id": "" if rank == 0 else f"worker_{k}"}
    assert seed.distribute(SEED, **hidden) == ((SEED,) if rank == 0 else (SEED + k + 1,))
    assert value.distribute("m", '{"1": "a", "2": "b"}', **hidden) == (("m",) if rank == 0 else ("ab"[k],))
    # rank 0 is the master whatever it is handed
    assert seed.distribute(SEED, is_worker=True, worker_id="worker_4") == ((SEED,) if rank == 0 else (SEED + 5,))


def test_seed_and_value_per_rank_three_ranks():
    _run(_w_seeds_and_values, 3)


def _image(seed):
    return torch.rand(1, 8, 6, 3, generator=torch.Generator().manual_seed(seed))


def _pack_cpu(images):     # test doubles of the GPU pack kernels (same arithmetic as the oracle)
    return torch.from_numpy(orc.quantize_u8(images.numpy()))


def _unpack_cpu(q):
    return torch.from_numpy(orc.dequantize_u8(q.numpy()))


def _w_txt2img(rank, world, orchestrated):
    """DistributedSeed -> sampler (torch.rand seeded with the node's output) -> DistributedCollector, on every rank."""
    from comfyui_distributed_b200.nodes import DistributedSeed, collector
    collector.collect_images = functools.partial(collector.collect_images, pack=_pack_cpu, unpack=_unpack_cpu)
    if orchestrated:        # hidden inputs as the reference's orchestrator sets them; ranks hold the ids in reverse
        enabled = [f"worker_{k}" for k in range(world - 1)]
        wid = "" if rank == 0 else f"worker_{world - 1 - rank}"
        seed_hidden = {"is_worker": rank != 0, "worker_id": wid}
        coll_hidden = dict(seed_hidden, enabled_worker_ids=json.dumps(enabled))
    else:                   # plain SPMD launch: nothing injected but the job id
        enabled = [f"rank{r}" for r in range(1, world)]        # the ids the collector gives ranks that have none
        seed_hidden, coll_hidden = {}, {}
    (seed_out,) = DistributedSeed().distribute(SEED, **seed_hidden)
    images, _ = collector.DistributedCollectorNode().run(_image(seed_out), multi_job_id="txt2img", **coll_hidden)
    if rank != 0:
        return
    # master, worker_0, worker_1, ...: the images for SEED, SEED + 1, SEED + 2, as the reference's own launch gives
    per_participant = [_image(SEED + i).numpy() for i in range(world)]
    ref = orc.collector_combine(per_participant[0], dict(zip(enabled, per_participant[1:])), enabled)
    assert images.shape[0] == world
    assert np.array_equal(images.numpy(), ref)


@pytest.mark.parametrize("orchestrated", [False, True], ids=["spmd", "orchestrator_ids"])
def test_txt2img_chain_collects_seeds_in_order_three_ranks(orchestrated):
    _run(_w_txt2img, 3, orchestrated)
