"""oracle.collector_combine == the reference's own DistributedCollector arithmetic (worker PNG round trip,
master decode, _reorder_and_combine_tensors), loaded from /root/reference by oracle/ref_collector.py.
Where the reference tree is absent, tests/golden/collector_ref.json and tests/golden/reference_results.json
(tests/recorded.py) pin the same."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import ref_collector
import usdu_oracle as orc
from recorded import digest, reference_digest

G = os.path.join(os.path.dirname(__file__), "golden")
CASES = json.load(open(os.path.join(G, "collector_ref.json")))["cases"]


def _inputs(case):
    g = torch.Generator().manual_seed(case["seed"])
    H, W = case["H"], case["W"]
    master = torch.rand(case["master_b"], H, W, 3, generator=g)
    workers = {w: torch.rand(b, H, W, 3, generator=g) for w, b in case["workers"]}
    return master, workers


@pytest.mark.parametrize("case", CASES, ids=lambda c: c["name"])
def test_oracle_collector_matches_golden(case):
    master, workers = _inputs(case)
    out = orc.collector_combine(master.numpy(), {w: t.numpy() for w, t in workers.items()}, case["order"], case["delegate"])
    assert hashlib.sha256(np.ascontiguousarray(out, dtype=np.float32).tobytes()).hexdigest() == case["sha256"]
    assert list(out.shape) == case["shape"]


@pytest.mark.skipif(not ref_collector.available(), reason="reference tree not present")
@pytest.mark.parametrize("case", CASES, ids=lambda c: c["name"])
def test_reference_collector_matches_golden_and_oracle(case):
    master, workers = _inputs(case)
    ref = ref_collector.combine(master, workers, case["order"], case["delegate"]).numpy()
    assert hashlib.sha256(np.ascontiguousarray(ref, dtype=np.float32).tobytes()).hexdigest() == case["sha256"]
    out = orc.collector_combine(master.numpy(), {w: t.numpy() for w, t in workers.items()}, case["order"], case["delegate"])
    assert np.array_equal(out, ref)


def test_audio_combination_matches_reference():
    """nodes/collector.py:121-174 side by side with our combine_audio on random piece sets (missing audio,
    empty waveforms, non-default sample rates, unexpected worker ids)."""
    from __graft_entry__ import load_package
    load_package()
    from comfyui_distributed_b200.nodes.collector import combine_audio
    empty = {"waveform": torch.zeros(1, 2, 1), "sample_rate": 44100}
    rng = np.random.default_rng(0)
    cases = []
    for _ in range(200):
        def piece():
            k = rng.integers(0, 4)
            if k == 0:
                return None
            n = 0 if k == 1 else int(rng.integers(1, 50))
            return {"waveform": torch.from_numpy(rng.random((1, 2, n), dtype=np.float32)), "sample_rate": int(rng.choice([44100, 48000, 22050]))}
        master = piece()
        ids = ["w1", "w2", "w3", "zz"]
        workers = {w: piece() for w in ids if rng.random() < 0.8}
        order = [w for w in ["w2", "w1", "w3"] if rng.random() < 0.8]
        cases.append((master, workers, order))

    def reference():
        collector, _, _ = ref_collector.load()
        node = collector.DistributedCollectorNode()
        return [(ref["sample_rate"], ref["waveform"]) for ref in (node._combine_audio(m, w, empty, o) for m, w, o in cases)]

    got = []
    for master, workers, order in cases:
        seq = [master] + [workers.get(w) for w in order] + [workers[w] for w in sorted(workers) if w not in order]
        a = combine_audio(seq, empty)
        got.append((a["sample_rate"], a["waveform"]))
    assert digest(got) == reference_digest("collector/combine_audio/200_random_piece_sets", ref_collector.available(), reference)
