"""Results of the reference (robertvoy/ComfyUI-Distributed @ a91f9fb), recorded as SHA-256 digests in
tests/golden/reference_results.json, so that the tests which compare against it run wherever its source tree is
absent.  Where the reference can be loaded, its live result is checked against the recording first;
USDU_RECORD_REFERENCE=1 rewrites the recording instead (run the affected tests with the reference present)."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

PATH = os.path.join(os.path.dirname(__file__), "golden", "reference_results.json")
RECORD = os.environ.get("USDU_RECORD_REFERENCE") == "1"


def digest(x) -> str:
    """Digest of a nest of tensors, arrays, lists, tuples, dicts and plain values (types, shapes and bytes)."""
    h = hashlib.sha256()

    def walk(v):
        if isinstance(v, torch.Tensor):
            v = v.detach().cpu().contiguous().numpy()
        if isinstance(v, np.ndarray):
            h.update(f"A{v.dtype.str}{v.shape}".encode())
            h.update(np.ascontiguousarray(v).tobytes())
        elif isinstance(v, (list, tuple)):
            h.update(f"{type(v).__name__}{len(v)}(".encode())
            for e in v:
                walk(e)
            h.update(b")")
        elif isinstance(v, dict):
            h.update(f"dict{len(v)}(".encode())
            for k in sorted(v, key=repr):
                h.update(repr(k).encode() + b":")
                walk(v[k])
            h.update(b")")
        else:
            h.update(f"{type(v).__name__}:{v!r};".encode())

    walk(x)
    return h.hexdigest()


def _load() -> dict:
    if not os.path.isfile(PATH):
        return {}
    with open(PATH) as f:
        return json.load(f)["digests"]


def reference_digest(key: str, available: bool, run_reference) -> str:
    """Digest of what the reference returns for `key`: run_reference() when `available`, else the recording."""
    db = _load()
    if available:
        live = digest(run_reference())
        if RECORD:
            db[key] = live
            with open(PATH, "w") as f:
                json.dump({"source": "robertvoy/ComfyUI-Distributed @ a91f9fb, tests/recorded.py", "digests": dict(sorted(db.items()))},
                          f, indent=0)
                f.write("\n")
        else:
            assert db.get(key) == live, f"{key}: the reference's live result differs from its recording"
        return live
    if key not in db:
        pytest.fail(f"{key}: no recorded reference result in {os.path.basename(PATH)}")
    return db[key]
