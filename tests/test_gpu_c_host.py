"""A host with no Python: csrc/tools/usdu_c_job.c runs whole single-GPU jobs through the C ABI alone (plan, canvas,
feather masks, per wave crop -> T0 sampler -> blend), and its u8 result must hash to what the REAL reference produced
for the same job: every sweep case (tests/golden/sweep_ref_digests.json) and the full-size cfg2 / cfg5 workloads at one
GPU (tests/golden/bench_digests.json, the `reference` entries)."""
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest
import torch

from __graft_entry__ import PKG_DIR, load_package
from inputs import make_input, sweep_cases, sweep_sampler

load_package()
from comfyui_distributed_b200 import planner  # noqa: E402
from comfyui_distributed_b200.denoise import T0Denoiser  # noqa: E402

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
TOOL = os.path.join(PKG_DIR, "usdu_c_job")
SWEEP = json.load(open(os.path.join(G, "sweep_ref_digests.json")))["digests"]
BENCH = json.load(open(os.path.join(G, "bench_digests.json")))
BENCH_JOBS = {"cfg2_4k_to_8k_sdxl_512px": (1, 4320, 7680, 512, 32, 8), "cfg5_video_17f_4k": (17, 2160, 3840, 512, 32, 8)}


def run_c_job(tmp_path, img: np.ndarray, tw, th, pad, blur, uniform, seed, denoise) -> str:
    """SHA-256 of the u8 canvas usdu_c_job leaves for `img` [B, H, W, 3] under the T0 sampler (seed, denoise)."""
    B, H, W, _ = img.shape
    p = planner.get_plan(W, H, tw, th, pad, blur, uniform)
    den = T0Denoiser(seed, denoise)
    img_f, noise_f, out_f = (str(tmp_path / n) for n in ("image.f32", "noise.bin", "out.u8"))
    np.ascontiguousarray(img, dtype=np.float32).tofile(img_f)
    with open(noise_f, "wb") as f:                    # one record per processing size, pre-scaled like T0Denoiser
        for ph, pw in sorted({(t.ph, t.pw) for t in p.tiles}):
            f.write(np.array([ph, pw], np.int32).tobytes())
            f.write(den.noise((B, ph, pw, 3), "cpu").numpy().tobytes())
    r = subprocess.run([TOOL, str(W), str(H), str(B), str(tw), str(th), str(pad), str(blur), str(int(uniform)), repr(float(denoise)),
                        img_f, noise_f, out_f], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = np.fromfile(out_f, dtype=np.uint8)
    assert out.size == B * H * W * 3
    for f in (img_f, noise_f, out_f):
        os.remove(f)
    return hashlib.sha256(out.tobytes()).hexdigest()


@pytest.mark.parametrize("case", sweep_cases(), ids=lambda c: f"{c[0]}-{c[1]}-b{c[2]}-{c[4]}x{c[3]}-t{c[5]}x{c[6]}-p{c[7]}-m{c[8]}-{'u' if c[9] else 'n'}")
def test_c_host_sweep_matches_reference(case, tmp_path):
    i, kind, B, H, W, tw, th, pad, blur, uniform = case
    seed, den = sweep_sampler(i)
    assert run_c_job(tmp_path, make_input(kind, i, B, H, W), tw, th, pad, blur, uniform, seed, den) == SWEEP[str(i)]


@pytest.mark.parametrize("name", list(BENCH_JOBS))
def test_c_host_full_size_matches_reference(name, tmp_path):
    B, H, W, tile, pad, blur = BENCH_JOBS[name]
    entry = BENCH["digests"][f"{name}/n1/reference"]
    assert entry["source"] == "reference"
    g = torch.Generator().manual_seed(0)                     # bench.py's canvas: torch.rand floored to k/255
    img = (torch.floor(torch.rand(B, H, W, 3, generator=g) * 255) / 255).numpy()
    assert run_c_job(tmp_path, img, tile, tile, pad, blur, True, 123, 0.5) == entry["sha256"]
