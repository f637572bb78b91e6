"""The GPU stored-PNG + base64 encoder (usdu_png_base64_u8 behind nodes/collector._native_png_b64) against the numpy
model png_model.png_stored_b64, byte for byte, and this package's node as a collector worker on the GPU beside a
reference worker, both posting to the reference's master over HTTP on 127.0.0.1."""
import json

import numpy as np
import pytest
import torch

import collector_master
import png_model
import usdu_oracle as orc
from __graft_entry__ import load_package

load_package()
from comfyui_distributed_b200 import _native as nat  # noqa: E402
from comfyui_distributed_b200.nodes import collector  # noqa: E402

pytestmark = pytest.mark.gpu
SHAPES = [(1, 1), (1, 37), (29, 1), (60, 1000), (200, 333)]
DIVIDING_W = {2: 127, 3: 28, 4: 64}          # 1 + W*C divides 65535


def _frames(seed, B, H, W, C=3, dtype=torch.float32, device="cuda"):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand((B, H, W, C), generator=g, dtype=torch.float32) * 1.02 - 0.01   # a few values outside [0, 1]
    return x.to(dtype).to(device)


def _gpu_texts(x):
    return [bytes(t) for t in collector._native_png_b64(collector._native_pack(x))]


def _want(x):
    arr = x.cpu().float().numpy() if x.dtype == torch.bfloat16 else x.cpu().numpy()
    return [png_model.png_stored_b64(orc.quantize_u8(f)) for f in arr]


def _check(x):
    got, want = _gpu_texts(x), _want(x)
    assert len(got) == len(want)
    for b, (g, w) in enumerate(zip(got, want)):
        assert len(g) == len(w), (b, len(g), len(w))
        if g != w:
            i = next(i for i in range(len(w)) if g[i] != w[i])
            pytest.fail(f"frame {b}: first difference at text byte {i} of {len(w)}")


@pytest.mark.parametrize("C", [2, 3, 4])
def test_shapes_match_the_oracle(C):
    for k, (H, W) in enumerate(SHAPES + [(300, DIVIDING_W[C])]):
        _check(_frames(100 * C + k, 2, H, W, C))


def test_sizes_match_the_layout():
    for H, W, C in [(1, 1, 3), (720, 1280, 3), (4320, 7680, 3), (5, 64, 4)]:
        raw = H * (1 + W * C)
        nblk = -(-raw // 65535)
        png, text, staging = nat.png_sizes(H, W, C)
        assert png == 63 + 17 * nblk + raw and text == 4 * -(-png // 3) and staging >= png
    with pytest.raises(nat.NativeError):
        nat.png_sizes(8, 8, 1)


def test_batch_of_81_720p_frames(monkeypatch):
    x = _frames(7, 81, 720, 1280)
    _check(x)
    _, text_len, _ = nat.png_sizes(720, 1280, 3)
    monkeypatch.setattr(collector, "PNG_TEXT_BUDGET", 3 * text_len + 5)     # 27 groups of 3 frames
    _check(x)


def test_one_8k_frame():
    _check(_frames(8, 1, 4320, 7680))                                       # 1,521 stored blocks


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16, torch.float64])
@pytest.mark.parametrize("device", ["cuda", "cpu"])
def test_input_dtypes(dtype, device):
    _check(_frames(9, 3, 67, 245, 3, dtype, device))


def test_channel_count_is_rejected():
    with pytest.raises(TypeError):
        collector.send_to_master(_frames(1, 1, 4, 4, 1), None, "j", "http://127.0.0.1:9", "w1")


@pytest.mark.timeout(600)
@pytest.mark.parametrize("B,H,W", [(1, 544, 544), (4, 300, 420)])
def test_mixed_fleet_over_http(B, H, W):
    """The reference's master, w1 = this package's node on the GPU, w2 = the reference's worker; the combined result
    and audio are bit-identical to a run where both workers are the reference's."""
    master = _frames(20, 1, H, W, device="cpu")
    a, b = _frames(21, B, H, W), _frames(22, 2, H, W, device="cpu")
    audio = {"waveform": torch.rand(1, 2, 500, generator=torch.Generator().manual_seed(3)), "sample_rate": 48000}
    ids = ["w1", "w2"]

    def run(ours: bool):
        with collector_master.Master() as m:
            fut = m.collect(master, "job-mixed", ids)
            if ours:
                out, _ = collector.DistributedCollectorNode().run(a, audio=audio, multi_job_id="job-mixed",
                                                                  is_worker=True, master_url=m.url, worker_id="w1",
                                                                  enabled_worker_ids=json.dumps(ids))
                assert out is a
            else:
                m.worker_send(a.cpu(), audio, "job-mixed", "w1")
            m.worker_send(b, None, "job-mixed", "w2")
            return fut.result(300)

    ours, ref = run(True), run(False)
    assert torch.equal(ours[0], ref[0]) and ours[0].shape[0] == 1 + B + 2
    assert torch.equal(ours[1]["waveform"], ref[1]["waveform"]) and ours[1]["sample_rate"] == ref[1]["sample_rate"]
    want = orc.collector_combine(master.numpy(), {"w1": a.cpu().numpy(), "w2": b.numpy()}, ids)
    assert np.array_equal(ours[0].numpy(), want)
