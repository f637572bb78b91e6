"""This package's node as the collector master of HTTP workers on the GPU (http_collector.py, csrc/usdu_png_decode.cu):
the decode kernel across its ring depths up to 16,384 RGBA pixels, the gather-unpack assembly, and whole jobs where the
reference's worker and this package's worker post to this package's master.  Each result and its audio must equal, bit
for bit, what the reference's master (tests/collector_master.Master) returns given the same POSTs."""
import json
import threading

import numpy as np
import pytest
import torch

import collector_master
import usdu_oracle as orc
from __graft_entry__ import load_package
from test_gpu_http_master import decode_on_gpu
from test_http_collector import JOB, Ours, body, post, ref_master, same_result
from test_http_master import image, png_of

load_package()
from comfyui_distributed_b200 import _native as nat  # noqa: E402
from comfyui_distributed_b200 import http_master as hm  # noqa: E402
from comfyui_distributed_b200.nodes import collector  # noqa: E402

pytestmark = pytest.mark.gpu
MODES = {"L": 1, "LA": 2, "RGB": 3, "RGBA": 4}


def _steps():
    """(depth, the largest row bytes at that depth) for every ring depth the kernel uses up to the row limit."""
    out, lo = [], 1
    while lo <= nat.PNG_MAX_ROW_BYTES:
        d = nat.png_decode_warps(lo)
        a, b = lo, nat.PNG_MAX_ROW_BYTES          # the last row bytes with depth d
        while a < b:
            m = (a + b + 1) // 2
            if nat.png_decode_warps(m) == d:
                a = m
            else:
                b = m - 1
        out.append((d, a))
        lo = a + 1
    return out


def test_ring_depths():
    steps = _steps()
    assert steps[0][0] == 16 and steps[-1] == (3, 65536)
    assert [d for d, _ in steps] == list(range(16, 2, -1))
    assert nat.png_decode_warps(14336) == 16                           # what the tile master launched before
    with pytest.raises(nat.NativeError):
        nat.png_decode_warps(65537)


def test_decode_on_both_sides_of_every_depth_step():
    files = []
    for k, (d, last) in enumerate(_steps()):
        mode = list(MODES)[k % 4]
        C = MODES[mode]
        for w in (last // C, last // C + 1):          # the widest row at depth d, and one pixel more
            if w * C <= nat.PNG_MAX_ROW_BYTES:
                files.append(png_of(image(mode, d + 3, w, k * 7 + w), (k + w) % 2))
    files.append(png_of(image("RGBA", 5, 16384, 1), 0))
    files.append(png_of(image("RGBA", 7, 16384, 2), 1))
    infos = [hm.parse_png(f) for f in files]
    models = [hm.unfilter_model(i, f) for i, f in zip(infos, files)]
    depths = set()
    for f, info, want in zip(files, infos, models):   # one launch per file: each picks its own depth
        depths.add(nat.png_decode_warps(info.W * info.C))
        n = info.H * info.W * 3
        got = decode_on_gpu([f], [0], n + 16)[:n].reshape(want.shape)
        assert np.array_equal(got, want), (info.W, info.C)
    assert depths == set(range(3, 17))
    offs, cur = [], 16
    for info in infos:
        offs.append(cur)
        cur += (info.H * info.W * 3 + 15) // 16 * 16
    out = decode_on_gpu(files, offs, cur + 16)        # all in one launch: the widest row sets the depth (3)
    for o, want in zip(offs, models):
        assert np.array_equal(out[o: o + want.size].reshape(want.shape), want)


@pytest.mark.parametrize("where", ["pinned", "device"])
@pytest.mark.parametrize("H,W,head", [(17, 15, 0), (33, 41, 3), (9, 7, 1)])
def test_gather_unpack(where, H, W, head):
    """81 frames holding every byte value, scattered over two device buffers, into one fp32 result after `head`
    floats of something else (so the frames land at every alignment)."""
    n, e = 81, H * W * 3
    rng = np.random.default_rng(H * W + head)
    frames = rng.integers(0, 256, (n, e), dtype=np.uint8)
    frames.reshape(-1)[:256] = np.arange(256, dtype=np.uint8)          # every byte value
    bufs = [torch.from_numpy(frames[: n // 2].copy()).cuda(), torch.from_numpy(frames[n // 2:].copy()).cuda()]
    ptrs = [bufs[0].data_ptr() + i * e for i in range(n // 2)] + [bufs[1].data_ptr() + i * e for i in range(n - n // 2)]
    total = head + n * e + 5
    dst = (torch.full((total,), -1.0, pin_memory=True) if where == "pinned"
           else torch.full((total,), -1.0, device="cuda"))
    d_ptrs = torch.tensor(ptrs, dtype=torch.int64).cuda()
    nat.gather_unpack_f32(d_ptrs.data_ptr(), n, e, dst.data_ptr() + 4 * head, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    got = dst.cpu().numpy()
    assert (got[:head] == -1).all() and (got[head + n * e:] == -1).all()
    want = frames.astype(np.float32) / np.float32(255)
    assert np.array_equal(got[head: head + n * e].reshape(n, e), want)
    assert np.array_equal(got[head: head + 256], orc.dequantize_u8(np.arange(256, dtype=np.uint8)))


# --------------------------------------------------------------------------------------
# whole jobs
# --------------------------------------------------------------------------------------
def _x(seed, B, H, W, dtype=torch.float32, device="cpu"):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand((B, H, W, 3), generator=g) * 1.02 - 0.01).to(dtype).to(device)


def fleet(master, w1, w2, delegate_only=False, audio=(None, None, None)):
    """w1: the reference's worker (send_batch_to_master); w2: this package's worker on the GPU; both post to this
    package's master node.  Then the reference's master gets the same POSTs.  -> (ours, reference's, node)."""
    enabled = ["w1", "w2"]
    with Ours() as ours, collector_master.Master(keep_bodies=False) as refw:
        node = collector.DistributedCollectorNode()
        out = {}

        def go():
            out["r"] = node.run(master, audio=audio[0], multi_job_id=JOB, enabled_worker_ids=json.dumps(enabled),
                                delegate_only=delegate_only)
        t = threading.Thread(target=go)
        t.start()
        if w1 is not None:
            ref_node = refw.collector.DistributedCollectorNode()
            refw._call(ref_node.send_batch_to_master(w1, audio[1], JOB, ours.url, "w1"), timeout=600)
        if w2 is not None:
            collector.DistributedCollectorNode().run(w2, audio=audio[2], multi_job_id=JOB, is_worker=True,
                                                     master_url=ours.url, worker_id="w2")
        t.join(600)
        assert not t.is_alive() and "r" in out
        bodies = list(ours.bodies)
    want = ref_master(master, enabled, bodies, audio=audio[0], delegate_only=delegate_only)
    return out["r"], want, node


@pytest.mark.timeout(900)
@pytest.mark.parametrize("B,H,W", [(1, 544, 544), (4, 300, 420), (81, 720, 1280), (1, 24, 4800)])
def test_mixed_fleet(B, H, W):
    master = _x(1, 1, H, W)
    w1, w2 = _x(2, B, H, W), _x(3, B, H, W, device="cuda")
    aud = [{"waveform": torch.rand(1, 2, 100 + i, generator=torch.Generator().manual_seed(i)), "sample_rate": 44100 + i}
           for i in range(3)]
    got, want, node = fleet(master, w1, w2, audio=tuple(aud))
    same_result(got, want)
    assert got[0].shape == (1 + 2 * B, H, W, 3) and got[0].dtype == torch.float32 and not got[0].is_cuda
    assert np.array_equal(got[0].numpy(), orc.collector_combine(master.numpy(), {"w1": w1.numpy(),
                                                                                  "w2": w2.cpu().numpy()}, ["w1", "w2"]))
    assert node.last_stats["order"] == ["w1", "w2"] and node.last_stats["decode_launches"] >= 1


@pytest.mark.parametrize("variant", ["delegate", "fp16_cuda", "cuda", "fp16"])
def test_master_variants(variant):
    master = _x(4, 2, 64, 96, dtype=torch.float16 if "fp16" in variant else torch.float32,
                device="cuda" if "cuda" in variant else "cpu")
    got, want, _ = fleet(master, _x(5, 2, 64, 96), _x(6, 3, 64, 96, device="cuda"), delegate_only=variant == "delegate")
    same_result(got, want)


def test_worker_without_is_last_times_out(monkeypatch):
    monkeypatch.setenv("COMFYUI_HEARTBEAT_TIMEOUT", "1")
    master = _x(7, 1, 40, 56)
    posts = [body("w1", 0, png_of(image("RGB", 40, 56, 1), 0), False),
             body("w1", 1, png_of(image("RGB", 40, 56, 2), 1), False),
             body("w2", 0, png_of(image("RGB", 40, 56, 3), 0), True)]
    got = _run_direct(master, ["w1", "w2"], posts)
    assert got[0].shape[0] == 4
    same_result(got, ref_master(master, ["w1", "w2"], posts, timeout=1))


def test_mismatched_sizes_fall_back():
    master = _x(8, 1, 40, 56)
    posts = [body("w1", 0, png_of(image("RGB", 40, 57, 1), 0), True)]
    got = _run_direct(master, ["w1"], posts)
    assert got[0] is master
    same_result(got, ref_master(master, ["w1"], posts))


def test_out_of_order_and_duplicate_batch_idx():
    master = _x(9, 2, 40, 56, device="cuda")
    p = lambda s, lv: png_of(image("RGB", 40, 56, s), lv)
    posts = [body("w2", 3, p(1, 0), False), body("w1", 2, p(2, 1), False), body("w2", 0, p(3, 1), False),
             body("w1", 0, p(4, 0), False), body("w2", 3, p(5, 0), False), body("w1", 2, p(6, 0), True),
             body("w2", 1, p(7, 1), True)]
    got = _run_direct(master, ["w1", "w2"], posts)
    assert got[0].shape[0] == 2 + 5
    same_result(got, ref_master(master, ["w1", "w2"], posts))


def _run_direct(master, enabled, posts):
    with Ours() as ours:
        out = {}
        t = threading.Thread(target=lambda: out.update(r=collector.DistributedCollectorNode().run(
            master, multi_job_id=JOB, enabled_worker_ids=json.dumps(enabled))))
        t.start()
        for raw in posts:
            assert post(ours.url, raw)[0] == 200
        t.join(120)
        assert "r" in out
        return out["r"]
