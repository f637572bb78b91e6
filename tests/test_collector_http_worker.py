"""DistributedCollector as an HTTP worker of the reference's master (nodes/collector.py:84-119 -> api/job_routes.py:
273-343): the stored-PNG layout of the numpy model (png_model.png_stored_b64, the byte-exact reference of the GPU encoder)
and the node's transport, with that encoder and a CPU cast injected, against the reference's own job_complete route
and collector master (collector_master.Master)."""
import io
import json
import zlib

import numpy as np
import pytest
import torch

import collector_master
import png_model
import ref_collector
import usdu_oracle as orc
from __graft_entry__ import load_package

load_package()
from comfyui_distributed_b200 import http_worker  # noqa: E402
from comfyui_distributed_b200.nodes import collector  # noqa: E402

pytestmark = pytest.mark.skipif(not collector_master.available(), reason="reference bundle (oracle/_ref) not present")
JOB = "job-collect"

# (H, W) per channel count: 1x1, one row, one column, a row length 1 + W*C that divides 65535, rows straddling block
# boundaries (3 blocks), several blocks
SHAPES = [(1, 1), (1, 37), (29, 1), (60, 1000), (200, 333)]
DIVIDING_W = {2: 127, 3: 28, 4: 64}          # 1 + W*C = 255, 85, 257


def _frames(seed, B, H, W, C=3):
    g = torch.Generator().manual_seed(seed)
    return torch.rand((B, H, W, C), generator=g, dtype=torch.float32)


def _cases():
    for C in (2, 3, 4):
        for H, W in SHAPES + [(300, DIVIDING_W[C])]:
            yield C, H, W


def _chunks(png: bytes):
    assert png[:8] == b"\x89PNG\r\n\x1a\n"
    pos, out = 8, []
    while pos < len(png):
        n = int.from_bytes(png[pos:pos + 4], "big")
        kind, data = png[pos + 4:pos + 8], png[pos + 8:pos + 8 + n]
        assert int.from_bytes(png[pos + 8 + n:pos + 12 + n], "big") == zlib.crc32(kind + data)
        out.append((kind, data))
        pos += 12 + n
    return out


@pytest.mark.parametrize("C,H,W", list(_cases()))
def test_oracle_png_decodes_to_the_reference_pixels(C, H, W):
    from PIL import Image
    _, _, image = collector_master.load()
    x = _frames(C * 1000 + H + W, 1, H, W, C)
    frame = orc.quantize_u8(x[0].numpy())
    png = png_model.png_stored(frame)
    with Image.open(io.BytesIO(png)) as im:
        im.load()                                   # PIL checks every chunk's CRC and the zlib stream while decoding
        got = np.array(im)
    want = np.array(image.tensor_to_pil(x, 0))
    assert got.shape == want.shape and np.array_equal(got, want)
    chunks = _chunks(png)
    raw = png_model.png_raw_stream(frame)
    nblk = -(-len(raw) // 65535)
    assert [k for k, _ in chunks] == [b"IHDR"] + [b"IDAT"] * (nblk + 1) + [b"IEND"]
    assert [len(d) for _, d in chunks[1:nblk + 1]] == [2 * (k == 0) + 5 + min(65535, len(raw) - 65535 * k)
                                                      for k in range(nblk)]
    assert zlib.decompress(b"".join(d for k, d in chunks if k == b"IDAT")) == raw
    assert len(png) == 63 + 17 * nblk + H * (1 + W * C)
    assert png_model.png_stored_b64(frame) == __import__("base64").b64encode(png)


def _cpu_pack(images):
    return torch.from_numpy(orc.quantize_u8(images.numpy()))


def _oracle_encode(q):
    return (png_model.png_stored_b64(f) for f in q.numpy())


def _our_node():
    node = collector.DistributedCollectorNode()
    node.pack, node.encode = _cpu_pack, _oracle_encode
    return node


def _audio(seed, samples, rate=22050):
    g = torch.Generator().manual_seed(seed)
    return {"waveform": torch.rand((1, 2, samples), generator=g), "sample_rate": rate}


def _fleet(master_images, workers, delegate_only=False, master_audio=None, worker_timeout=60):
    """workers: [(kind "ours" | "ref", worker id, images, audio)], posted one after another in this order, while the
    reference's master collects.  -> (combined images, combined audio, the bodies the master accepted)."""
    ids = [w[1] for w in workers]
    with collector_master.Master(worker_timeout) as m:
        fut = m.collect(master_images, JOB, ids, audio=master_audio, delegate_only=delegate_only)
        for kind, wid, images, audio in workers:
            if kind == "ours":
                out, out_audio = _our_node().run(images, audio=audio, multi_job_id=JOB, is_worker=True,
                                                 master_url=m.url, worker_id=wid, enabled_worker_ids=json.dumps(ids))
                assert out is images                 # a worker hands its input through (collector.py:239-243)
                assert out_audio is (audio if audio is not None else collector.DistributedCollectorNode.EMPTY_AUDIO)
            else:
                m.worker_send(images, audio, JOB, wid)
        combined, combined_audio = fut.result(300)
        return combined, combined_audio, list(m.received)


def _check_bodies(bodies, job, wid, B, audio):
    """Every check of job_complete's validation (job_routes.py:291-305), plus the order and the audio field."""
    assert len(bodies) == B
    for i, raw in enumerate(bodies):
        d = json.loads(raw)
        assert isinstance(d["job_id"], str) and d["job_id"].strip() == job
        assert isinstance(d["worker_id"], str) and d["worker_id"].strip() == wid
        assert isinstance(d["batch_idx"], int) and not isinstance(d["batch_idx"], bool) and d["batch_idx"] == i
        assert isinstance(d["image"], str) and d["image"].startswith("data:image/png;base64,")
        assert isinstance(d["is_last"], bool) and d["is_last"] == (i == B - 1)
        has_audio = audio is not None and i == B - 1
        assert ("audio" in d) == has_audio
        if has_audio:
            assert isinstance(d["audio"], dict)
            assert d["audio"] == http_worker.encode_audio_payload(audio)


def _same(a, b):
    assert a[0].dtype == b[0].dtype and a[0].shape == b[0].shape and torch.equal(a[0], b[0])
    assert a[1]["sample_rate"] == b[1]["sample_rate"] and torch.equal(a[1]["waveform"], b[1]["waveform"])


@pytest.mark.timeout(300)
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("with_audio", [False, True], ids=["no_audio", "audio"])
def test_node_worker_against_the_reference_master(B, with_audio):
    master = _frames(1, 2, 48, 40)
    imgs = _frames(2 + B, B, 48, 40)
    audio = _audio(7, 300) if with_audio else None
    ours = _fleet(master, [("ours", "w1", imgs, audio)])
    ref = _fleet(master, [("ref", "w1", imgs, audio)])
    _same(ours[:2], ref[:2])
    assert np.array_equal(ours[0].numpy(), orc.collector_combine(master.numpy(), {"w1": imgs.numpy()}, ["w1"]))
    assert torch.equal(ours[0], ref_collector.combine(master, {"w1": imgs}, ["w1"]))
    _check_bodies(ours[2], JOB, "w1", B, audio)


@pytest.mark.timeout(300)
def test_delegate_only_and_two_workers_in_enabled_order():
    """The master contributes nothing; enabled_worker_ids is ["w2", "w1"] (not sorted): w2 is this package's node, w1
    the reference's worker, and the combined batch and audio follow that order."""
    master = _frames(3, 1, 36, 52)
    a, b = _frames(4, 2, 36, 52), _frames(5, 3, 36, 52)
    audio_a, audio_b = _audio(8, 120, 44100), _audio(9, 80, 44100)
    workers = [("ours", "w2", b, audio_b), ("ref", "w1", a, audio_a)]
    ours = _fleet(master, workers, delegate_only=True)
    # enabled order = order of `workers`: w2 first
    assert torch.equal(ours[0], ref_collector.combine(master, {"w2": b, "w1": a}, ["w2", "w1"], delegate_only=True))
    ref = _fleet(master, [("ref", w, x, au) for _, w, x, au in workers], delegate_only=True)
    _same(ours[:2], ref[:2])
    assert ours[0].shape[0] == 5


@pytest.mark.timeout(300)
def test_worker_with_no_images_sends_nothing():
    """B = 0 posts nothing, as the reference's worker; the master gives up on it after its worker timeout and returns
    what the other worker sent."""
    master = _frames(10, 1, 20, 24)
    empty, imgs = torch.zeros((0, 20, 24, 3)), _frames(11, 2, 20, 24)
    ours = _fleet(master, [("ours", "w1", empty, None), ("ref", "w2", imgs, None)], worker_timeout=2)
    ref = _fleet(master, [("ref", "w1", empty, None), ("ref", "w2", imgs, None)], worker_timeout=2)
    _same(ours[:2], ref[:2])
    assert len(ours[2]) == 2 and all(json.loads(b)["worker_id"] == "w2" for b in ours[2])


def test_one_channel_raises_type_error_before_any_request(monkeypatch):
    calls = []
    monkeypatch.setattr(http_worker, "_call", lambda *a, **k: calls.append(a) or (200, b""))
    with pytest.raises(TypeError):
        _our_node().run(_frames(12, 2, 8, 8, 1), multi_job_id=JOB, is_worker=True, master_url="http://127.0.0.1:9",
                        worker_id="w1", enabled_worker_ids='["w1"]')
    with pytest.raises(TypeError):
        png_model.png_stored(orc.quantize_u8(_frames(12, 1, 8, 8, 1)[0].numpy()))
    assert calls == []


def test_audio_over_the_limit_raises_before_any_request(monkeypatch):
    calls = []
    monkeypatch.setattr(http_worker, "_call", lambda *a, **k: calls.append(a) or (200, b""))
    monkeypatch.setenv("COMFYUI_MAX_AUDIO_PAYLOAD_BYTES", "100")
    with pytest.raises(ValueError):
        _our_node().run(_frames(13, 1, 8, 8), audio=_audio(1, 50), multi_job_id=JOB, is_worker=True,
                        master_url="http://127.0.0.1:9", worker_id="w1", enabled_worker_ids='["w1"]')
    assert calls == []


def test_audio_payload_matches_the_reference():
    import sys
    collector_master.load()
    ref_audio = sys.modules[f"{ref_collector.PKG}.utils.audio_payload"]
    for a in (None, {"waveform": torch.zeros(1, 2, 0)}, {"waveform": torch.rand(1, 2, 5, dtype=torch.float64)},
              {"waveform": torch.rand(2, 1, 7), "sample_rate": "bad"}, {"waveform": torch.rand(1, 1, 3), "sample_rate": 8000.7}):
        assert http_worker.encode_audio_payload(a) == ref_audio.encode_audio_payload(a)


@pytest.mark.timeout(120)
def test_master_answering_4xx_makes_the_node_raise():
    """An empty worker id fails job_complete's validation: HTTP 400, which the node raises, with no retry."""
    with collector_master.Master() as m:
        with pytest.raises(http_worker.HttpError) as e:
            _our_node().run(_frames(14, 2, 8, 8), multi_job_id=JOB, is_worker=True, master_url=m.url, worker_id="",
                            enabled_worker_ids='["w1"]')
        assert e.value.status == 400
        assert m.received == []
