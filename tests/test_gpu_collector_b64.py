"""The collector master's job_complete checks on the device (csrc/usdu_b64.cu, http_collector.DeviceChecks): the kernel's
verdict and bytes against this interpreter's b64decode(validate=True), its table against the numpy model, the live
route against the host path for every envelope, whole jobs against the reference's master, the loop left free during
the device wait, and the device buffer pool's bound."""
import asyncio
import base64
import json
import threading

import numpy as np
import pytest
import torch

import b64_model as bm
from test_gpu_collector_master import _x, fleet
from test_http_collector import JOB, Ours, _free_port, _route_table, body, data_url, post
from test_http_master import _corruptions, image, png_of

import usdu_oracle as orc

hc, nat = bm.hc, bm.nat
pytestmark = pytest.mark.gpu


def run_kernel(text: bytes):
    """-> (table, decoded bytes) of usdu_b64_png_check on `text` from pinned memory."""
    n = len(text)
    pinned = torch.zeros((n + 15) // 16 * 16 or 16, dtype=torch.uint8, pin_memory=True)
    pinned.numpy()[:n] = np.frombuffer(text, np.uint8)
    out = torch.empty(max(16, nat.b64_png_bytes(n)), dtype=torch.uint8, device="cuda")
    tab = torch.empty(nat.B64_TABLE_WORDS, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream()
    nat.b64_png_check(pinned.data_ptr(), n, out.data_ptr(), tab.data_ptr(), s.cuda_stream)
    torch.cuda.synchronize()
    t = tab.cpu().numpy()
    m = int(t[3])
    return t, out[:max(m, 0)].cpu().numpy().tobytes()


def test_kernel_on_the_corpus():
    for name, text in bm.corpus():
        if isinstance(text, str):
            try:
                text = text.encode("ascii")
            except UnicodeEncodeError:
                continue                          # the route refuses it before the kernel
        want = bm.interpreter(text)
        t, got = run_kernel(text)
        assert (int(t[3]) >= 0) == (want is not None), name
        if want is not None:
            assert got == want, name
        assert np.array_equal(bm.used_words(t), bm.used_words(bm.table_model(text)[0])), name


@pytest.mark.parametrize("mode,h,w", [("RGBA", 2160, 3840), ("RGB", 2160, 3840), ("RGB", 720, 1280)])
def test_kernel_on_whole_frames(mode, h, w):
    rng = np.random.default_rng(h + w)
    a = rng.integers(0, 256, (h, w, 4 if mode == "RGBA" else 3), dtype=np.uint8)
    data = png_of(a, 0)
    text = base64.b64encode(data)
    t, got = run_kernel(text)
    assert got == data
    assert np.array_equal(bm.used_words(t), bm.used_words(bm.table_model(text)[0]))
    info = hc.check_png_tables(t, len(data))
    ref = hc.parse_png(data)
    assert (info.W, info.H, info.C, info.segs, info.idat, info.trailer) == \
        (ref.W, ref.H, ref.C, ref.segs, ref.idat, ref.trailer)
    # the corruptions of a frame this size: the same reason as parse_png
    for name, bad in _corruptions(data)[:6]:
        t, _ = run_kernel(base64.b64encode(bad))
        try:
            hc.parse_png(bad)
            want = None
        except ValueError as e:
            want = str(e)
        try:
            hc.check_png_tables(t, int(t[3]))
            got = None
        except hc.HostParse:
            continue
        except ValueError as e:
            got = str(e)
        assert got == want, name


class HostRoutes:
    """http_collector's routes with the host path, on the loop of `ours`, a store of their own."""

    def __init__(self, ours):
        from aiohttp import web
        self.store = hc.CollectorStore()
        routes = web.RouteTableDef()
        hc.register(routes, self.store, ours.loop, checks=False)
        app = web.Application(client_max_size=1 << 30)
        app.add_routes(routes)
        self.runner = web.AppRunner(app)
        ours.call(self.runner.setup())
        self.port = _free_port()
        ours.call(web.TCPSite(self.runner, "127.0.0.1", self.port).start())
        self.url = f"http://127.0.0.1:{self.port}"
        self.ours = ours

    def close(self):
        self.ours.call(self.runner.cleanup())


def _envelopes():
    rows = [raw for _, raw, _ in _route_table()]
    j = lambda img: json.dumps({"job_id": JOB, "worker_id": "w1", "batch_idx": 0, "image": img,
                                "is_last": False}).encode()
    for name, text in bm.corpus():
        t = text if isinstance(text, str) else text.decode("latin-1")
        rows += [j(t), j("data:image/png;base64," + t)]
    for mode, h, w, level in (("RGB", 544, 544, 0), ("RGBA", 37, 70, 0), ("L", 53, 1, 0), ("RGB", 37, 70, 6)):
        data = png_of(image(mode, h, w, 5), level)
        rows += [j(data_url(data))] + [j(data_url(bad)) for _, bad in _corruptions(data)]
    return rows


def test_route_answers_as_the_host_path(monkeypatch):
    monkeypatch.setattr(hc, "JOB_INIT_GRACE_PERIOD", 0.2)
    with Ours() as ours:
        host = HostRoutes(ours)
        try:
            assert hc.device_checks() is not None
            before = dict(hc.device_checks().stats)
            for url in (ours.url, host.url):
                assert post(url, json.dumps({"multi_job_id": JOB}).encode(), "/distributed/prepare_job")[0] == 200
            rows = _envelopes()
            for raw in rows:
                assert post(ours.url, raw) == post(host.url, raw), raw[:200]
            assert hc.device_checks().stats["device"] > before["device"]
            mine = ours.call(hc.STORE.drain(JOB))
            theirs = ours.call(host.store.drain(JOB))
            assert len(mine) == len(theirs) > 10
            for a, b in zip(mine, theirs):
                assert a["png"] == b["png"]
                assert vars_of(a["info"]) == vars_of(b["info"])
        finally:
            host.close()


def vars_of(info):
    return (info.W, info.H, info.C, info.segs, info.inflated, info.idat, info.trailer)


@pytest.mark.timeout(900)
def test_master_4k_frame_equals_the_reference():
    H, W = 2160, 3840
    master = _x(11, 1, H, W)
    w1, w2 = _x(12, 1, H, W), _x(13, 1, H, W, device="cuda")
    got, want, node = fleet(master, w1, w2)
    assert torch.equal(got[0], want[0])
    assert np.array_equal(got[0].numpy(), orc.collector_combine(master.numpy(), {"w1": w1.numpy(),
                                                                                  "w2": w2.cpu().numpy()}, ["w1", "w2"]))
    assert node.last_stats["device_frames"] == 2


@pytest.mark.timeout(900)
def test_master_720p_81_frames_device_path():
    master = _x(14, 1, 720, 1280)
    w1, w2 = _x(16, 1, 720, 1280), _x(15, 81, 720, 1280, device="cuda")
    checks = hc.device_checks(torch.device("cuda", torch.cuda.current_device()))
    before = checks.stats["device"]
    got, want, node = fleet(master, w1, w2)
    assert torch.equal(got[0], want[0]) and got[0].shape[0] == 83
    assert node.last_stats["device_frames"] == 82
    assert checks.stats["device"] - before == 82          # checked on the master's device


def test_loop_is_free_while_the_device_checks(monkeypatch):
    """While one 4K POST's device checks have not finished (its stream is held behind a spin kernel), prepare_job is
    answered."""
    data = png_of(np.random.default_rng(3).integers(0, 256, (2160, 3840, 3), dtype=np.uint8), 0)
    raw = body("w1", 0, data, True)
    checks = hc.device_checks()
    waiting = threading.Event()
    seen = {}
    real = hc.device_wait

    async def watched(event):
        seen["event"] = event
        waiting.set()
        await real(event)

    monkeypatch.setattr(hc, "device_wait", watched)
    with Ours() as ours:
        assert post(ours.url, json.dumps({"multi_job_id": JOB}).encode(), "/distributed/prepare_job")[0] == 200
        with torch.cuda.stream(checks.stream):
            torch.cuda._sleep(4_000_000_000)           # about 2 s of the route stream, ahead of the POST's kernels
        res = {}
        t = threading.Thread(target=lambda: res.update(r=post(ours.url, raw)))
        t.start()
        assert waiting.wait(120)
        assert post(ours.url, json.dumps({"multi_job_id": "other"}).encode(), "/distributed/prepare_job") == \
            (200, {"status": "success"})
        assert not seen["event"].query() and "r" not in res     # answered while the checks were still on the device
        t.join(120)
        assert res["r"] == (200, {"status": "success"})


def _host_answers(monkeypatch, raws):
    with Ours() as ours:
        host = HostRoutes(ours)
        try:
            for url in (ours.url, host.url):
                assert post(url, json.dumps({"multi_job_id": JOB}).encode(), "/distributed/prepare_job")[0] == 200
            for raw in raws:
                assert post(ours.url, raw) == post(host.url, raw), raw[:200]
            mine, theirs = ours.call(hc.STORE.drain(JOB)), ours.call(host.store.drain(JOB))
            assert len(mine) == len(theirs) and all(a["png"] == b["png"] for a, b in zip(mine, theirs))
            return mine
        finally:
            host.close()


def _oom_bodies():
    good = png_of(image("RGB", 40, 56, 7), 0)
    bad = _corruptions(good)
    return [body("w1", 0, good, False)] + [body("w1", 1, b, False) for _, b in bad[:4]] + \
        [json.dumps({"job_id": JOB, "worker_id": "w1", "batch_idx": 2, "image": "QU=D", "is_last": False}).encode()]


def test_device_out_of_memory_takes_the_host_path(monkeypatch):
    checks = hc.device_checks()

    def full(*a, **k):
        raise torch.OutOfMemoryError("CUDA out of memory (test)")
    monkeypatch.setattr(checks.pool, "take", full)
    before = dict(checks.stats)
    raws = _oom_bodies()
    items = _host_answers(monkeypatch, raws)
    assert checks.stats["device"] == before["device"] and checks.stats["host"] - before["host"] == len(raws)
    assert items and not any(isinstance(it["png"], hc.DevicePng) for it in items)


def test_table_out_of_memory_takes_the_host_path(monkeypatch):
    checks = hc.device_checks()
    real = torch.empty

    def empty(*a, **k):
        if k.get("dtype") == torch.int64 and k.get("device") is not None:
            raise torch.OutOfMemoryError("CUDA out of memory (test)")
        return real(*a, **k)
    monkeypatch.setattr(torch, "empty", empty)
    before = dict(checks.stats)
    raws = _oom_bodies()
    _host_answers(monkeypatch, raws)
    assert checks.stats["device"] == before["device"] and checks.stats["host"] - before["host"] == len(raws)
    monkeypatch.undo()
    import gc
    gc.collect()
    assert checks.pool.used == 0


def test_refusals_deep_in_long_texts():
    """A bad byte, a '=' followed by data and short padding far into a 4K frame's text: the verdict's reductions across
    warps, CTAs and grid-stride iterations."""
    data = png_of(np.random.default_rng(9).integers(0, 256, (2160, 3840, 3), dtype=np.uint8), 0)
    text = bytearray(base64.b64encode(data))
    n = len(text)
    assert n > 8 * 1056 * 256 * 16 // 2               # several grid-stride iterations on an H100
    cases = []
    for at in (n - 1, n - 17, n // 2 + 5, 5_000_001, 20_000_003, 4_325_377, 31 * 4096 + 7):
        for v in (b"$", b"=", b" ", b"\x80"):
            t = bytearray(text)
            t[at:at + 1] = v
            cases.append(bytes(t))
    cases += [bytes(text[:-1]), bytes(text[:n // 2]) + b"=" + bytes(text[n // 2:]), bytes(text) + b"=", bytes(text) + b"A"]
    for t in cases:
        want = bm.interpreter(t)
        tab, got = run_kernel(t)
        assert (int(tab[3]) >= 0) == (want is not None)
        if want is not None:
            assert got == want
        bad, first, end, _ = bm.b64_words(t)
        assert (int(tab[0]), int(tab[1]), int(tab[2])) == (int(bad), first, end)


def test_pool_bound_falls_back_to_the_host_path(monkeypatch):
    checks = hc.device_checks()
    pngs = [u8(s) for s in range(5)]
    nbytes = max(16, nat.b64_png_bytes(len(base64.b64encode(pngs[0]))))
    assert {len(p) for p in pngs} == {len(pngs[0])}
    monkeypatch.setattr(checks, "pool", hc.DevicePool(2 * nbytes + nbytes // 2))     # room for two
    with Ours() as ours:
        assert post(ours.url, json.dumps({"multi_job_id": JOB}).encode(), "/distributed/prepare_job")[0] == 200
        before = dict(checks.stats)
        for i, p in enumerate(pngs):
            assert post(ours.url, body("w1", i, p, False))[0] == 200
        assert checks.stats["device"] - before["device"] == 2 and checks.stats["host"] - before["host"] == 3
        assert checks.pool.used <= checks.pool.limit
        items = ours.call(hc.STORE.drain(JOB))
        assert [it["png"] == p for it, p in zip(items, pngs)] == [True] * 5
        assert sum(isinstance(it["png"], hc.DevicePng) for it in items) == 2
        del items
    import gc
    gc.collect()
    assert checks.pool.used == 0


def u8(seed):
    return png_of(image("RGB", 64, 96, seed), 0)
