"""Synthetic canvases shared by the golden generator and the tests (values k/255 fp32)."""
import numpy as np
import torch


def make_input(kind: str, seed: int, B: int, H: int, W: int) -> np.ndarray:
    if kind == "noise":
        g = torch.Generator().manual_seed(seed)
        x = torch.rand(B, H, W, 3, generator=g)
        return (torch.floor(x * 255) / 255).numpy().astype(np.float32)
    if kind == "smooth":
        g = torch.Generator().manual_seed(seed)
        yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
        base = np.stack([xx / max(W - 1, 1), yy / max(H - 1, 1), (xx + yy) / max(W + H - 2, 1)], -1)
        n = torch.rand(B, H, W, 3, generator=g).numpy() * 0.1
        v = np.clip(base[None] * 0.9 + n, 0, 1)
        return (np.floor(v * 255) / 255).astype(np.float32)
    if kind == "checker":
        yy, xx = np.mgrid[0:H, 0:W]
        c = (((xx // 3) + (yy // 5)) % 2).astype(np.float32)
        img = np.stack([c, 1 - c, c], -1)[None].repeat(B, 0)
        return img.astype(np.float32)
    raise ValueError(kind)


def make_mask(kind: str, seed: int, B: int, H: int, W: int) -> np.ndarray:
    """Conditioning masks fp32 [B, H, W] in [0, 1] (NOT pre-quantised: the truncating cast is part
    of what is tested)."""
    g = torch.Generator().manual_seed(seed)
    if kind == "noise":
        return torch.rand(B, H, W, generator=g).numpy().astype(np.float32)
    if kind == "blob":
        yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
        out = []
        for b in range(B):
            cx, cy = (0.3 + 0.2 * b) * W, (0.6 - 0.1 * b) * H
            r = np.sqrt((xx - cx) ** 2 + (yy - cy) ** 2) / (0.35 * max(W, H))
            out.append(np.clip(1.2 - r, 0, 1) * (0.9 + 0.1 * torch.rand(H, W, generator=g).numpy()))
        return np.stack(out).astype(np.float32)
    raise ValueError(kind)


# (name, kind, seed, B, (Hm, Wm), region, canvas (W, H), tile (pw, ph)) -- shared by oracle/gen_golden.py and the tests
MASK_CROP_CASES = [
    ("pad_v", "noise", 1, 2, (96, 64), (10, 20, 170, 150), (300, 260), (160, 136)),
    ("interior_1080p", "blob", 2, 1, (135, 240), (480, 440, 1056, 1016), (1920, 1080), (544, 544)),
    ("corner_pad_v", "noise", 3, 1, (64, 64), (0, 0, 300, 200), (512, 512), (304, 208)),
    ("pad_h", "blob", 4, 2, (200, 100), (100, 37, 413, 260), (700, 500), (320, 224)),
    ("tall_pad_h", "noise", 5, 1, (50, 50), (20, 10, 180, 300), (200, 320), (256, 256)),
    ("last_tile_downscale", "noise", 6, 1, (300, 260), (724, 524, 1300, 1100), (1300, 1100), (544, 544)),
    ("mask_is_canvas", "blob", 7, 1, (1100, 1300), (0, 0, 544, 544), (1300, 1100), (544, 544)),
    ("upsample_tile", "noise", 8, 1, (90, 160), (992, 512, 1280, 800), (1280, 800), (544, 544)),
]


# (name, kind, seed, B, H, W, tile, padding, blur, uniform, n_workers, denoise seed, denoise) -- multi-worker jobs run
# through the REAL reference's HTTP static mode by oracle/gen_golden.py (oracle/ref_static_run.py)
STATIC_REF_CASES = [
    ("w1_700x520_t256", "noise", 3, 1, 520, 700, 256, 32, 8, True, 1, 9, 0.5),
    ("w2_1300x1100_t512", "noise", 4, 1, 1100, 1300, 512, 32, 8, True, 2, 11, 0.5),
    ("w1_b5_420x300_t128", "smooth", 5, 5, 300, 420, 128, 16, 8, True, 1, 13, 0.4),
    ("w3_nonuniform_900x640_t256", "noise", 6, 1, 640, 900, 256, 16, 16, False, 3, 15, 0.6),
]


def sweep_cases():
    """Seeded sweep over the node's parameter space on small canvases (tests/test_gpu_sweep.py; the real
    reference's digests for the same cases: tests/golden/sweep_ref_digests.json by oracle/gen_golden.py).
    -> (id, kind, B, H, W, tile_w, tile_h, padding, mask_blur, uniform); input seed = id, T0 seed = 1000 + id,
    denoise = 0.25 + 0.05 * (id % 10)."""
    rng = np.random.default_rng(20260921)
    out = []
    for i in range(40):
        W = int(rng.integers(24, 700))
        H = int(rng.integers(24, 500))
        tw = int(rng.choice([64, 72, 96, 128, 200, 256, 512]))
        th = int(rng.choice([64, 80, 128, 256, 384]))
        pad = int(rng.choice([0, 8, 16, 32, 64, 128]))
        blur = int(rng.choice([0, 1, 4, 8, 16, 40, 97]))
        uniform = bool(rng.integers(0, 2))
        B = int(rng.choice([1, 1, 1, 2, 5]))
        kind = ["noise", "smooth", "checker"][int(rng.integers(0, 3))]
        out.append((i, kind, B, H, W, tw, th, pad, blur, uniform))
    out += [(100, "noise", 1, 64, 48, 512, 512, 32, 8, True),      # canvas << tile: 544 -> 48 needs 68 taps (generic kernels)
            (101, "noise", 1, 37, 1021, 64, 64, 8, 8, True),       # odd width, wide and flat
            (102, "checker", 1, 515, 33, 128, 128, 16, 255, True),  # narrow, blur far larger than the canvas
            (103, "smooth", 17, 96, 120, 64, 64, 16, 8, True)]      # WAN-style 4n+1 frame batch
    return out


def sweep_sampler(i: int):
    return 1000 + i, 0.25 + 0.05 * (i % 10)


# (id, B, H, W, tile_w, tile_h, padding, mask_blur, uniform, whole_job) -- the node's tile / padding / blur range up to its
# limits (tests/test_gpu_wide_range.py).  whole_job: also run end to end; the real reference's digests of those jobs are in
# tests/golden/wide_ref_digests.json (oracle/gen_golden.py gen_wide_digests; input "noise" seed = id, sampler wide_sampler).
WIDE_CASES = [
    (0, 1, 500, 700, 128, 128, 48, 8, True, True),          # tensor-core crop staged with LDG (patch > 48 rows)
    (1, 1, 500, 700, 128, 128, 96, 8, True, True),          # ... with two k-steps (crop down-scale ~1.5)
    (2, 2, 400, 520, 128, 128, 96, 8, True, True),          # ... also from the fp32 image; two-k-step blend, 16-row blocks
    (3, 5, 300, 420, 128, 128, 48, 64, True, False),
    (4, 2, 640, 900, 256, 256, 192, 128, True, True),
    (5, 1, 640, 900, 256, 256, 256, 256, True, False),
    (6, 1, 301, 427, 128, 128, 32, 256, True, True),        # width not a multiple of 4, ramp wider than the tile
    (7, 1, 700, 1000, 256, 384, 96, 64, False, False),
    (8, 1, 1300, 1800, 768, 768, 192, 128, True, True),
    (9, 1, 1600, 2304, 1024, 1024, 64, 64, True, True),
    (10, 1, 1500, 2200, 1024, 1024, 256, 256, False, False),
    (11, 1, 1200, 2200, 2048, 2048, 128, 64, True, False),  # two 2176-px tiles, each nearly the whole canvas
    (12, 1, 2100, 2500, 2048, 2048, 256, 64, False, True),
    (13, 1, 64, 64, 2048, 2048, 256, 8, True, True),        # canvas << tile: 2304 -> 64 back-resize, 4x4 generic blocks
    (14, 1, 80, 48, 2048, 2048, 256, 8, True, False),
    (15, 1, 24, 1024, 2048, 2048, 256, 8, True, False),
    (16, 1, 32, 32, 1024, 1024, 256, 8, True, False),
]


def wide_sampler(i: int):
    return 2000 + i, 0.3 + 0.05 * (i % 8)
