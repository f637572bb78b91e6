"""The reference's float -> u8 cast, `(255 * arr).astype(np.uint8)` (utils/image.py:10), as the tests check it.

ref_u8 is numpy's literal operation.  model_u8 restates its rule with torch integer ops so that expected bytes can be
computed on the GPU next to the kernels: for the product p = 255 * x rounded in x's dtype, trunc(p) & 255 when p is
finite and -2^31 <= p < 2^31, else 0 (x86 cvttss2si / cvttsd2si return 0x80000000 there).  torch's own
.to(torch.uint8) is not a reference: out of range it does not do what numpy does.  tests/test_u8_cast_model.py pins
model_u8 to ref_u8 on the host."""
import numpy as np
import torch

SPECIAL_BITS = [
    0x00000000, 0x80000000,                                   # +-0
    0x00000001, 0x80000001, 0x00000002, 0x007FFFFF, 0x807FFFFF, 0x00400000, 0x80400000,   # denormals
    0x00800000, 0x80800000,                                   # +-FLT_MIN
    0x7F800000, 0xFF800000,                                   # +-inf
    0x7FC00000, 0xFFC00000, 0x7FFFFFFF, 0xFFFFFFFF,           # quiet NaNs
    0x7F800001, 0xFF800001, 0x7FBFFFFF, 0xFFBFFFFF,           # signalling NaNs
    0x7F7FFFFF, 0xFF7FFFFF,                                   # +-FLT_MAX
]
SPECIAL_VALUES = [1.0, 1.004, 1.01, 2.0, -0.01, -0.001, 1e10, -1e10, 8.42e6, -8.42e6, 0.5, 1.0 / 255, 254.0 / 255]


def ref_u8(x) -> np.ndarray:
    """numpy's cast, multiplying in the input's own dtype."""
    x = np.asarray(x)
    with np.errstate(over="ignore", invalid="ignore"):
        return (255 * x).astype(np.uint8)


def model_u8(p: torch.Tensor) -> torch.Tensor:
    """u8 bytes of the products p (already rounded in the input's dtype), on p's device."""
    ok = torch.isfinite(p) & (p >= -2.0 ** 31) & (p < 2.0 ** 31)
    return (torch.where(ok, p, torch.zeros_like(p)).trunc().to(torch.int64) & 255).to(torch.uint8)


def model_u8_of(x: torch.Tensor) -> torch.Tensor:
    return model_u8(x * 255)


def bits_to_f32(bits) -> np.ndarray:
    return np.asarray(bits, dtype=np.int64).astype(np.uint32).view(np.float32)


def special_f32() -> np.ndarray:
    return np.concatenate([bits_to_f32(SPECIAL_BITS), np.asarray(SPECIAL_VALUES, dtype=np.float32)])


def edge_f32(seed: int = 0) -> np.ndarray:
    """fp32 inputs where a cast goes wrong, if it does: every (sign, exponent) with edge and seeded mantissas, +-4 ulp
    around every x where fl(255 x) crosses an integer in [-300, 300], +-64 ulp around 255 x = +-2^24 and +-2^31, and the
    special values."""
    rng = np.random.default_rng(seed)
    se = np.arange(512, dtype=np.int64)[:, None] << 23
    mant = np.concatenate([[0, 1, 2, 3, 0x3FFFFF, 0x400000, 0x400001, 0x7FFFFD, 0x7FFFFE, 0x7FFFFF],
                           rng.integers(0, 1 << 23, 16)])[None, :]
    out = [bits_to_f32((se | mant).ravel())]
    with np.errstate(over="ignore"):
        centres = np.concatenate([np.arange(-300, 301) / 255.0, np.array([2.0 ** 24, -2.0 ** 24, 2.0 ** 31, -2.0 ** 31]) / 255.0])
    c = centres.astype(np.float32).view(np.uint32).astype(np.int64)
    near = np.concatenate([(c[:601, None] + np.arange(-4, 5)[None]).ravel(), (c[601:, None] + np.arange(-64, 65)[None]).ravel()])
    out.append(bits_to_f32(near[(near & 0x7FFFFFFF) < 0x7F800000]))     # (the steps around 0 stay finite)
    out.append(special_f32())
    return np.concatenate(out)


def seeded_f32(seed: int, n: int) -> np.ndarray:
    """n seeded random fp32 bit patterns."""
    return np.random.default_rng(seed).integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32)


class WildSampler:
    """A deterministic elementwise test sampler whose output leaves [0, 1]: 1.25 x - 0.1 (each op rounded in fp32,
    nothing clamped), then NaN, +-inf, +-1e10 and values just above 1 and just below 0 at fixed in-tile positions
    (corners and centre, so that some of them land where the blend mask is opaque).  `dtype` is the dtype it returns.
    The same callable drives the CUDA engine (device tensors), the oracle and the reference (CPU tensors)."""
    cuda_graph_safe = True
    VALUES = [float("nan"), float("inf"), float("-inf"), 1e10, -1e10, 1.0 + 1.0 / 255, 1.01, 2.0, -0.001, -0.01, 1.004]

    def __init__(self, dtype=torch.float32):
        self.dtype = dtype
        self.graph_key = ("wild", str(dtype))

    def __call__(self, x: torch.Tensor, rows=None) -> torch.Tensor:
        y = torch.sub(torch.mul(x, 1.25), 0.1)
        h, w = y.shape[-3], y.shape[-2]
        for i, v in enumerate(self.VALUES):
            for r, c in ((i % h, (3 * i) % w), (h // 2 + i % (h - h // 2), w // 2 + (2 * i) % (w - w // 2))):
                y[..., r, c, i % 3] = v
        return y.to(self.dtype)

    def numpy(self):
        """The oracle's DenoiseFn of the same sampler."""
        return lambda tile, t: self(torch.from_numpy(np.ascontiguousarray(tile))).numpy()
