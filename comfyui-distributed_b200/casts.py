"""The reference's float -> u8 cast for tensors that are not fp32.

The reference casts every image, sampler output and mask to bytes with numpy's ``(255 * arr).astype(np.uint8)``
(utils/image.py:10, utils/usdu_utils.py:17).  The multiply rounds in the array's own dtype, and numpy's cast on x86
(cvttss2si / cvttsd2si, then the low byte) gives ``trunc(p) & 255`` for a product -2^31 <= p < 2^31 and 0 for NaN,
+-inf and every product outside that range.  The kernels apply this rule to fp32 (csrc/usdu_common.cuh quant_u8).
For fp16 and fp64 the product has to be rounded in that dtype, so reference_f32 computes the byte here and hands the
kernels the exact fp32 k / 255, which every one of them truncates back to k.
"""
from __future__ import annotations

import numpy as np
import torch

_CODES = torch.from_numpy(np.arange(256, dtype=np.float32) / np.float32(255))     # IEEE k / 255, as the kernels' dequantise
_codes_on = {}


def reference_f32(x: torch.Tensor) -> torch.Tensor:
    """The fp32 tensor (same device and shape) whose truncating u8 cast in the kernels equals the reference's cast of x.

    fp32 comes back as it is, without a copy.  bf16 and any other dtype are converted to fp32 as they are: the
    reference cannot take bf16 at all (``.numpy()`` raises), so there is no byte to match."""
    if x.dtype == torch.float32:
        return x
    if x.dtype not in (torch.float16, torch.float64):
        return x.to(torch.float32)
    p = x * 255
    ok = torch.isfinite(p) & (p >= -2.0 ** 31) & (p < 2.0 ** 31)
    k = torch.where(ok, p, torch.zeros_like(p)).trunc().to(torch.int64) & 255
    codes = _codes_on.get(x.device)
    if codes is None:
        codes = _codes_on[x.device] = _CODES.to(x.device)
    return codes[k]
