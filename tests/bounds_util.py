"""The per-element check shared by the fp64 bound tests: |out - ref| <= bound at every element, and the output types' rounding
constants the bounds are written in."""

import math

import numpy as np
import torch

from gpu_util import BF16, F16, F32, record_parity

U = 2.0 ** -24  # fp32 unit roundoff
TF32 = 3  # type code 3 of the jimm_k_* entry points: fp32 rounded to tf32
# output type: (torch dtype, type code of the jimm_k_* entry points, unit roundoff, half the smallest subnormal step)
OUT = {"f16": (torch.float16, F16, 2.0 ** -11, 2.0 ** -25), "bf16": (torch.bfloat16, BF16, 2.0 ** -8, 2.0 ** -134),
       "f32": (torch.float32, F32, 2.0 ** -24, 2.0 ** -150), "tf32": (torch.float32, TF32, 2.0 ** -11, 2.0 ** -137)}


def assert_within(case, what, out, ref, bound, dtype="fp32"):
    """Assert |out - ref| <= bound at every element (NaN in out - ref fails); record and return max |out - ref| / bound."""
    out, ref = torch.as_tensor(out).double(), torch.as_tensor(ref).double()
    bound = torch.as_tensor(bound, dtype=torch.float64, device=out.device).expand_as(out)
    err = (out - ref).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    ratio = torch.nan_to_num(ratio, nan=math.inf, posinf=math.inf)
    flat = int(ratio.argmax())
    worst = float(ratio.flatten()[flat])
    record_parity(case, what, dtype, "fp64", 1.0, worst)
    if not worst <= 1.0:
        idx = tuple(int(i) for i in np.unravel_index(flat, tuple(out.shape)))
        o, r, b = (float(t.flatten()[flat]) for t in (out, ref, bound))
        raise AssertionError(f"{case} / {what} [{dtype}]: |out - ref| / bound = {worst:.3g} at {idx}: out={o!r} ref={r!r} bound={b!r}")
    return worst
