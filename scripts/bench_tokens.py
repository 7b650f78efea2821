#!/usr/bin/env python
"""Cost of per-token hidden states against the pooled calls, and what stopping the encoder early saves.

    python scripts/bench_tokens.py [--rounds 5] [--steps 10] [--out FILE.json]

Models: a CLIP ViT-L/14-336 image tower and a CLIP-L text tower (CLIP(336, 24, 1024, 14, 77, 49408, 768, 12, 12)), fp16, random init
with the reference's distributions as bench.build_model does.  Inputs: B = 64 device-resident images of 336 x 336 and B = 256 device
token rows of T = 77.  Variants, timed in turn for --rounds rounds after every variant has been warmed up, each --steps calls between
CUDA events:
  image  pooled     encode_image
         llava      encode_image_tokens(layers=-2, dtype=fp16): x_23 of 24 blocks, the encoder stopping after block 23
         final      encode_image_tokens(layers=None, dtype=fp16, return_pooled=True): ln_post(x_24) and encode_image's result
  text   pooled     encode_text
         final      encode_text_tokens(layers=None, dtype=fp16, return_pooled=True)
Reported: ms per call of each round and, from each variant's median round, the early exit's time over the pooled call (23 of 24
blocks run: 0.958), the token output's cost over the pooled call, and the tokens_out kernel (jimm_k_tokens_out, fp32 -> fp16 of the image tower's [64 * 577, 1024] residual stream)
in GB/s over the bytes it must move (4 read + 2 written per element).  return_pooled's pooled rows are asserted equal, bit for bit, to
the pooled calls'.  The card name and power limit are read in the same run.
"""

from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def timed(fn, steps: int) -> float:
    """ms per call of fn over `steps` calls between CUDA events."""
    import torch

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    sys.path.insert(0, HERE)
    import torch

    from jimm_b200 import Rngs, _lib
    from jimm_b200.models import CLIP

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    res = dict(device=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip(), rounds=args.rounds, steps=args.steps)
    model = CLIP(336, 24, 1024, 14, 77, 49408, 768, 12, 12, dtype=torch.float16, rngs=Rngs(0))
    g = torch.Generator().manual_seed(0)
    img = torch.randn((64, 336, 336, 3), generator=g).half().cuda()
    ids = torch.randint(1, 49407, (256, 77), generator=g)
    ids[torch.arange(256), torch.randint(1, 77, (256,), generator=g)] = 49407
    ids = ids.cuda()
    out = {}
    variants = {
        "image_pooled": lambda: out.__setitem__("image_pooled", model.encode_image(img)),
        "image_llava": lambda: out.__setitem__("image_llava", model.encode_image_tokens(img, -2, dtype=torch.float16)),
        "image_final": lambda: out.__setitem__("image_final", model.encode_image_tokens(img, None, dtype=torch.float16, return_pooled=True)),
        "text_pooled": lambda: out.__setitem__("text_pooled", model.encode_text(ids)),
        "text_final": lambda: out.__setitem__("text_final", model.encode_text_tokens(ids, None, dtype=torch.float16, return_pooled=True)),
    }
    for fn in variants.values():
        fn()
    torch.cuda.synchronize()
    assert out["image_llava"].shape == (64, 577, 1024) and out["image_final"][0].shape == (64, 577, 1024)
    assert torch.equal(out["image_final"][1], out["image_pooled"]), "return_pooled differs from encode_image"
    assert torch.equal(out["text_final"][1], out["text_pooled"]), "return_pooled differs from encode_text"
    runs = {k: [] for k in variants}
    for _ in range(args.rounds):
        for k, fn in variants.items():
            runs[k].append(timed(fn, args.steps))
    med = {k: sorted(v)[len(v) // 2] for k, v in runs.items()}  # the median round
    res["ms_per_call"] = {k: [round(t, 3) for t in v] for k, v in runs.items()}
    res["image_llava_over_pooled"] = round(med["image_llava"] / med["image_pooled"], 4)
    res["image_final_over_pooled"] = round(med["image_final"] / med["image_pooled"], 4)
    res["text_final_over_pooled"] = round(med["text_final"] / med["text_pooled"], 4)

    # the copy kernel alone on the image tower's residual stream
    lib = _lib.load()
    rows, D = 64 * 577, 1024
    x = torch.randn((rows, D), device="cuda")
    y = torch.empty((rows, D), dtype=torch.float16, device="cuda")
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def copy():
        _lib.check(lib.jimm_k_tokens_out(C.c_void_p(x.data_ptr()), rows, D, C.c_void_p(y.data_ptr()), _lib.F16, s))

    copy()
    torch.cuda.synchronize()
    assert torch.equal(y, x.half())
    ms = min(timed(copy, 50) for _ in range(args.rounds))
    nbytes = rows * D * (4 + 2)
    res["tokens_out"] = dict(rows=rows, D=D, out="fp16", bytes=nbytes, ms=round(ms, 4), gb_per_s=round(nbytes / ms / 1e6, 1))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
