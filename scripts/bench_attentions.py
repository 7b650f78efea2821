#!/usr/bin/env python
"""Cost of returning attention weights, and the attention-weights (probs) kernel's time and achieved bytes/s.

    python scripts/bench_attentions.py [--rounds 5] [--steps 10] [--out FILE.json]

Workloads, fp16, random init with the reference's distributions (Rngs(0)), device-resident inputs:
  vit    ViT-B/16 @224, B = 64: model(x) against forward_attentions(x, None, dtype=fp16) -- all 12 blocks, [64, 12, 197, 197] each
  clip   CLIP ViT-L/14-336 image tower, B = 64: encode_image against encode_image_attentions(x, -1, dtype=fp16) -- block 23 of 24,
         [64, 16, 577, 577]
Each variant is warmed up, then timed in turn for --rounds rounds of --steps calls between CUDA events (ms per call).  A separate
torch.profiler run of one call per attention variant gives the probs kernel's CUDA time (the sum over its launches) and its achieved
bytes/s over the bytes it must move: B * H * S^2 * 2 written, plus 2 passes x B * S * 2 * D * 2 read (q and k, fp16) per launch.
The card name and power limit are read in the same run.
"""

from __future__ import annotations

import argparse
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


def probs_kernel_ms(fn):
    """(CUDA ms summed over the attn_probs_kernel launches of one call of fn, number of launches), from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if "attn_probs_kernel" in e.name and e.device_type.name == "CUDA"]
    return sum(e.device_time for e in ev) / 1e3, len(ev)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    sys.path.insert(0, HERE)
    import torch

    from jimm_b200 import Rngs
    from jimm_b200.models import CLIP, VisionTransformer

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    res = dict(device=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip(), rounds=args.rounds, steps=args.steps)
    g = torch.Generator().manual_seed(0)
    vit = VisionTransformer(dtype=torch.float16, rngs=Rngs(0))
    clip = CLIP(336, 24, 1024, 14, 77, 49408, 768, 12, 12, dtype=torch.float16, rngs=Rngs(0))
    x224 = torch.randn((64, 224, 224, 3), generator=g).half().cuda()
    x336 = torch.randn((64, 336, 336, 3), generator=g).half().cuda()
    # (B, H, S, D, launches per call) of each attention variant
    shapes = {"vit_attn": (64, 12, 197, 768, 12), "clip_attn": (64, 16, 577, 1024, 1)}
    out = {}
    variants = {
        "vit_pooled": lambda: out.__setitem__("vit_pooled", vit(x224)),
        "vit_attn": lambda: out.__setitem__("vit_attn", vit.forward_attentions(x224, None, dtype=torch.float16)),
        "clip_pooled": lambda: out.__setitem__("clip_pooled", clip.encode_image(x336)),
        "clip_attn": lambda: out.__setitem__("clip_attn", clip.encode_image_attentions(x336, -1, dtype=torch.float16)),
    }
    for fn in variants.values():
        fn(), fn()
    torch.cuda.synchronize()
    assert len(out["vit_attn"]) == 12 and out["vit_attn"][0].shape == (64, 12, 197, 197)
    assert out["clip_attn"].shape == (64, 16, 577, 577)
    for k in ("vit_attn", "clip_attn"):  # every row of weights sums to 1
        w = out[k][-1] if isinstance(out[k], tuple) else out[k]
        assert torch.allclose(w.float().sum(-1), torch.ones(1, device="cuda"), atol=2e-2), k
    runs = {k: [] for k in variants}
    for _ in range(args.rounds):
        for k, fn in variants.items():
            runs[k].append(timed(fn, args.steps))
    med = {k: sorted(v)[len(v) // 2] for k, v in runs.items()}  # the median round
    res["ms_per_call"] = {k: [round(t, 3) for t in v] for k, v in runs.items()}
    res["vit_attn_over_pooled"] = round(med["vit_attn"] / med["vit_pooled"], 3)
    res["clip_attn_over_pooled"] = round(med["clip_attn"] / med["clip_pooled"], 3)
    for k, (B, H, S, D, launches) in shapes.items():
        ms, n = probs_kernel_ms(variants[k])
        assert n == launches, (k, n)
        nbytes = launches * (B * H * S * S * 2 + 2 * B * S * 2 * D * 2)
        res[f"{k}_probs_kernel"] = dict(launches=n, ms=round(ms, 4), bytes=nbytes, gb_per_s=round(nbytes / ms / 1e6, 1))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
