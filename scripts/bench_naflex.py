#!/usr/bin/env python
"""Throughput of a SigLIP 2 NaFlex image tower on the HF processor's layout: one packed call against one call per image, and against the
cost of HF's padded layout.

    python scripts/bench_naflex.py [--images 256] [--rounds 3] [--steps 2] [--out FILE.json]

Model: a random-init SigLIP2-B/16 NaFlex tower (width 768, 12 layers, a 16 x 16 = 256-row position table, patch 16), fp16.  Input:
--images seeded aspect ratios drawn log-uniformly from 1:4 to 4:1, each given the largest patch grid of that ratio with at most
max_num_patches = 256 patches, as pixel_values [B, 256, 768] with spatial_shapes (padding rows filled with NaN).  Variants, timed in turn
for --rounds rounds after a warm-up, each run --steps passes over all images between CUDA events:
  packed    one encode_image(pixel_values, spatial_shapes=...) call: each image's own tokens, no padding computed;
  per_image one such call per image;
  padded    what HF's padded layout costs: the same tower on every image as 256 tokens, timed as the dense encode_image of 256 x 256
            images (jimm_encode_image).
Reported: images/s per variant and the tokens computed.  The packed outputs are asserted equal, bit for bit, to the per-image outputs.  The
card name and power limit are read in the same run.
"""

from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D, L, P, G, MAX_PATCHES = 768, 12, 16, 16, 256


def grids(count: int, seed: int):
    """(patch rows, patch columns) of `count` seeded aspect ratios from 1:4 to 4:1, at most MAX_PATCHES patches each."""
    import numpy as np

    rng = np.random.default_rng(seed)
    out = []
    for r in np.exp(rng.uniform(math.log(0.25), math.log(4.0), count)):  # r = width / height
        gh = max(1, int(math.sqrt(MAX_PATCHES / r)))
        gw = max(1, min(int(gh * r), MAX_PATCHES // gh))
        out.append((gh, gw))
    return out


def timed(fn, steps: int):
    import torch

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3 / steps


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--seed", type=int, default=2025)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    sys.path.insert(0, HERE)
    import torch

    from jimm_b200 import Rngs
    from jimm_b200.models import SigLIP

    if not torch.cuda.is_available():
        raise SystemExit("bench_naflex.py needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    # the text tower is not timed: one small layer keeps the random init short
    model = SigLIP(G * P, L, D, P, 16, 1000, D, D // 64, 1, rngs=Rngs(0), dtype=torch.float16, naflex=True).eval()
    model.set_max_batch(args.images)
    hw = grids(args.images, args.seed)
    g = torch.Generator().manual_seed(args.seed)
    pv = torch.full((args.images, MAX_PATCHES, P * P * 3), float("nan"))
    for b, (gh, gw) in enumerate(hw):
        pv[b, : gh * gw] = torch.randn((gh * gw, P * P * 3), generator=g)
    pv, shapes = pv.cuda(), torch.tensor(hw, dtype=torch.int64)
    dense = torch.randn((args.images, G * P, G * P, 3), generator=g).cuda()
    out = {}

    def packed():
        out["packed"] = model.encode_image(pv, spatial_shapes=shapes)

    def per_image():
        out["per_image"] = [model.encode_image(pv[b:b + 1, : gh * gw], spatial_shapes=shapes[b:b + 1]) for b, (gh, gw) in enumerate(hw)]

    def padded():
        model.encode_image(dense)

    variants = {"packed": packed, "per_image": per_image, "padded": padded}
    for fn in variants.values():  # warms up every shape each variant runs
        fn()
    torch.cuda.synchronize()
    assert torch.equal(out["packed"], torch.cat(out["per_image"])), "packed rows differ from the per-image calls"
    runs = {k: [] for k in variants}
    for _ in range(args.rounds):
        for k, fn in variants.items():
            runs[k].append(timed(fn, args.steps))
    res = dict(device=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip(), images=len(hw), max_num_patches=MAX_PATCHES,
               tokens=sum(gh * gw for gh, gw in hw), padded_tokens=len(hw) * MAX_PATCHES, steps=args.steps, rounds=args.rounds,
               images_per_sec={k: [round(len(hw) / t, 1) for t in v] for k, v in runs.items()})
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
