#!/usr/bin/env python
"""Throughput of the vision towers at image sizes other than the trained one (interpolate_pos_encoding=True) against the native size.

    python scripts/bench_resolution.py [--rounds 3] [--steps 10] [--warmup 2] [--batch 256] [--out FILE.json]

Points: ViT-B/16 (trained at 224) at 224 and 384; SigLIP-B/16 (trained at 256) image-text pairs at 256, 384 and 512.  fp16, random
init (bench.build_model), device-resident inputs, each handle sized once with set_max_image_size for its largest point so no call
rebuilds it.  Every shape is warmed up; then the points of a model are timed in turn, native first, for --rounds rounds, each run
--steps calls between CUDA events.  Reported per point: images/s (pairs/s for SigLIP), and model TFLOP/s from the FLOP count below.
The card name and power limit are read in the same run.
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# name -> (bench.py workload, trained size, sizes, text tower (T, width, layers) or None)
POINTS = {"vit_b16": ("vit_b16", 224, [224, 384], None), "siglip_b16": ("siglip_b16", 256, [256, 384, 512], (64, 768, 12))}


def encoder_flops(S: int, D: int, M: int, L: int) -> float:
    """Multiply-adds x 2 of L pre-LN blocks on S tokens: QKV, Q.K^T, P.V, out-projection, MLP."""
    return L * (2 * S * D * 3 * D + 2 * 2 * S * S * D + 2 * S * D * D + 2 * 2 * S * D * M)


def image_flops(name: str, size: int) -> float:
    """FLOPs of one image (ViT-B/16 with its classifier) or one image-text pair (SigLIP-B/16, MAP head and text tower)."""
    D, M, L, P = 768, 3072, 12, 16
    n = (size // P) ** 2
    f = 2 * n * P * P * 3 * D
    if name == "vit_b16":
        return f + encoder_flops(n + 1, D, M, L) + 2 * D * 1000
    T, Dt, Lt = POINTS[name][3]
    f += encoder_flops(n, D, M, L) + 2 * n * D * 2 * D + 2 * 2 * n * D + 2 * D * D + 2 * 2 * D * 4 * D  # tower, MAP head
    return f + encoder_flops(T, Dt, 4 * Dt, Lt) + 2 * Dt * Dt  # text tower, projection (the B x B logits are left out)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    sys.path.insert(0, HERE)
    import torch

    import bench

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    B = args.batch
    res = dict(device=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip(), batch=B, steps=args.steps, rounds=args.rounds, points={})
    for name, (wl, native, sizes, text) in POINTS.items():
        model, _, tx = bench.build_model(wl, "float16")
        model.set_max_batch(B).set_max_image_size(max(sizes), max(sizes))
        g = torch.Generator().manual_seed(1234)
        ids = bench.synthetic_tokens(B, tx[0], tx[1], tx[2], seed=4321).to(torch.int32).cuda() if tx else None
        calls = {}
        for s in sizes:
            img = torch.randn(B, s, s, 3, generator=g).cuda()
            interp = s != native
            calls[s] = (lambda x=img, i=interp: model(x, ids, interpolate_pos_encoding=i)) if tx else (lambda x=img, i=interp: model(x, interpolate_pos_encoding=i))
        for fn in calls.values():
            for _ in range(args.warmup):
                fn()
        torch.cuda.synchronize()
        runs = {s: [] for s in sizes}
        for _ in range(args.rounds):
            for s, fn in calls.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                runs[s].append(B * args.steps / (e0.elapsed_time(e1) * 1e-3))
        for s in sizes:
            res["points"][f"{name}@{s}"] = dict(unit="pairs/sec" if tx else "images/sec", native=s == native,
                                                per_sec=[round(r, 1) for r in runs[s]],
                                                model_tflops=[round(r * image_flops(name, s) / 1e12, 1) for r in runs[s]])
            print(json.dumps({f"{name}@{s}": res["points"][f"{name}@{s}"]}), file=sys.stderr, flush=True)
        del model, calls
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
