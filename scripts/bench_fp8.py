#!/usr/bin/env python
"""End-to-end throughput of the FP8 compute mode (dtype=torch.float8_e4m3fn) against fp16 on the same weights (H100).

    python scripts/bench_fp8.py [--reps 3] [--steps 20] [--warmup 3] [--out FILE.json]

Workloads, at bench.py's batch and model shapes: ViT-B/16 @224 B=256, SigLIP-B/16 @256 B=256 pairs, ViT-L/16 @384 MAP B=128.  Each
model is built twice from one random init (bench.build_model), in fp16 and in FP8; inputs are device resident.  The two modes
alternate --reps times per workload, each run timing --steps forwards between CUDA events after --warmup untimed ones.  Also reported:
max |FP8 - fp16| / max |fp16| of the outputs.  Prints one JSON object (and writes it to --out) with the card name, power limit and max
SM clock read in the same run.
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKLOADS = {"vit_b16": 256, "siglip_b16": 256, "vit_l16_map": 128}


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    sys.path.insert(0, HERE)
    import torch

    import bench

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    res = dict(device=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip(), steps=args.steps, reps=args.reps, workloads={})
    for wl, B in WORKLOADS.items():
        steps = {}
        outs = {}
        for mode in ("float16", "float8_e4m3fn"):
            model, img_size, text = bench.build_model(wl, mode)
            model.set_max_batch(B)
            g = torch.Generator().manual_seed(1234)
            img = torch.randn(B, img_size, img_size, 3, generator=g).cuda()
            if text is not None:
                ids = bench.synthetic_tokens(B, text[0], text[1], text[2], seed=4321).to(torch.int32).cuda()
                steps[mode] = (lambda m=model, x=img, t=ids: m(x, t))
            else:
                steps[mode] = (lambda m=model, x=img: m(x))
        runs = {m: [] for m in steps}
        for _ in range(args.reps):
            for mode, fn in steps.items():
                for _ in range(args.warmup):
                    outs[mode] = fn()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                runs[mode].append(round(B * args.steps / (e0.elapsed_time(e1) * 1e-3), 1))
        a, b = outs["float16"].double(), outs["float8_e4m3fn"].double()
        res["workloads"][wl] = dict(batch=B, unit="pairs/sec" if wl.startswith("siglip") else "images/sec", fp16=runs["float16"],
                                    fp8=runs["float8_e4m3fn"], fp8_beats_fp16_every_rep=all(f > h for f, h in zip(runs["float8_e4m3fn"], runs["float16"])),
                                    mean_speedup=round(sum(runs["float8_e4m3fn"]) / sum(runs["float16"]), 3),
                                    output_rel_diff=float((a - b).abs().max() / a.abs().max()))
        print(json.dumps({wl: res["workloads"][wl]}), file=sys.stderr, flush=True)
        del steps, outs
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
