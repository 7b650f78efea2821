#!/usr/bin/env python
"""Cost of the zero-shot / classification epilogue at real label and caption counts.

    python scripts/bench_postprocess.py [--rounds 5] [--window-ms 300] [--out FILE.json]

Shapes: [1, 21843] and [256, 21843] (an ImageNet-21k head), [5000, 25000] (COCO's images x captions retrieval scores) and
[1, 2^20] (one query against a gallery of 2^20 embeddings); fp32 device-resident logits, randn * 8.  Each shape is warmed up, then
`zero_shot` (probabilities and the full descending order: rows wider than 4096 columns sorted as 4096-key runs merged in global
memory) and `classify` (argmax only: one block reduction per row) are timed in turn for --rounds rounds, each a window of CUDA
events around as many calls as take about --window-ms.  Reported: ms per call and rows x cols per second of every round.  The
card name and power limit are read in the same run.
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(1, 21843), (256, 21843), (5000, 25000), (1, 2**20)]


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
    ap.add_argument("--window-ms", type=float, default=300.0)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    sys.path.insert(0, HERE)
    import torch

    from jimm_b200.postprocess import classify, zero_shot

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    res = dict(device=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip(), rounds=args.rounds, window_ms=args.window_ms, shapes=[])
    g = torch.Generator(device="cuda").manual_seed(0)
    for rows, cols in SHAPES:
        x = torch.randn(rows, cols, generator=g, device="cuda") * 8.0
        calls = {"zero_shot": lambda: zero_shot(x), "classify": lambda: classify(x)}
        for fn in calls.values():
            fn()
        steps = {name: max(1, int(args.window_ms / timed(fn, 3))) for name, fn in calls.items()}
        ms = {name: [] for name in calls}
        for _ in range(args.rounds):
            for name, fn in calls.items():
                ms[name].append(timed(fn, steps[name]))
        entry = dict(rows=rows, cols=cols, steps=steps)
        for name in calls:
            entry[name] = dict(ms=[round(v, 4) for v in ms[name]], elements_per_s=[round(rows * cols / (v * 1e-3)) for v in ms[name]])
        res["shapes"].append(entry)
        print(json.dumps(entry), flush=True)
        del x
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
