#!/usr/bin/env python
"""Throughput of a list of prompts of different lengths through the text tower: one packed call (a list of token sequences,
variable-length causal attention) against the padded [N, context_length] call and one call per distinct length.

    python scripts/bench_packed_text.py [--prompts 4096] [--rounds 3] [--steps 2] [--out FILE.json]

Models: the CLIP-B/32 and SigLIP-B/16 text towers (encode_text), fp16, random init (bench.build_model), at the default max_batch.  Input:
--prompts device-resident prompts whose lengths are drawn (seeded) from 6 to 32 tokens, EOT (the largest id) last.  Variants, timed in
turn for --rounds rounds after every shape has been warmed up, each run --steps passes over all prompts between CUDA events:
  packed      one call on the list;
  padded      one [N, context_length] call on the prompts padded with EOT -- CLIP only: SigLIP pools the last token, so its padded call
              computes something else;
  per_length  one call per distinct length on the stacked prompts of that length.
Reported: prompts/s and text-tower TFLOP/s, the FLOPs counted from each prompt's own token count (below) for every variant, so the
padding a variant computes is not counted as work.  The packed rows are asserted equal, bit for bit, to the padded rows (CLIP) and to
the per-length rows.  The card name and power limit are read in the same run.
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# name: (width, layers, context_length, vocabulary) of the text tower (bench.build_model)
TOWERS = {"clip_b32": (512, 12, 77, 49408), "siglip_b16": (768, 12, 64, 32000)}


def prompt_flops(name: str, S: int) -> float:
    """Multiply-adds x 2 of one prompt of S tokens: per block QKV, Q.K^T and P.V (the full S x S, as the kernel's tiles are counted for the
    images), out-projection and the 4x MLP; then the projection of the pooled row."""
    D, L, _, _ = TOWERS[name]
    return L * (2 * S * D * 3 * D + 2 * 2 * S * S * D + 2 * S * D * D + 2 * 2 * S * D * 4 * D) + 2 * D * D


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
    ap.add_argument("--prompts", type=int, default=4096)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--seed", type=int, default=2024)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    sys.path.insert(0, HERE)
    import torch

    import bench

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    g = torch.Generator().manual_seed(args.seed)
    lens = torch.randint(6, 33, (args.prompts,), generator=g).tolist()
    res = dict(device=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip(), prompts=len(lens), tokens=sum(lens),
               distinct_lengths=len(set(lens)), steps=args.steps, rounds=args.rounds, models={})
    for name in ("clip_b32", "siglip_b16"):
        _, _, T, V = TOWERS[name]
        model, _, _ = bench.build_model(name, "float16")
        eot = V - 1
        seqs = []
        for L in lens:
            s = torch.randint(1, eot, (L,), generator=g)
            s[-1] = eot
            seqs.append(s.cuda())
        padded = torch.full((len(lens), T), eot, dtype=torch.int64)
        for i, s in enumerate(seqs):
            padded[i, :len(s)] = s.cpu()
        padded = padded.cuda()
        groups = {}
        for i, L in enumerate(lens):
            groups.setdefault(L, []).append(i)
        stacks = {L: torch.stack([seqs[i] for i in idx]) for L, idx in groups.items()}
        order = torch.tensor([i for idx in groups.values() for i in idx])
        out = {}

        def packed():
            out["packed"] = model.encode_text(seqs)

        def padded_call():
            out["padded"] = model.encode_text(padded)

        def per_length():
            out["per_length"] = [model.encode_text(stacks[L]) for L in groups]

        variants = {"packed": packed, "per_length": per_length}
        if name == "clip_b32":
            variants["padded"] = padded_call
        for fn in variants.values():  # warms up every shape each variant runs
            fn()
        torch.cuda.synchronize()
        per = torch.empty_like(out["packed"])
        per[order.cuda()] = torch.cat(out["per_length"])
        assert torch.equal(out["packed"], per), f"{name}: packed rows differ from the per-length calls"
        if "padded" in out:
            assert torch.equal(out["packed"], out["padded"]), f"{name}: packed rows differ from the padded call"
        flops = sum(prompt_flops(name, L) for L in lens)
        runs = {k: [] for k in variants}
        for _ in range(args.rounds):
            for k, fn in variants.items():
                runs[k].append(timed(fn, args.steps))
        res["models"][name] = dict(max_batch=model.native().max_batch, context_length=T,
                                   **{k: dict(prompts_per_sec=[round(len(lens) / t, 1) for t in v],
                                              text_tflops=[round(flops / t / 1e12, 1) for t in v]) for k, v in runs.items()})
        print(json.dumps({name: res["models"][name]}), file=sys.stderr, flush=True)
        del model, out, seqs, stacks, padded
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
