#!/usr/bin/env python
"""Throughput of a batch of images of different sizes: one packed call (a list of images, variable-length attention) against one
interpolate_pos_encoding call per distinct size and one call per image.

    python scripts/bench_packed_images.py [--images 256] [--rounds 3] [--steps 2] [--out FILE.json]

Models: ViT-B/16 (with its classifier) and the SigLIP-B/16 image tower (encode_image), fp16, random init (bench.build_model).  Input:
--images device-resident images whose sides are drawn (seeded) from 160 to 512 in steps of 16 with aspect ratios from 1:2 to 2:1.  Each
handle is sized once with set_max_image_size(512, 512) and max_batch = --images, so no call rebuilds it.  Variants, timed in turn for
--rounds rounds after every shape has been warmed up, each run --steps passes over all images between CUDA events:
  packed    one call on the list;
  per_size  one call per distinct size on the stacked images of that size;
  per_image one call per image.
Reported: images/s and model TFLOP/s (FLOPs from each image's token count, computed below).  The packed attention kernel alone is timed
against one launch per image on the same packed qkv (ViT-B/16 shapes).  The packed outputs are asserted equal, bit for bit, to the
per-image outputs.  The card name and power limit are read in the same run.
"""

from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D, M, L, P, HEADS = 768, 3072, 12, 16, 12


def encoder_flops(S: int) -> float:
    """Multiply-adds x 2 of the 12 blocks on S tokens: QKV, Q.K^T, P.V, out-projection, MLP."""
    return L * (2 * S * D * 3 * D + 2 * 2 * S * S * D + 2 * S * D * D + 2 * 2 * S * D * M)


def image_flops(name: str, h: int, w: int) -> float:
    n = (h // P) * (w // P)
    f = 2 * n * P * P * 3 * D
    if name == "vit_b16":
        return f + encoder_flops(n + 1) + 2 * D * 1000
    return f + encoder_flops(n) + 2 * n * D * 2 * D + 2 * 2 * n * D + 2 * D * D + 2 * 2 * D * 4 * D  # SigLIP tower with its MAP head


def sizes(count: int, seed: int):
    import numpy as np

    rng = np.random.default_rng(seed)
    sides = np.arange(160, 513, 16)
    out = []
    while len(out) < count:
        h, w = (int(v) for v in rng.choice(sides, 2))
        if h <= 2 * w and w <= 2 * h:
            out.append((h, w))
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


def attention_alone(hw, rounds: int, reps: int = 20):
    """Packed attention kernel vs one launch per image on the same packed qkv (fp16, ViT-B/16 heads, CLS token)."""
    import numpy as np
    import torch

    from jimm_b200 import _lib

    lib = _lib.load()
    lens = [(h // P) * (w // P) + 1 for h, w in hw]
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    T = int(off[-1])
    qkv = torch.randn((T, 3 * D), device="cuda", dtype=torch.float16)
    out = torch.empty((T, D), device="cuda", dtype=torch.float16)
    off_d = torch.from_numpy(off).cuda()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    hd = D // HEADS

    def packed():
        _lib.check(lib.jimm_k_attention_packed(C.c_void_p(qkv.data_ptr()), _lib.F16, C.c_void_p(out.data_ptr()), _lib.F16,
                                               C.c_void_p(off_d.data_ptr()), len(lens), max(lens), HEADS, hd, 0, st))

    def singles():
        for b, S in enumerate(lens):
            o = int(off[b])
            _lib.check(lib.jimm_k_attention_hd(C.c_void_p(qkv[o].data_ptr()), _lib.F16, C.c_void_p(out[o].data_ptr()), _lib.F16, 1, S, HEADS,
                                               hd, 0, 0, st))

    packed(), singles()
    torch.cuda.synchronize()
    flops = sum(2 * 2 * S * S * D for S in lens)
    res = {"packed": [], "per_image": []}
    for _ in range(rounds):
        for k, fn in (("packed", packed), ("per_image", singles)):
            res[k].append(timed(fn, reps))
    return {k: dict(ms=[round(t * 1e3, 3) for t in v], tflops=[round(flops / t / 1e12, 1) for t in v]) for k, v in res.items()}


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=256)
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
    hw = sizes(args.images, args.seed)
    g = torch.Generator().manual_seed(args.seed)
    imgs = [torch.randn(h, w, 3, generator=g).cuda() for h, w in hw]
    groups = {}
    for i, s in enumerate(hw):
        groups.setdefault(s, []).append(i)
    stacks = {s: torch.stack([imgs[i] for i in idx]) for s, idx in groups.items()}
    res = dict(device=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip(), images=len(hw), distinct_sizes=len(groups),
               tokens=sum((h // P) * (w // P) for h, w in hw), steps=args.steps, rounds=args.rounds, models={})
    for name in ("vit_b16", "siglip_b16"):
        model, _, _ = bench.build_model(name, "float16")
        model.set_max_batch(len(hw)).set_max_image_size(512, 512)
        call = model if name == "vit_b16" else model.encode_image
        out = {}

        def packed():
            out["packed"] = call(imgs, interpolate_pos_encoding=True)

        def per_size():
            for s, idx in groups.items():
                call(stacks[s], interpolate_pos_encoding=True)

        def per_image():
            out["per_image"] = [call(x[None], interpolate_pos_encoding=True) for x in imgs]

        variants = {"packed": packed, "per_size": per_size, "per_image": per_image}
        for fn in variants.values():  # warms up every shape each variant runs
            fn()
        torch.cuda.synchronize()
        assert torch.equal(out["packed"], torch.cat(out["per_image"])), f"{name}: packed rows differ from the per-image calls"
        flops = sum(image_flops(name, h, w) for h, w in hw)
        runs = {k: [] for k in variants}
        for _ in range(args.rounds):
            for k, fn in variants.items():
                runs[k].append(timed(fn, args.steps))
        res["models"][name] = {k: dict(images_per_sec=[round(len(hw) / t, 1) for t in v], model_tflops=[round(flops / t / 1e12, 1) for t in v])
                               for k, v in runs.items()}
        print(json.dumps({name: res["models"][name]}), file=sys.stderr, flush=True)
        del model, call, out
        torch.cuda.empty_cache()
    res["attention_alone"] = attention_alone(hw, args.rounds)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
