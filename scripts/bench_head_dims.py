#!/usr/bin/env python
"""Throughput of attention at head widths other than 64, and of the models that need them (H100).

    python scripts/bench_head_dims.py [--iters 300] [--out FILE.json]

(a) The flash attention kernel alone (jimm_k_attention_hd, fp16 in / fp16 out), CUDA events over --iters launches after a warm-up, at
    a fixed model width: S = 257, D = 1280 (20 heads of 64 against ViT-H/14's 16 heads of 80) and S = 64, D = 1152 (18 heads of 64
    against SigLIP so400m text's 16 heads of 72); plus 8 heads of 128 at each width where it divides.  Reported: useful TFLOP/s
    4 B H S^2 d / t and padded TFLOP/s with the padded width DP the kernel computes at.
(b) End to end, fp16, random init, inputs resident on the device: ViT-H/14 @224 (32 layers, batch 128), images/s; the SigLIP so400m
    notebook model (batch 256 images + 256 texts of 64 tokens), pairs/s.

Prints one JSON object (and writes it to --out); the card name and power limit are read in the same run.
"""

from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def padded(d: int) -> int:
    """attention.cu padded_head_dim."""
    return next(p for p in (16, 32, 64, 80, 96, 128) if d <= p)


def device_line() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return dict(device=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip())


def time_cuda(fn, iters: int, warmup: int = 20) -> float:
    """Seconds per call: CUDA events around `iters` back-to-back calls after `warmup` calls."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3 / iters


def attention_kernel(lib, iters: int) -> list:
    rows = []
    for S, D, B in ((257, 1280, 64), (64, 1152, 256)):
        for d in (64, 80, 72, 128):
            if D % d:
                continue
            H = D // d
            g = torch.Generator(device="cpu").manual_seed(d)
            qkv = torch.randn(B * S, 3 * D, generator=g).half().cuda()
            out = torch.empty(B * S, D, dtype=torch.float16, device="cuda")
            s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
            args = (C.c_void_p(qkv.data_ptr()), 1, C.c_void_p(out.data_ptr()), 1, B, S, H, d, 0, 0, s)
            assert lib.jimm_k_attention_hd(*args) == 0, lib.jimm_last_error()
            t = time_cuda(lambda: lib.jimm_k_attention_hd(*args), iters)
            flop = 4.0 * B * H * S * S * d
            rows.append(dict(S=S, D=D, B=B, H=H, d=d, DP=padded(d), us=t * 1e6, useful_tflops=flop / t / 1e12,
                             padded_tflops=flop * padded(d) / d / t / 1e12))
    for r in rows:  # the padding bound: d / DP of the d = 64 useful rate at the same (S, D)
        base = next(x for x in rows if x["S"] == r["S"] and x["d"] == 64)["useful_tflops"]
        r["bound_tflops"] = base * r["d"] / r["DP"]
        r["of_bound"] = r["useful_tflops"] / r["bound_tflops"]
    return rows


def end_to_end(steps: int) -> list:
    from jimm_b200.common.vit import VisionTransformerBase
    from jimm_b200.models import SigLIP

    res = []
    torch.manual_seed(0)
    B = 128
    m = VisionTransformerBase(img_size=224, patch_size=14, in_channels=3, hidden_size=1280, num_layers=32, num_heads=16, mlp_dim=5120,
                              pooling_type="CLS", layernorm_epsilon=1e-6, dtype=torch.float16)
    img = torch.randn(B, 224, 224, 3, device="cuda")
    t = time_cuda(lambda: m(img), steps, warmup=3)
    res.append(dict(model="ViT-H/14 @224, 32 layers, fp16", batch=B, ms=t * 1e3, images_per_s=B / t))
    del m
    B = 256
    m = SigLIP(image_resolution=224, vision_layers=27, vision_width=1152, vision_patch_size=14, context_length=64, vocab_size=32000,
               transformer_width=1152, transformer_heads=16, transformer_layers=27, dtype=torch.float16)
    img = torch.randn(B, 224, 224, 3, device="cuda")
    txt = torch.randint(1, 31999, (B, 64), device="cuda", dtype=torch.int32)
    t = time_cuda(lambda: m(img, txt), steps, warmup=3)
    res.append(dict(model="SigLIP so400m notebook (27+27 layers, 1152 wide, text heads of 72), fp16", batch=B, ms=t * 1e3, pairs_per_s=B / t))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=300)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_head_dims: no CUDA device")
    from jimm_b200 import _lib

    lib = _lib.load()
    r = dict(device_line(), attention=attention_kernel(lib, a.iters), end_to_end=end_to_end(a.steps))
    s = json.dumps(r, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
