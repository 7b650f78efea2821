#!/usr/bin/env python
"""Throughput of the SigLIP 2 NaFlex image front-end (NaFlexPreprocessor, jimm_preproc_run_naflex) on camera frames, and of frames to
embeddings through a SigLIP2-B/16 NaFlex tower.

    python scripts/bench_naflex_frames.py [--frames 256] [--rounds 3] [--hf-frames 24] [--out FILE.json]

Input: --frames seeded photo-like uint8 RGB frames (a low-frequency field plus noise), device-resident, in six camera classes (640x480,
1080p, 4K, 12 MP, 24 MP, 8K by pixel count) at aspect ratios drawn log-uniformly from 1:4 to 4:1; patch 16, max_num_patches 256, fp16.
Timed in turn for --rounds rounds after a warm-up, between CUDA events:
  frontend_one_call   (a) the front-end on all frames in one call;
  frontend_per_image  (b) the same front-end called once per frame;
  frames_to_embeds    (c) encode_image(frames) of a random-init SigLIP2-B/16 NaFlex tower with the front-end attached;
  tower_only          (d) that tower's encode_image on the precomputed pixel_values / spatial_shapes;
  per class           (a) on the frames of each size class alone, with the path the planner gives that class's frames.
Also: (e) transformers' Siglip2ImageProcessorPil on the host CPU for the first --hf-frames frames (frames/s of a host-CPU pipeline, not
a GPU figure); the algorithmic bytes of (a) (frames read + pixel_values written) over its time; the host time of one library call
(planning and enqueueing, the stream not waited for); the card name and power limit, read in the same run.  The one-call output is
asserted equal, bit for bit, to the per-image calls.
"""

from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D, L, P, G, MAX_PATCHES = 768, 12, 16, 16, 256
CLASSES = {"640x480": 640 * 480, "1080p": 1920 * 1080, "4K": 3840 * 2160, "12MP": 4032 * 3024, "24MP": 6000 * 4000, "8K": 7680 * 4320}


def frame_sizes(count: int, seed: int):
    """(class, height, width) of `count` frames: the classes in turn, each at a log-uniform aspect ratio from 1:4 to 4:1."""
    import numpy as np

    rng = np.random.default_rng(seed)
    names = list(CLASSES)
    out = []
    for i in range(count):
        name = names[i % len(names)]
        r = math.exp(rng.uniform(math.log(0.25), math.log(4.0)))  # width / height
        w = max(1, int(round(math.sqrt(CLASSES[name] * r))))
        out.append((name, max(1, CLASSES[name] // w), w))
    return out


def make_frame(h: int, w: int, g):
    """A photo-like uint8 [h, w, 3] frame on the GPU: a bilinearly upsampled coarse field plus noise."""
    import torch
    import torch.nn.functional as F

    coarse = torch.randint(0, 256, (1, 3, max(2, h // 64), max(2, w // 64)), generator=g, device="cuda").float()
    field = F.interpolate(coarse, size=(h, w), mode="bilinear", align_corners=False)[0].permute(1, 2, 0)
    noise = torch.randint(-24, 25, (h, w, 3), generator=g, device="cuda").float()
    return (field + noise).clamp_(0, 255).to(torch.uint8).contiguous()


def timed(fn, steps: int = 1):
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
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--hf-frames", type=int, default=24)
    ap.add_argument("--seed", type=int, default=2026)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    sys.path.insert(0, HERE)
    import numpy as np
    import torch

    from jimm_b200 import Rngs
    from jimm_b200.models import SigLIP
    from jimm_b200.preprocess import BILINEAR, NaFlexPreprocessor, plan

    if not torch.cuda.is_available():
        raise SystemExit("bench_naflex_frames.py needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    sizes = frame_sizes(args.frames, args.seed)
    g = torch.Generator(device="cuda").manual_seed(args.seed)
    frames = [make_frame(h, w, g) for _, h, w in sizes]
    pre = NaFlexPreprocessor(patch_size=P, max_num_patches=MAX_PATCHES)
    dt = torch.float16
    # the text tower is not timed: one small layer keeps the random init short
    model = SigLIP(G * P, L, D, P, 16, 1000, D, D // 64, 1, rngs=Rngs(0), dtype=dt, naflex=True).eval()
    model.set_max_batch(args.frames)
    model.set_preprocessor(pre)
    out = {}

    def one_call():
        out["one"] = pre(frames, dtype=dt)

    def per_image():
        out["per"] = [pre([f], dtype=dt) for f in frames]

    def frames_to_embeds():
        out["emb"] = model.encode_image(frames)

    r0 = pre(frames, dtype=dt)
    pv, ss = r0["pixel_values"], r0["spatial_shapes"]

    def tower_only():
        out["tower"] = model.encode_image(pv, spatial_shapes=ss)

    by_class = {}
    for k, (name, _, _) in enumerate(sizes):
        by_class.setdefault(name, []).append(k)
    class_fns = {name: (lambda ks=ks: pre([frames[k] for k in ks], dtype=dt)) for name, ks in by_class.items()}
    variants = {"frontend_one_call": one_call, "frontend_per_image": per_image, "frames_to_embeds": frames_to_embeds, "tower_only": tower_only}
    variants.update({f"class_{n}": fn for n, fn in class_fns.items()})
    for fn in variants.values():  # warms up every shape each variant runs
        fn()
    torch.cuda.synchronize()
    assert torch.equal(out["one"]["pixel_values"], torch.cat([r["pixel_values"] for r in out["per"]])), "one call differs from per-image calls"
    assert torch.equal(out["emb"], out["tower"]), "frames -> embeddings differs from the tower on the front-end's pixel_values"
    runs = {k: [] for k in variants}
    for _ in range(args.rounds):
        for k, fn in variants.items():
            runs[k].append(timed(fn))

    # host time of one library call: planning + enqueue, the stream not waited for
    B = len(frames)
    ptrs = (C.c_void_p * B)(*[f.data_ptr() for f in frames])
    Hs, Ws = (C.c_int * B)(*[f.shape[0] for f in frames]), (C.c_int * B)(*[f.shape[1] for f in frames])
    host = []
    for _ in range(5):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        rc = pre.lib.jimm_preproc_run_naflex(pre.handle, ptrs, B, Hs, Ws, MAX_PATCHES, C.c_void_p(pv.data_ptr()), 1, None, None,
                                             C.c_void_p(torch.cuda.current_stream().cuda_stream))
        host.append(time.perf_counter() - t0)
        assert rc == 0
    torch.cuda.synchronize()

    paths = {}
    for name, ks in by_class.items():
        seen = set()
        for k in ks:
            _, h, w = sizes[k]
            gh, gw = pre.grid(h, w)
            path, tier, ty, _ = plan(h, w, size={"height": gh * P, "width": gw * P}, resample=BILINEAR)
            seen.add("two-pass" if path == 1 else f"fused tier {tier} TY {ty}")
        paths[name] = sorted(seen)

    # (e) the host processor on the first frames (host-CPU figure)
    hf = None
    try:
        from PIL import Image
        from transformers import Siglip2ImageProcessorPil

        proc = Siglip2ImageProcessorPil(patch_size=P, max_num_patches=MAX_PATCHES)
        pil = [Image.fromarray(f.cpu().numpy()) for f in frames[: args.hf_frames]]
        t0 = time.perf_counter()
        proc(images=pil, return_tensors="np")
        hf = round(len(pil) / (time.perf_counter() - t0), 1)
    except ImportError:
        pass

    in_bytes = sum(f.numel() for f in frames)
    out_bytes = pv.numel() * pv.element_size()
    best = min(runs["frontend_one_call"])
    res = dict(device=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip(), frames=B, patch=P, max_num_patches=MAX_PATCHES,
               dtype="float16", frame_bytes=in_bytes, pixel_values_bytes=out_bytes, rounds=args.rounds,
               frames_per_sec={k: [round(B / t, 1) for t in v] for k, v in runs.items() if not k.startswith("class_")},
               frontend_one_call_ms=[round(t * 1e3, 3) for t in runs["frontend_one_call"]],
               frontend_one_call_algorithmic_GBps=round((in_bytes + out_bytes) / best / 1e9, 1),
               host_ms_per_call=round(min(host) * 1e3, 3),
               classes={n: dict(frames=len(ks), ms=[round(t * 1e3, 3) for t in runs[f"class_{n}"]], paths=paths[n]) for n, ks in by_class.items()},
               hf_processor_host_cpu_frames_per_sec=hf, hf_frames=min(args.hf_frames, B))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
