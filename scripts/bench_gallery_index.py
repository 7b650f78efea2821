#!/usr/bin/env python
"""Cost of the gallery index against one-shot search and torch.

    python scripts/bench_gallery_index.py [--rounds 3] [--window-ms 300] [--Q 5000] [--N 1048576] [--E 768] [--out FILE.json]

Q queries against an index of N rows of width E (default 5000 x 2^20 x 768, the CLIP-L width) through a 1-layer random-init CLIP of
that width, at k = 5 and 100, on two galleries: Gaussian embeddings, and clustered ones (300 centroids plus noise, so that each
query has thousands of near ties).  Compared:
  * `index.search(q, k)` -- the index built once, outside the timed window;
  * `model.search(q, gallery, k)` -- the one-shot exact search, the same bits;
  * torch: normalise, fp32 matmul (TF32 off), torch.topk -- an exact-class answer, not the same bits;
  * torch: normalise, fp16 matmul, torch.topk -- an APPROXIMATE answer (fp16 scores), listed for scale only.
Reported: ms per call (each round a window of CUDA events around as many calls as take about --window-ms, interleaved round by
round), whether index.search gave model.search's bits, the screen's kernel time from a torch.profiler run of one search (the
fp16 gemm_wgmma_kernel launches) with its rate 2 Q N E / time and the share of the 989 TFLOP/s FP16 data-sheet rate, the rows
rescored per query and the fallbacks (jimm_search_stats), and the index's build time and bytes.  The card name and power limit
are read in the same run.
"""

from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FP16_PEAK = 989e12  # H100 SXM data sheet, dense FP16 tensor core


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


def rounds(calls: dict, n_rounds: int, window_ms: float) -> dict:
    """{name: [ms per call of each round]}, the calls warmed up and interleaved round by round."""
    for fn in calls.values():
        fn()
    steps = {name: max(1, int(window_ms / timed(fn, 1))) for name, fn in calls.items()}
    ms = {name: [] for name in calls}
    for _ in range(n_rounds):
        for name, fn in calls.items():
            ms[name].append(timed(fn, steps[name]))
    return ms


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--window-ms", type=float, default=300.0)
    ap.add_argument("--Q", type=int, default=5000)
    ap.add_argument("--N", type=int, default=2**20)
    ap.add_argument("--E", type=int, default=768)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    sys.path.insert(0, HERE)
    import torch
    from torch.profiler import ProfilerActivity, profile

    from jimm_b200 import _lib
    from jimm_b200.models import CLIP

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True)
    res = dict(device=torch.cuda.get_device_name(0), nvidia_smi=smi.stdout.strip(), rounds=args.rounds, window_ms=args.window_ms,
               runs=[])
    Q, N, E = args.Q, args.N, args.E
    m = CLIP(32, 1, 64, 16, 8, 64, E, E // 64, 1, dtype=torch.float16)
    m.set_flat_param("logit_scale", torch.tensor(math.log(100.0)))
    lib = _lib.load()
    scale = m.logit_scale.float().reshape(1).cuda()
    g = torch.Generator(device="cuda").manual_seed(0)
    centroids = torch.randn(300, E, generator=g, device="cuda")

    def gallery(kind, n):
        if kind == "gaussian":
            return torch.randn(n, E, generator=g, device="cuda")
        lab = torch.randint(0, centroids.shape[0], (n,), generator=g, device="cuda")
        return centroids[lab] + 0.3 * torch.randn(n, E, generator=g, device="cuda")

    chunk = 1024  # torch paths: query rows per matmul, a [1024, N] fp32 score block at a time

    def torch_path(qe, ge, k, dtype):
        torch.backends.cuda.matmul.allow_tf32 = False
        a = (qe / torch.linalg.norm(qe, dim=-1, keepdim=True)).to(dtype)
        b = (ge / torch.linalg.norm(ge, dim=-1, keepdim=True)).to(dtype)
        return [torch.topk(scale.exp() * (a[r0:r0 + chunk] @ b.T).float(), k, dim=1) for r0 in range(0, Q, chunk)]

    def stats_of(index, qe, k):
        v = torch.empty((Q, k), device="cuda")
        i = torch.empty((Q, k), dtype=torch.int32, device="cuda")
        st = _lib.SearchStats()
        _lib.check(lib.jimm_index_search(index.handle, C.c_void_p(qe.data_ptr()), Q, k, C.c_void_p(v.data_ptr()), C.c_void_p(i.data_ptr()),
                                         C.byref(st), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        torch.cuda.synchronize()
        return st

    default_tf32 = torch.backends.cuda.matmul.allow_tf32
    flops = 2.0 * Q * N * E
    for kind in ("gaussian", "clustered"):
        ge = gallery(kind, N)
        qe = gallery(kind, Q)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        index = m.index(ge)
        e1.record()
        torch.cuda.synchronize()
        build_ms = e0.elapsed_time(e1)
        for k in (5, 100):
            v, i = index.search(qe, k)
            rv, ri = m.search(qe, ge, k)
            same = bool(torch.equal(i, ri) and torch.equal(v.view(torch.int32), rv.view(torch.int32)))
            st = stats_of(index, qe, k)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                index.search(qe, k)
                torch.cuda.synchronize()
            screen_us = sum(e.device_time_total for e in prof.key_averages() if "gemm_wgmma_kernel" in e.key)
            calls = {"index.search": lambda: index.search(qe, k), "model.search": lambda: m.search(qe, ge, k),
                     "torch fp32 matmul (TF32 off) + topk": lambda: torch_path(qe, ge, k, torch.float32),
                     "torch fp16 matmul + topk (approximate)": lambda: torch_path(qe, ge, k, torch.float16)}
            ms = rounds(calls, args.rounds, args.window_ms)
            torch.backends.cuda.matmul.allow_tf32 = default_tf32
            screen_s = screen_us * 1e-6
            r = dict(data=kind, Q=Q, N=N, E=E, k=k, bit_equal_to_model_search=same, ms=ms,
                     screen_ms=screen_s * 1e3, screen_tflops=flops / screen_s / 1e12 if screen_s else None,
                     screen_share_of_fp16_peak=flops / screen_s / FP16_PEAK if screen_s else None,
                     rows_rescored_per_query=st.rows_rescored / Q, fallbacks=st.fallbacks, chunks_screened=st.chunks_screened,
                     index_build_ms=build_ms, index_bytes=N * (6 * E + 4))
            res["runs"].append(r)
            print(json.dumps(r), flush=True)
        index.close()
        del index, ge, qe
        torch.cuda.empty_cache()
    out = json.dumps(res, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(out)
    print(out)
    return 0


if __name__ == "__main__":
    sys.exit(main())
