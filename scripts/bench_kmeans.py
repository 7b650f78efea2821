#!/usr/bin/env python
"""Spherical k-means over a gallery index (index.kmeans) against the same loop written with the library's hooks and with torch.

    python scripts/bench_kmeans.py [--rounds 3] [--N 1048576] [--E 768] [--C 1024 16384] [--iters 10] [--out FILE.json]

N rows of width E (default 2^20 x 768) in an index of a 1-layer random-init CLIP, Gaussian and clustered (1000 planted centres plus
noise), with C clusters sampled from seed 0 and at most --iters steps.  For each (data, C):
  * `index.kmeans(C, iters)`: ms per call, the steps it ran (it stops early when an assignment repeats) and ms per step; rows rescored
    per row and step, fallbacks and chunks screened (jimm_search_stats);
  * from one torch.profiler run of a call: the kernel time of the screen GEMM (gemm_wgmma_kernel) and its TFLOP/s on the
    2 rows (C - 256) E FLOP per step it screens, the update kernels' share (kmeans_*), and the rest (assignment: seed block, rescore,
    fallback, merges);
  * the same loop through the hooks: jimm_k_logits at scale 0 in row chunks, top_k(., 1), the fixed-point sums in torch int64 and
    jimm_k_l2_normalize, run for the same number of steps and checked to give the same bits;
  * torch fp32 matmul + argmax + index_add_ + normalize (not bit-equal; for scale) and torch fp16 matmul + argmax (approximate), per step.
Every timing is one warm-up call, then the fastest of --rounds calls, each ended by a synchronise.  The card name and power limit are
read in the same run.
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


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--N", type=int, default=2**20)
    ap.add_argument("--E", type=int, default=768)
    ap.add_argument("--C", type=int, nargs="+", default=[1024, 16384])
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    sys.path.insert(0, HERE)
    import torch
    from torch.profiler import ProfilerActivity, profile

    from jimm_b200 import _lib
    from jimm_b200.models import CLIP
    from jimm_b200.postprocess import top_k

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True)
    res = dict(device=torch.cuda.get_device_name(0), nvidia_smi=smi.stdout.strip(), rounds=args.rounds, runs=[])
    print(json.dumps(dict(device=res["device"], nvidia_smi=res["nvidia_smi"])), flush=True)
    N, E = args.N, args.E
    m = CLIP(32, 1, 64, 16, 8, 64, E, E // 64, 1, dtype=torch.float16)
    lib = _lib.load()
    st = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    zero = torch.zeros(1, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(0)

    def timed(fn, rounds):
        fn()
        torch.cuda.synchronize()
        best = math.inf
        for _ in range(rounds):
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            best = min(best, time.perf_counter() - t0)
        return best * 1e3

    def normalize(x):
        out = torch.empty_like(x)
        _lib.check(lib.jimm_k_l2_normalize(p(x), p(out), E, x.shape[0], E, st()))
        return out

    def hook_assign(x, c):
        Cn = c.shape[0]
        step = max(1, (1 << 28) // Cn)
        a = torch.empty(x.shape[0], dtype=torch.int32, device="cuda")
        s = torch.empty(x.shape[0], device="cuda")
        for r0 in range(0, x.shape[0], step):
            r = min(step, x.shape[0] - r0)
            out = torch.empty((r, Cn), device="cuda")
            _lib.check(lib.jimm_k_logits(p(x[r0:]), p(c), p(zero), None, p(out), r, Cn, E, Cn, st()))
            v, i = top_k(out, 1)
            a[r0:r0 + r], s[r0:r0 + r] = i[:, 0], v[:, 0]
        return a, s

    def hook_loop(x, m0, steps):
        """The definition's loop for exactly `steps` assignment steps (the count index.kmeans ran)."""
        mcur = m0.clone()
        c = normalize(mcur)
        for t in range(steps):
            a, s = hook_assign(x, c)
            if t + 1 == steps:
                return c, a, s
            al = a.long()
            S = torch.zeros((c.shape[0], E), dtype=torch.int64, device="cuda").index_add_(0, al, torch.round(x * 2.0**30).long())
            n = torch.bincount(al, minlength=c.shape[0])
            mn = torch.where((n > 0)[:, None], (S.double() * 2.0**-30 / n.clamp_min(1).double()[:, None]).float(), mcur)
            cn = normalize(mn)
            bad = ~torch.isfinite(cn).all(dim=1)
            mcur, c = torch.where(bad[:, None], mcur, mn), torch.where(bad[:, None], c, cn)

    def torch_fp32_step(x, c):
        a = (x @ c.T).argmax(dim=1)
        s = torch.zeros_like(c).index_add_(0, a, x)
        return torch.nn.functional.normalize(s, dim=1)

    def torch_fp16_step(xh, c):
        return (xh @ c.half().T).argmax(dim=1)

    centres = torch.randn(1000, E, generator=g, device="cuda")
    for kind in ("gaussian", "clustered"):
        if kind == "gaussian":
            raw = torch.randn(N, E, generator=g, device="cuda")
        else:
            raw = centres[torch.randint(0, 1000, (N,), generator=g, device="cuda")] + 0.3 * torch.randn(N, E, generator=g, device="cuda")
        index = m.index(raw)
        x = normalize(raw)
        xh = x.half()
        del raw
        for Cn in args.C:
            km = index.kmeans(Cn, iters=args.iters, seed=0)
            steps = km.iterations
            call_ms = timed(lambda: index.kmeans(Cn, iters=args.iters, seed=0), args.rounds)
            # stats through the C entry point
            outs = [torch.empty((Cn, E), device="cuda"), torch.empty(N, dtype=torch.int32, device="cuda"), torch.empty(N, device="cuda"),
                    torch.empty(Cn, dtype=torch.int64, device="cuda")]
            sst, it = _lib.SearchStats(), C.c_int()
            _lib.check(lib.jimm_index_kmeans(index.handle, Cn, None, None, 0, args.iters, None, *[p(t) for t in outs], C.byref(it),
                                             C.byref(sst), st()))
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                index.kmeans(Cn, iters=args.iters, seed=0)
                torch.cuda.synchronize()
            ev = [e for e in prof.key_averages() if e.device_time_total > 0 and "Memcpy" not in e.key and "Memset" not in e.key]
            total_us = sum(e.device_time_total for e in ev)
            screen_us = sum(e.device_time_total for e in ev if "gemm_wgmma_kernel" in e.key)
            update_us = sum(e.device_time_total for e in ev if "kmeans_" in e.key and "kmeans_keys" not in e.key and "kmeans_gather" not in e.key)
            screen_flop = 2.0 * N * max(Cn - 256, 0) * E * steps
            # the hook loop, same steps, same bits (every row is clusterable here, so the sampled rows follow from N, C and the seed)
            init_rows = _sampled_rows(N, Cn, 0)
            t0 = time.perf_counter()
            hc, ha, hs = hook_loop(x, x[init_rows.cuda()], steps)
            torch.cuda.synchronize()
            hook_ms = (time.perf_counter() - t0) * 1e3
            same = bool(torch.equal(ha, km.assign) and torch.equal(hc.view(torch.int32), km.centroids.view(torch.int32))
                        and torch.equal(hs.view(torch.int32), km.scores.view(torch.int32)))
            c = torch.nn.functional.normalize(x[init_rows.cuda()], dim=1)
            fp32_ms = timed(lambda: torch_fp32_step(x, c), args.rounds)
            fp16_ms = timed(lambda: torch_fp16_step(xh, c), args.rounds)
            out = dict(data=kind, N=N, E=E, C=Cn, iters=args.iters, steps=steps, kmeans_ms=call_ms, kmeans_ms_per_step=call_ms / steps,
                       rows_rescored_per_row_step=sst.rows_rescored / (N * steps), fallbacks=sst.fallbacks, chunks_screened=sst.chunks_screened,
                       kernel_ms=total_us * 1e-3, screen_kernel_ms=screen_us * 1e-3,
                       screen_tflops=screen_flop / (screen_us * 1e-6) / 1e12 if screen_us else None,
                       update_share_of_kernel_time=update_us / total_us if total_us else None,
                       assignment_share_of_kernel_time=1 - update_us / total_us if total_us else None,
                       hook_loop_ms=hook_ms, hook_loop_ms_per_step=hook_ms / steps, hook_loop_bit_equal=same,
                       torch_fp32_ms_per_step=fp32_ms, torch_fp16_assign_ms_per_step=fp16_ms)
            res["runs"].append(out)
            print(json.dumps(out), flush=True)
        index.close()
        del x, xh, index
        torch.cuda.empty_cache()
    out = json.dumps(res, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(out)
    print(out)
    return 0


def _sampled_rows(N: int, Cn: int, seed: int):
    """The rows index.kmeans starts from when every row is clusterable: tests/kmeans_oracle.py's sampling rule."""
    import numpy as np
    import torch

    sys.path.insert(0, os.path.join(HERE, "tests"))
    import kmeans_oracle

    return torch.from_numpy(kmeans_oracle.sample_init(np.arange(N), seed, Cn).astype(np.int64))


if __name__ == "__main__":
    sys.exit(main())
