#!/usr/bin/env python
"""Cost of the gallery index's threshold search and near-duplicate pairs against torch.

    python scripts/bench_range_search.py [--rounds 3] [--window-ms 300] [--Q 5000] [--N 1048576] [--E 768] [--pairs-N 1048576]
                                         [--out FILE.json]

Through a 1-layer random-init CLIP of width E (default the CLIP-L width 768):
  * `index.range_search(q, t)` of Q queries against an index of N rows (default 5000 x 2^20), at thresholds giving about 10 and about
    1000 hits per query, on Gaussian embeddings and on clustered ones (300 centroids plus noise).  Baseline: torch's fp32 matmul
    (TF32 off) in 1024-query blocks, `>=` and `nonzero` -- an exact-class answer, not the same bits.
  * `index.pairs(t)` on pairs-N clustered rows with 1 % of them planted near-duplicates (a copy of another row plus 1e-3 noise), at a
    threshold just below the planted pairs' scores.  Baseline: a chunked fp16 torch self-join (upper triangle, `>=`, `nonzero`), which
    is APPROXIMATE (fp16 scores) and listed for scale only.
Reported: ms per call (each round a window of CUDA events around as many calls as take about --window-ms, interleaved round by round),
hits, whether range_search and pairs gave the hook matrix's CSR bit for bit (checked outside the timed windows, on a sample of query
rows for range_search), the rows rescored per query and the fallbacks (jimm_search_stats), and the screen's kernel time from a separate
torch.profiler run (the fp16 gemm_wgmma_kernel launches) with its rate and the share of the 989 TFLOP/s FP16 data-sheet rate.  The card
name and power limit are read in the same run.
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
CHUNK = 1024  # torch paths: query rows per matmul


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
    ap.add_argument("--pairs-N", type=int, default=2**20)
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
    cur = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    g = torch.Generator(device="cuda").manual_seed(0)
    centroids = torch.randn(300, E, generator=g, device="cuda")

    def embeddings(kind, n):
        if kind == "gaussian":
            return torch.randn(n, E, generator=g, device="cuda")
        lab = torch.randint(0, centroids.shape[0], (n,), generator=g, device="cuda")
        return centroids[lab] + 0.3 * torch.randn(n, E, generator=g, device="cuda")

    def normalised(x):
        out = torch.empty_like(x)
        for r0 in range(0, x.shape[0], 2**20):
            n = min(2**20, x.shape[0] - r0)
            _lib.check(lib.jimm_k_l2_normalize(p(x[r0:]), p(out[r0:]), E, n, E, cur()))
        return out

    def hook(qn, gn):
        out = torch.empty((qn.shape[0], gn.shape[0]), device="cuda")
        _lib.check(lib.jimm_k_logits(p(qn), p(gn), p(scale), None, p(out), qn.shape[0], gn.shape[0], E, gn.shape[0], cur()))
        return out

    def hook_csr(qn, gn, t, upper=False, row0=0):
        """The hook matrix's CSR >= t for the rows qn (stored rows row0 .. when upper: only columns past the row's own)."""
        counts, scores, idx = [], [], []
        step = max(1, (1 << 28) // gn.shape[0])
        for r0 in range(0, qn.shape[0], step):
            L = hook(qn[r0:r0 + step], gn)
            mask = L >= t
            if upper:
                rows = torch.arange(row0 + r0, row0 + r0 + L.shape[0], device="cuda")
                mask &= torch.arange(gn.shape[0], device="cuda")[None, :] > rows[:, None]
            counts.append(mask.sum(1))
            scores.append(L[mask])
            idx.append(mask.nonzero()[:, 1].to(torch.int32))
        return torch.cat(counts), torch.cat(scores), torch.cat(idx)

    def stats_of(call, *a):
        h = C.c_void_p()
        st = _lib.SearchStats()
        _lib.check(getattr(lib, call)(*a, C.byref(h), C.byref(st), cur()))
        _lib.check(lib.jimm_hits_destroy(h))
        return st

    def screen_time(fn):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        return sum(e.device_time_total for e in prof.key_averages() if "gemm_wgmma_kernel" in e.key) * 1e-6

    def torch_range(qe, ge, t):
        torch.backends.cuda.matmul.allow_tf32 = False
        a = qe / torch.linalg.norm(qe, dim=-1, keepdim=True)
        b = ge / torch.linalg.norm(ge, dim=-1, keepdim=True)
        out = []
        for r0 in range(0, Q, CHUNK):
            s = scale.exp() * (a[r0:r0 + CHUNK] @ b.T)
            mask = s >= t
            out.append((mask.nonzero(), s[mask]))
        return out

    default_tf32 = torch.backends.cuda.matmul.allow_tf32
    for kind in ("gaussian", "clustered"):
        ge, qe = embeddings(kind, N), embeddings(kind, Q)
        index = m.index(ge)
        qn, gn = normalised(qe), normalised(ge)
        sample = hook(qn[:64], gn).flatten().sort(descending=True).values
        for hits in (10, 1000):
            t = sample[hits * 64 - 1].item()
            o, s, i = index.range_search(qe, t)
            rows = torch.linspace(0, Q - 1, 64, device="cuda").long()
            rc, rs, ri = hook_csr(qn[rows], gn, t)
            got_i = torch.cat([i[o[r]:o[r + 1]] for r in rows.tolist()])
            got_s = torch.cat([s[o[r]:o[r + 1]] for r in rows.tolist()])
            same = bool(torch.equal(o.diff()[rows], rc) and torch.equal(got_i, ri) and torch.equal(got_s.view(torch.int32), rs.view(torch.int32)))
            nnz = o[-1].item()
            del o, s, i
            st = stats_of("jimm_index_range_search", index.handle, p(qe), Q, t)
            screen_s = screen_time(lambda: index.range_search(qe, t))
            ms = rounds({"index.range_search": lambda: index.range_search(qe, t),
                         "torch fp32 matmul (TF32 off) + >= + nonzero": lambda: torch_range(qe, ge, t)}, args.rounds, args.window_ms)
            torch.backends.cuda.matmul.allow_tf32 = default_tf32
            flops = 2.0 * Q * N * E
            r = dict(call="range_search", data=kind, Q=Q, N=N, E=E, threshold=t, hits=nnz, hits_per_query=nnz / Q,
                     bit_equal_to_hook_on_64_rows=same, ms=ms, rows_rescored_per_query=st.rows_rescored / Q, fallbacks=st.fallbacks,
                     chunks_screened=st.chunks_screened, screen_ms=screen_s * 1e3,
                     screen_tflops=flops / screen_s / 1e12 if screen_s else None,
                     screen_share_of_fp16_peak=flops / screen_s / FP16_PEAK if screen_s else None)
            res["runs"].append(r)
            print(json.dumps(r), flush=True)
        index.close()
        del index, ge, qe, qn, gn
        torch.cuda.empty_cache()

    # pairs: clustered rows, 1 % of them near-duplicates of another row
    P = args.pairs_N
    ge = embeddings("clustered", P)
    perm = torch.randperm(P, generator=g, device="cuda")
    dup, src = perm[: P // 100], perm[P // 100: 2 * (P // 100)]  # a copied row is never itself overwritten
    ge[dup] = ge[src] + 1e-3 * torch.randn(dup.numel(), E, generator=g, device="cuda")
    index = m.index(ge)
    gn = normalised(ge)
    planted = (hook(gn[dup[:256]], gn).gather(1, src[:256, None])).flatten()
    t = planted.min().item() - 1.0
    i, j, s = index.pairs(t)
    nnz = i.numel()
    rows = torch.linspace(0, P - 1, 64, device="cuda").long()
    same = True
    for r in rows.tolist():  # sampled rows of the upper triangle against the hook matrix
        rc, rs, ri = hook_csr(gn[r:r + 1], gn, t, upper=True, row0=r)
        sel = i == r
        same = same and bool(torch.equal(j[sel], ri) and torch.equal(s[sel].view(torch.int32), rs.view(torch.int32)))
    del i, j, s
    st = stats_of("jimm_index_pairs", index.handle, t)
    screen_s = screen_time(lambda: index.pairs(t))

    def torch_pairs():
        h = gn.half()
        out = []
        for r0 in range(0, P, CHUNK):
            sc = scale.exp() * (h[r0:r0 + CHUNK] @ h[r0:].T).float()
            mask = torch.triu(sc >= t, 1)
            out.append(mask.nonzero())
        return out

    ms = rounds({"index.pairs": lambda: index.pairs(t), "torch fp16 self-join, upper triangle (approximate)": torch_pairs}, args.rounds, args.window_ms)
    # what the screen multiplies: each chunk of 2048 rows against the 65536-row chunks from the one holding its first row on
    flops = sum(2.0 * E * min(2048, P - q0) * (P - q0 // 65536 * 65536) for q0 in range(0, P, 2048))
    r = dict(call="pairs", data="clustered, 1 % planted near-duplicates", N=P, E=E, threshold=t, pairs=nnz, planted=int(dup.numel()),
             bit_equal_to_hook_on_64_rows=same, ms=ms, rows_rescored_per_row=st.rows_rescored / P, fallbacks=st.fallbacks,
             chunks_screened=st.chunks_screened, screen_ms=screen_s * 1e3, screen_flop=flops,
             screen_tflops=flops / screen_s / 1e12 if screen_s else None,
             screen_share_of_fp16_peak=flops / screen_s / FP16_PEAK if screen_s else None)
    res["runs"].append(r)
    print(json.dumps(r), flush=True)
    out = json.dumps(res, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(out)
    print(out)
    return 0


if __name__ == "__main__":
    sys.exit(main())
