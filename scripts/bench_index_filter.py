#!/usr/bin/env python
"""Cost of removed rows and filters on the gallery index.

    python scripts/bench_index_filter.py [--rounds 3] [--window-ms 200] [--Q 5000] [--N 1048576] [--E 768] [--out FILE.json]

Q queries against an index of N rows of width E (default 5000 x 2^20 x 768) through a 1-layer random-init CLIP of that width, at k = 5
and 100, on Gaussian and clustered galleries (300 centroids plus noise, as scripts/bench_gallery_index.py).  Cases: the index with
nothing removed and no filter (the unchanged path, the baseline); one row removed; 10 % removed; filters keeping 50, 10, 1 and 0.1 %
of the rows (random, fixed seed).  For each case, with A the allowed rows:
  * `index.search(q, k[, keep])`, ms per call;
  * `model.search(q, raw[A], k)` -- the one-shot exact search of those rows, the same bits (checked);
  * torch: gather raw[A], normalise, fp16 matmul, torch.topk -- an APPROXIMATE answer, for scale only;
  * rows rescored per query and fallbacks (jimm_search_stats), and from one torch.profiler run of the search the share of its
    kernel time spent listing the allowed rows and gathering them (allowed_*_kernel, gather_rows_kernel).
Each round is a window of CUDA events around as many calls as take about --window-ms, interleaved round by round.  Then
range_search and pairs under the 10 % filter, with the unfiltered range_search for comparison: each warmed up by one call, then the
fastest of --rounds single calls.  The card name and power
limit are read in the same run.
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
sys.path.insert(0, os.path.join(HERE, "scripts"))

from bench_gallery_index import rounds, timed  # noqa: E402


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--window-ms", type=float, default=200.0)
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
               runs=[], range_and_pairs=[])
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

    chunk = 1024

    def torch_fp16(qe, ge, A, k):
        b = ge[A]
        b = (b / torch.linalg.norm(b, dim=-1, keepdim=True)).half()
        a = (qe / torch.linalg.norm(qe, dim=-1, keepdim=True)).half()
        kk = min(k, b.shape[0])
        return [torch.topk(scale.exp() * (a[r0:r0 + chunk] @ b.T).float(), kk, dim=1) for r0 in range(0, Q, chunk)]

    def stats_of(index, qe, k, keep):
        v = torch.empty((Q, k), device="cuda")
        i = torch.empty((Q, k), dtype=torch.int32, device="cuda")
        st = _lib.SearchStats()
        _lib.check(lib.jimm_index_search_keep(index.handle, C.c_void_p(qe.data_ptr()), Q, k,
                                              C.c_void_p(keep.data_ptr()) if keep is not None else None, C.c_void_p(v.data_ptr()),
                                              C.c_void_p(i.data_ptr()), C.byref(st), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        torch.cuda.synchronize()
        return st

    gen = torch.Generator(device="cuda").manual_seed(1)
    for kind in ("gaussian", "clustered"):
        ge = gallery(kind, N)
        qe = gallery(kind, Q)
        r = torch.rand(N, generator=gen, device="cuda")
        base = m.index(ge)
        one = m.index(ge)
        one.remove(N // 2)
        ten = m.index(ge)
        ten.remove((r < 0.1).nonzero().flatten())
        all_rows = torch.arange(N, device="cuda")
        cases = [("baseline", base, None, all_rows), ("1 row removed", one, None, all_rows[all_rows != N // 2]),
                 ("10% removed", ten, None, (r >= 0.1).nonzero().flatten())]
        for p in (0.5, 0.1, 0.01, 0.001):
            keep = r < p
            cases.append((f"filter {p * 100:g}%", base, keep, keep.nonzero().flatten()))
        for k in (5, 100):
            for name, index, keep, A in cases:
                v, i = index.search(qe, k, keep=keep)
                rv, ri = m.search(qe, ge[A], k)
                same = bool(torch.equal(i, A[ri.long()].int()) and torch.equal(v.view(torch.int32), rv.view(torch.int32)))
                st = stats_of(index, qe, k, keep)
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    index.search(qe, k, keep=keep)
                    torch.cuda.synchronize()
                ev = prof.key_averages()
                total_us = sum(e.device_time_total for e in ev if e.device_time_total > 0 and "Memcpy" not in e.key and "Memset" not in e.key)
                gather_us = sum(e.device_time_total for e in ev if "gather_rows_kernel" in e.key or "allowed_" in e.key)
                calls = {"index.search": lambda: index.search(qe, k, keep=keep), "model.search(raw[A])": lambda: m.search(qe, ge[A], k),
                         "torch gather + fp16 matmul + topk (approximate)": lambda: torch_fp16(qe, ge, A, k)}
                ms = rounds(calls, args.rounds, args.window_ms)
                out = dict(data=kind, case=name, Q=Q, N=N, E=E, k=k, allowed=int(A.numel()), bit_equal_to_model_search=same, ms=ms,
                           rows_rescored_per_query=st.rows_rescored / Q, fallbacks=st.fallbacks, chunks_screened=st.chunks_screened,
                           gather_share_of_kernel_time=gather_us / total_us if total_us else None, gather_ms=gather_us * 1e-3)
                res["runs"].append(out)
                print(json.dumps(out), flush=True)
        # range search and pairs under the 10 % filter
        keep = r < 0.1
        t = float(base.search(qe[:256], 100)[0][:, -1].median())
        hits_f = int(base.range_search(qe, t, keep=keep)[0][-1])  # each call once before it is timed
        base.range_search(qe, t)
        rs_f = min(timed(lambda: base.range_search(qe, t, keep=keep), 1) for _ in range(args.rounds))
        rs_u = min(timed(lambda: base.range_search(qe, t), 1) for _ in range(args.rounds))
        sub = keep.nonzero().flatten()
        tp = float(m.search(ge[sub[:256]], ge[sub], 2)[0][:, -1].median())
        npairs = int(base.pairs(tp, keep=keep)[0].numel())
        pr_ms = min(timed(lambda: base.pairs(tp, keep=keep), 1) for _ in range(args.rounds))
        out = dict(data=kind, Q=Q, N=N, E=E, allowed=int(sub.numel()), range_threshold=t, range_search_filtered_ms=rs_f,
                   range_search_unfiltered_ms=rs_u, range_hits_filtered=hits_f, pairs_threshold=tp, pairs_filtered_ms=pr_ms, pairs=npairs)
        res["range_and_pairs"].append(out)
        print(json.dumps(out), flush=True)
        for x in (base, one, ten):
            x.close()
        del base, one, ten, ge, qe
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
