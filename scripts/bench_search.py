#!/usr/bin/env python
"""Cost of top-k selection and of gallery search.

    python scripts/bench_search.py [--rounds 3] [--window-ms 300] [--Q 5000] [--N 1048576] [--E 768] [--out FILE.json]

top_k: `top_k` against `zero_shot` (full order) and `classify` (argmax) on [256, 21843] (an ImageNet-21k head), [5000, 25000]
(COCO's images x captions) and [1, 2^20] (one query against a gallery), fp32 randn * 8 on the device, k = 5 and 100.

search: Q queries against N gallery rows of width E (default 5000 x 2^20 x 768, the CLIP-L width) through a 1-layer random-init
CLIP of that width, at k = 5 and 100, against (a) the test-hook path -- jimm_k_l2_normalize + jimm_k_logits over row chunks of the
queries, then top_k of each chunk, the same bits -- and (b) torch: normalise, matmul, torch.topk, with TF32 off (fp32 FMA, the
same arithmetic class) and with torch's default matmul precision.  Search is FMA-bound: its FLOP count is 2 Q N E, reported as
achieved TFLOP/s and as a share of the 67 TFLOP/s FP32 data-sheet rate of the H100 SXM.

Every timing is a window of CUDA events around as many calls as take about --window-ms (at least one), repeated --rounds times;
the spread over rounds is reported.  The card name and power limit are read in the same run.
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
TOPK_SHAPES = [(256, 21843), (5000, 25000), (1, 2**20)]
FP32_PEAK = 67e12  # H100 SXM data sheet, dense FP32


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

    from jimm_b200 import _lib
    from jimm_b200.models import CLIP
    from jimm_b200.postprocess import classify, top_k, zero_shot

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    res = dict(device=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip(), rounds=args.rounds, window_ms=args.window_ms,
               top_k=[], search=[])
    g = torch.Generator(device="cuda").manual_seed(0)
    for rows, cols in TOPK_SHAPES:
        x = torch.randn(rows, cols, generator=g, device="cuda") * 8.0
        calls = {"zero_shot": lambda: zero_shot(x), "classify": lambda: classify(x),
                 "top_k(5)": lambda: top_k(x, 5), "top_k(100)": lambda: top_k(x, 100)}
        ms = rounds(calls, args.rounds, args.window_ms)
        res["top_k"].append(dict(shape=[rows, cols], ms={k: v for k, v in ms.items()}))
        print(json.dumps(res["top_k"][-1]), flush=True)
        del x

    Q, N, E = args.Q, args.N, args.E
    m = CLIP(32, 1, 64, 16, 8, 64, E, E // 64, 1, dtype=torch.float16)
    m.set_flat_param("logit_scale", torch.tensor(math.log(100.0)))
    qe = torch.randn(Q, E, generator=g, device="cuda")
    ge = torch.randn(N, E, generator=g, device="cuda")
    lib = _lib.load()
    scale = m.logit_scale.float().reshape(1).cuda()
    chunk = max(1, (2 << 30) // (4 * N))  # hook path: rows of the score matrix per chunk, 2 GB at a time
    qn, gn = torch.empty_like(qe), torch.empty_like(ge)
    block = torch.empty((chunk, N), device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())

    def hook_path(k):
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        _lib.check(lib.jimm_k_l2_normalize(p(qe), p(qn), E, Q, E, st))
        _lib.check(lib.jimm_k_l2_normalize(p(ge), p(gn), E, N, E, st))
        outs = []
        for r0 in range(0, Q, chunk):
            r = min(chunk, Q - r0)
            _lib.check(lib.jimm_k_logits(C.c_void_p(qn[r0:].data_ptr()), p(gn), p(scale), None, p(block), r, N, E, N, st))
            outs.append(top_k(block[:r], k))
        return outs

    def torch_path(k, tf32):
        torch.backends.cuda.matmul.allow_tf32 = tf32
        a = qe / torch.linalg.norm(qe, dim=-1, keepdim=True)
        b = ge / torch.linalg.norm(ge, dim=-1, keepdim=True)
        outs = []
        for r0 in range(0, Q, chunk):
            outs.append(torch.topk(scale.exp() * (a[r0:r0 + chunk] @ b.T), k, dim=1))
        return outs

    default_tf32 = torch.backends.cuda.matmul.allow_tf32
    flops = 2.0 * Q * N * E
    for k in (5, 100):
        v, i = m.search(qe, ge, k)
        hv, hi = zip(*hook_path(k))
        same = bool(torch.equal(i, torch.cat(hi)) and torch.equal(v.view(torch.int32), torch.cat(hv).view(torch.int32)))
        calls = {"search": lambda: m.search(qe, ge, k), "hook logits chunks + top_k": lambda: hook_path(k),
                 "torch matmul fp32 (TF32 off) + topk": lambda: torch_path(k, False),
                 "torch matmul default + topk": lambda: torch_path(k, default_tf32)}
        ms = rounds(calls, args.rounds, args.window_ms)
        torch.backends.cuda.matmul.allow_tf32 = default_tf32
        best = min(ms["search"])
        res["search"].append(dict(Q=Q, N=N, E=E, k=k, bit_equal_to_hook_path=same, ms=ms, flop=flops,
                                  search_tflops=[flops / t / 1e9 for t in ms["search"]],
                                  search_share_of_fp32_peak=flops / (best * 1e-3) / FP32_PEAK))
        print(json.dumps(res["search"][-1]), flush=True)
    out = json.dumps(res, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(out)
    print(out)
    return 0


if __name__ == "__main__":
    sys.exit(main())
