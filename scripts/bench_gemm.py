#!/usr/bin/env python
"""Each encoder GEMM of the benchmark workloads timed alone, and the L2 -> shared-memory fill ceiling (H100).

    python scripts/bench_gemm.py [--root DIR] [--iters 50] [--out FILE.json]

(a) The four GEMMs of one encoder layer of vit_b16, siglip_b16 (vision tower) and vit_l16_map at the benchmark's batch, token count,
    width and operand type, with their epilogues: QKV (operand-type store), FC1 (+ tanh-GELU, operand-type store), and out-projection /
    FC2 as the fp32 residual reduce-add with the fused LayerNorm (jimm_k_gemm_residual_ln).  QKV and FC1 are also timed as the FP8
    compute mode runs them (e4m3 operands with row scales, fp16 output; rows "qkv e4m3" / "fc1+gelu e4m3", with their speed-up over the
    16-bit row).  CUDA events over --iters launches after a warm-up.  Reported: TFLOP/s, and the bytes the CTAs fill from L2 into shared
    memory per FLOP with the library's tile shape.
(b) jimm_k_l2_probe: TMA fills of 16 KB stages from an L2-resident buffer on every SM, mode 0 (each CTA its own tiles) and mode 2 with
    2-CTA clusters (each CTA loads half a tile and multicasts it to both).  Reported: bytes landed in shared memory per second.

--root picks the repository tree whose built library is timed (default: this one).  Prints one JSON object (and writes it to --out);
the card name, power limit and max SM clock are read in the same run.
"""

from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# workload: (batch, tokens per image, width, MLP width, operand dtype) as bench.py runs them
SHAPES = {
    "vit_b16": (256, 197, 768, 3072, "float16"),
    "siglip_b16": (256, 256, 768, 3072, "float16"),
    "vit_l16_map": (128, 576, 1024, 4096, "bfloat16"),
}


def device_line(torch) -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return dict(device=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip())


def tile_shape(root: str) -> tuple:
    """GEMM_TILE_M x GEMM_TILE_N from the tree's gemm.cuh (trees from before the shape was exported there used 128 x 128)."""
    src = open(os.path.join(root, "jimm_b200", "csrc", "gemm.cuh")).read()
    m, n = re.search(r"GEMM_TILE_M = (\d+)", src), re.search(r"GEMM_TILE_N = (\d+)", src)
    return (int(m.group(1)), int(n.group(1))) if m and n else (128, 128)


def time_cuda(torch, fn, iters: int, warmup: int = 10) -> float:
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


def gemms(torch, lib, tile, iters: int) -> list:
    vp = lambda t: None if t is None else C.c_void_p(t.data_ptr())  # noqa: E731
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    rows = []
    for wl, (B, S, D, F, dn) in SHAPES.items():
        dt = getattr(torch, dn)
        code = {torch.float16: 1, torch.bfloat16: 2}[dt]
        M = B * S
        g = torch.Generator(device="cuda").manual_seed(0)
        a_big = torch.randn(M, F, device="cuda", generator=g).to(dt)
        x = torch.randn(M, D, device="cuda", generator=g)
        h = torch.empty(M, D, device="cuda", dtype=dt)
        out = torch.empty(M, 3 * D if 3 * D > F else F, device="cuda", dtype=dt)
        scale, lbias = torch.ones(D, device="cuda"), torch.zeros(D, device="cuda")
        cnt = torch.zeros(M // 32 + 2, dtype=torch.int32, device="cuda")
        for name, N, K, kind in (("qkv", 3 * D, D, "store"), ("out_proj+ln", D, D, "residual_ln"), ("fc1+gelu", F, D, "gelu"),
                                 ("fc2+ln", D, F, "residual_ln")):
            A = a_big[:, :K]
            W = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).to(dt)
            bias = torch.zeros(N, device="cuda")
            if kind == "residual_ln":
                def fn(A=A, W=W, N=N, K=K, bias=bias):
                    rc = lib.jimm_k_gemm_residual_ln(code, vp(A), A.stride(0), vp(W), K, M, N, K, vp(bias), vp(x), D, vp(scale), vp(lbias),
                                                     1e-6, vp(h), code, D, vp(cnt), s)
                    assert rc == 0, lib.jimm_last_error().decode()
            else:
                act = 1 if kind == "gelu" else 0

                def fn(A=A, W=W, N=N, K=K, bias=bias, act=act):
                    rc = lib.jimm_k_gemm_ex(0, code, vp(A), A.stride(0), vp(W), K, M, N, K, vp(bias), act, None, None, 0, vp(out), code,
                                            out.stride(0), 0, 0, 0, 2, M, 0, 0, 0, 0, None, None, 0.0, None, 0, 0, None, s)
                    assert rc == 0, lib.jimm_last_error().decode()
            t = time_cuda(torch, fn, iters)
            flop = 2.0 * M * N * K
            BM, BN = tile
            BK = 64  # 128 B of 16-bit K per stage
            fill = math.ceil(M / BM) * math.ceil(N / BN) * math.ceil(K / BK) * (BM + BN) * 128
            rows.append(dict(workload=wl, gemm=name, M=M, N=N, K=K, dtype=dn, us=round(t * 1e6, 1), tflops=round(flop / t / 1e12, 1),
                             l2_fill_bytes_per_flop=round(fill / flop, 5), l2_fill_tb_s=round(fill / t / 1e12, 2)))
            print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
            if kind in ("store", "gelu"):  # the FP8 mode's form of QKV / FC1: e4m3 operands (128 K elements per stage), fp16 output
                A8 = torch.randn(M, K, device="cuda", generator=g).to(torch.float8_e4m3fn).view(torch.uint8)
                W8 = torch.randn(N, K, device="cuda", generator=g).to(torch.float8_e4m3fn).view(torch.uint8)
                sa, sb = torch.full((M,), 2.0 ** -4, device="cuda"), torch.full((N,), 1.0 / math.sqrt(K), device="cuda")
                out16 = out if dt == torch.float16 else torch.empty(out.shape, device="cuda", dtype=torch.float16)

                def fn8(N=N, K=K, bias=bias, act=act):
                    rc = lib.jimm_k_gemm_e4m3(0, vp(A8), K, vp(W8), K, M, N, K, vp(sa), vp(sb), vp(bias), act, vp(out16), 1, out16.stride(0),
                                              2, M, 0, s)
                    assert rc == 0, lib.jimm_last_error().decode()

                t8 = time_cuda(torch, fn8, iters)
                fill8 = math.ceil(M / BM) * math.ceil(N / BN) * math.ceil(K / 128) * (BM + BN) * 128
                rows.append(dict(workload=wl, gemm=name + " e4m3", M=M, N=N, K=K, dtype="float8_e4m3fn", us=round(t8 * 1e6, 1),
                                 tflops=round(flop / t8 / 1e12, 1), speedup_vs_16bit=round(t / t8, 3),
                                 l2_fill_bytes_per_flop=round(fill8 / flop, 5), l2_fill_tb_s=round(fill8 / t8 / 1e12, 2)))
                print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
                del A8, W8, out16
        del a_big, x, h, out, cnt
    return rows


def l2_probe(torch, lib) -> list:
    rows_ = 128 * 1024  # 16 MB: resident in the 50 MB L2
    buf = torch.randn(rows_, 64, device="cuda").to(torch.float16)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    iters = 4000
    res = []
    for mode, cluster in ((0, 1), (2, 2)):
        ms = C.c_float(0.0)
        rc = lib.jimm_k_l2_probe(C.c_void_p(buf.data_ptr()), rows_, mode, cluster, iters, C.byref(ms),
                                 C.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == 0, lib.jimm_last_error().decode()
        grid = sms // cluster * cluster
        landed = grid * iters * 128 * 128
        res.append(dict(mode=mode, cluster=cluster, ms=round(ms.value, 3), smem_fill_tb_s=round(landed / (ms.value / 1e3) / 1e12, 2),
                        l2_read_tb_s=round(landed / cluster / (ms.value / 1e3) / 1e12, 2)))
    return res


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=HERE, help="repository tree whose built library is timed")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    root = os.path.abspath(args.root)
    sys.path.insert(0, root)
    import torch

    from jimm_b200 import _lib

    lib = _lib.load()
    res = dict(root=root, tile=list(tile_shape(root)), **device_line(torch))
    res["gemms"] = gemms(torch, lib, tile_shape(root), args.iters)
    res["l2_probe"] = l2_probe(torch, lib)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
