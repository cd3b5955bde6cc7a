#!/usr/bin/env python
"""Per-shape timing of go1_gemm (impl 0/1) on the learner's GEMM shapes: TFLOP/s with CUDA events, L2 flushed between runs."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from go1_b200 import capi  # noqa: E402

SHAPES = [  # (M, N, K, note)
    (24576, 256, 2100, "adapt L1 fwd"), (24576, 512, 2100, "actor/critic L1 fwd"), (24576, 1280, 2100, "fused L1 fwd (3 nets)"),
    (24576, 256, 512, "L2 fwd"), (24576, 128, 256, "L3 fwd"), (24576, 12, 128, "actor out"), (24576, 512, 256, "dgrad L2"),
    (512, 2100, 24576, "wgrad L1 (actor)"), (256, 2100, 24576, "wgrad L1 (adapt)"), (1280, 2100, 24576, "fused wgrad L1"),
    (256, 512, 24576, "wgrad L2"), (128, 256, 24576, "wgrad L3"), (12, 128, 24576, "wgrad out"),
    (4096, 512, 2100, "rollout L1"), (4096, 1280, 2100, "rollout fused L1"), (4096, 256, 512, "rollout L2"),
]


def main():
    L = capi.lib()
    only = os.environ.get("GEMM_BENCH_ONLY")
    global SHAPES
    if only:
        SHAPES = [sh for sh in SHAPES if sh[3] in only.split(";")]
    impls = (1,) if os.environ.get("GEMM_BENCH_TC_ONLY") else (0, 1)
    flush = torch.empty(256 * 1024 * 1024 // 4, device="cuda")
    print(f"{'shape':>24s} {'note':>26s} {'impl0 us':>10s} {'TF/s':>7s} {'impl1 us':>10s} {'TF/s':>7s}")
    for M, N, K, note in SHAPES:
        # operand majors as the learner issues them: wgrad reads dz / activations as [K][M] / [K][N] (the first layers' read transposed
        # copies, K-major), dgrad reads W as [K][N]
        ta, tb = (1, 0) if ("wgrad" in note and "L1" not in note) else ((0, 0) if "dgrad" in note else (0, 1))
        if os.environ.get("GEMM_BENCH_KMAJOR"):
            ta, tb = 0, 1
        pad = lambda n: (n + 3) // 4 * 4
        A = torch.randn(K, pad(M), device="cuda") if ta else torch.randn(M, pad(K), device="cuda")
        B = torch.randn(N, pad(K), device="cuda") if tb else torch.randn(K, pad(N), device="cuda")
        Cm = torch.empty(M, N, device="cuda")
        res = []
        for impl in impls:
            ts = []
            for it in range(6):
                flush.fill_(it)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                capi.check(L.go1_gemm(ta, tb, M, N, K, capi.ptr(A), A.stride(0), capi.ptr(B), B.stride(0), capi.ptr(Cm), N, None, 0, 0, impl, capi.stream_ptr()), "gemm")
                e1.record(); torch.cuda.synchronize()
                if it >= 2:
                    ts.append(e0.elapsed_time(e1) * 1e3)
            us = sum(ts) / len(ts)
            res += [us, 2.0 * M * N * K / us / 1e6]
        res = ([0.0, 0.0] + res) if len(res) == 2 else res
        print(f"{str((M, N, K)):>24s} {note:>26s} {res[0]:10.1f} {res[1]:7.1f} {res[2]:10.1f} {res[3]:7.1f}")


if __name__ == "__main__":
    main()
