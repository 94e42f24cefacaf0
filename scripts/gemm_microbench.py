"""In-graph latency of the decode-step GEMM shapes (CUDA-graph replay of 100 back-to-back launches, CUDA events).

    python scripts/gemm_microbench.py                        # default GEMM mode (tc2)
    ESPNET_B200_GEMM=tc python scripts/gemm_microbench.py    # without chunked promotion
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from espnet_b200 import ops  # noqa: E402

SHAPES = [(640, 512, 32), (640, 512, 512), (640, 512, 2048), (640, 1536, 512), (640, 2048, 512), (640, 5000, 512), (320, 512, 512), (1280, 512, 512)]
REPS = 100
tag = "mode=" + ops.gemm_mode()
for M, N, K in SHAPES:
    a, b = ops.split_from(torch.randn(M, K, device="cuda")), ops.split_from(torch.randn(N, K, device="cuda") / K ** 0.5)
    bias = torch.randn(N, device="cuda")
    out = torch.zeros(M, N, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for _ in range(3):
            ops.linear(a, b, out, bias=bias)
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(REPS):
                ops.linear(a, b, out, bias=bias)
        for _ in range(3):
            g.replay()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        for _ in range(5):
            g.replay()
        e1.record(s)
        s.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / (5 * REPS)
    print(f"[gemm_microbench {tag}] M{M} N{N} K{K}: {us:7.2f} us/launch  ({6.0 * M * N * K / us / 1e6:7.1f} TFLOP/s 3xTF32-issued)")
