"""Every tensor-core GEMM of one conformer_large_joint_64x30s step (bench.py) at its real shape and epilogue, one at a time.

    python scripts/encoder_gemm_bench.py [--reps 5] [--dump DIR]

Each launch runs on a flushed L2 (256 MiB written before it) and is timed with CUDA events; the median over --reps launches is printed
with the algorithmic rate (2MNK per slice) as a share of the 3xTF32 ceiling (1/6 of the 989 TFLOP/s dense BF16 data-sheet peak) and
the minimum HBM traffic (A and B once, C written, R read) as a share of the 3.35 TB/s data-sheet bandwidth.  --dump DIR writes, for
the last launch of every shape, a .npy of row fingerprints of the output: per row of the last dimension an int64 sum of its 32-bit
words times odd weights, so any single changed bit changes its row's value (the full outputs are over 10 GB).  Inputs are seeded and
in-place residuals restored before every launch, so two builds can be compared bit for bit.
"""
import argparse
import math
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from espnet_b200 import ops  # noqa: E402

PEAK_TFLOPS = 989.0 / 6.0   # 3xTF32: three tf32 MMAs per product, tf32 at half the bf16 rate
PEAK_GBS = 3350.0

# conformer_large_joint_64x30s: 64 utterances of 30 s -> 3751 fbank frames -> T1 = 1875 x F1 = 39 -> T = 937 x F2 = 19 after Conv2dSubsampling
B, T, D, FF, H, V, L_DEC = 64, 937, 512, 2048, 8, 5000, 6
F2, T1H, F1H = 19, 938, 20
M = B * T


def gpu_identity():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        if out:
            return out
    except (OSError, subprocess.SubprocessError):
        pass
    return torch.cuda.get_device_name() + ", power limit unknown"


def fingerprint(out):
    rows = out.reshape(-1, out.shape[-1]).view(torch.int32)
    w = torch.arange(out.shape[-1], device=out.device, dtype=torch.long) * 2654435761 * 2 + 1
    step = max(1, (1 << 26) // out.shape[-1])
    return torch.cat([(rows[i:i + step].long() * w).sum(dim=1) for i in range(0, rows.shape[0], step)])


def rnd(*shape, scale=1.0):
    return torch.randn(*shape, device="cuda") * scale


def linear_case(name, N, K, *, act=ops.ACT_NONE, split_out=False, residual=False, alpha=1.0, count=1):
    """out[M, N] = epilogue(x[M, K] w[N, K]^T + b) as the encoder's linear() calls run it."""
    def make():
        x, w, b = rnd(2, M, K), rnd(2, N, K, scale=K ** -0.5), rnd(N)
        out = rnd(2, M, N) if split_out else rnd(M, N)
        keep = out.clone() if residual else None

        def reset():   # in-place residual: restore the input (outside the timed window)
            if keep is not None:
                out.copy_(keep)

        def run():
            ops.linear(x, w, out, bias=b, act=act, residual=out if residual else None, alpha=alpha, split_out=split_out)
        return reset, run, out
    c_bytes = (2 if split_out else 1) * M * N * 4
    return dict(name=name, make=make, flops=2.0 * M * N * K, bytes=2 * 4 * (M * K + N * K) + c_bytes + (M * N * 4 if residual else 0),
                count=count)


def conv2_case():
    """Conv2dSubsampling conv2 as implicit GEMM over the parity-split conv1 output (a_mode 1), split output."""
    C = D

    def make():
        c1, w, b = rnd(B, 8, F1H, T1H, C), rnd(2, C, 9 * C, scale=(9 * C) ** -0.5), rnd(C)
        c2 = torch.empty(2, B, F2, T, C, device="cuda")

        def run():
            ops.gemm(T, C, 9 * C, c1, 0, 0, w, C * 9 * C, 9 * C, c2, C, c_plane=B * F2 * T * C, split_out=True, bias=b, act=ops.ACT_RELU,
                     nbx=F2, nby=B, sc=(T * C, F2 * T * C), a_mode=1, conv=(T1H, F1H, C))
        return None, run, c2
    return dict(name="conv2 (a_mode 1)", make=make, flops=2.0 * T * C * 9 * C * F2 * B,
                bytes=4 * (B * 8 * F1H * T1H * C + 2 * C * 9 * C + 2 * B * F2 * T * C), count=1)


def embed_out_case():
    """embed.out: K = F2 * C split over f (kob), alpha sqrt(D), positional table as batch-broadcast residual."""
    C = D

    def make():
        c2, w, b, pe = rnd(2, B, F2, T, C), rnd(2, D, F2 * C, scale=(F2 * C) ** -0.5), rnd(D), rnd(T, D)
        x = torch.empty(M, D, device="cuda")

        def run():
            ops.gemm(T, D, F2 * C, c2, B * F2 * T * C, C, w, D * F2 * C, F2 * C, x, D, bias=b, alpha=math.sqrt(D), R=pe, ldr=D, nbx=1, nby=B,
                     sa=(T * C, F2 * T * C), sc=(0, T * D), kob=C // 32)
        return None, run, x
    return dict(name="embed.out (kob)", make=make, flops=2.0 * M * D * F2 * C, bytes=4 * (2 * M * F2 * C + 2 * D * F2 * C + M * D + T * D),
                count=1)


def kv_memory_case():
    """Decoder source-attention K or V projection of one layer: heads as batch-x (shared A), utterances as batch-y, dk = 64 columns."""
    dk = D // H

    def make():
        enc, w, b = rnd(2, M, D), rnd(2, D, D, scale=D ** -0.5), rnd(D)
        kv = torch.empty(B, H, T, dk, device="cuda")

        def run():
            ops.gemm(T, dk, D, enc, M * D, D, w, D * D, D, kv, dk, bias=b, nbx=H, nby=B, sa=(0, T * D), sb=(dk * D, 0), sc=(T * dk, H * T * dk),
                     sbias_x=dk)
        return None, run, kv
    return dict(name="decoder memory K|V", make=make, flops=2.0 * M * D * D, bytes=4 * (2 * M * D + 2 * D * D + M * D), count=2 * L_DEC)


CASES = [
    linear_case("ffn w1 (swish, split)", FF, D, act=ops.ACT_SWISH, split_out=True, count=24),
    linear_case("ffn w2 (residual, alpha 0.5)", D, FF, residual=True, alpha=0.5, count=24),
    linear_case("qkv (split)", 3 * D, D, split_out=True, count=12),
    linear_case("attention out (residual)", D, D, residual=True, count=12),
    linear_case("conv pw1", 2 * D, D, count=12),
    linear_case("conv pw2 (residual)", D, D, residual=True, count=12),
    conv2_case(),
    embed_out_case(),
    linear_case("ctc head", V, D, count=1),
    kv_memory_case(),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--dump", metavar="DIR", help="write every shape's output as .npy")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    print(f"[encoder_gemm_bench] {gpu_identity()}, gemm mode {ops.gemm_mode()}")
    if args.dump:
        os.makedirs(args.dump, exist_ok=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    total_ms = total_tf = 0.0
    for i, case in enumerate(CASES):
        torch.manual_seed(1000 + i)
        reset, run, out = case["make"]()
        run()   # first launch: module load, tensor-map setup
        times = []
        for _ in range(args.reps):
            if reset is not None:
                reset()
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run()
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        ms = float(np.median(times))
        tf = case["flops"] / (ms * 1e-3) / 1e12
        gbs = case["bytes"] / (ms * 1e-3) / 1e9
        total_ms += ms * case["count"]
        total_tf += case["flops"] * case["count"] / 1e12
        print(f"  {case['name']:<30} {ms:8.3f} ms  x{case['count']:<3} {tf:6.1f} TFLOP/s ({tf / PEAK_TFLOPS:5.1%} of 3xTF32 ceiling)  "
              f"min HBM {case['bytes'] / 1e9:6.2f} GB -> {gbs:6.0f} GB/s ({gbs / PEAK_GBS:5.1%} of 3.35 TB/s)")
        if args.dump:
            np.save(os.path.join(args.dump, f"{i:02d}.npy"), fingerprint(out).cpu().numpy())
        del reset, run, out
        torch.cuda.empty_cache()
    print(f"  per step (x counts): {total_ms:.1f} ms, {total_tf:.2f} TFLOP algorithmic -> {total_tf / (total_ms * 1e-3):.1f} TFLOP/s")


if __name__ == "__main__":
    main()
