"""Stand-alone timing of single hot kernels on bench-shaped synthetic data (CUDA events, L2 flushed between launches).

    python scripts/kernel_microbench.py softmax|srcattn|selfattn|all [reps]
"""
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from espnet_b200.lib import call, ptr  # noqa: E402

which = sys.argv[1] if len(sys.argv) > 1 else "all"
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
dev = "cuda"
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def timeit(name, fn, bytes_alg):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        flush.fill_(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    us = ts[len(ts) // 2]
    print(f"[kernel_microbench] {name}: median {us:9.1f} us  min {ts[0]:9.1f} us   algorithmic {bytes_alg / 1e6:8.1f} MB -> {bytes_alg / us / 1e6:6.2f} TB/s")


if which in ("softmax", "all"):
    B, H, T = 64, 8, 937
    Tp, Rp = 960, 1888
    ac = torch.randn(B * H * T, Tp, device=dev)
    bd = torch.randn(B * H * T, Rp, device=dev)
    probs = torch.empty(2, B * H * T, Tp, device=dev)
    lens = torch.full((B,), T, dtype=torch.int32, device=dev)
    alg = B * H * T * (2 * T + 2 * Tp) * 4
    timeit("relpos_softmax B64 H8 T937", lambda: call("espb_relpos_softmax_f32", ptr(ac), ptr(bd), B, H, T, Tp, Rp, ptr(lens), math.sqrt(64.0), ptr(probs),
                                                      B * H * T * Tp), alg)
    del ac, bd, probs

if which in ("srcattn", "all"):
    U, H, T, W, D = 64, 8, 937, 10, 512
    n = U * W
    q = torch.randn(n, D, device=dev)
    kv = torch.randn(2, U, H, T, 64, device=dev)
    ctx = torch.empty(2, n, D, device=dev)
    lens = torch.full((U,), T, dtype=torch.int32, device=dev)
    alg = 2 * U * H * T * 64 * 4
    timeit("dec_src_attn U64 H8 T937 W10", lambda: call("espb_dec_src_attn_f32", ptr(q), ptr(kv[0]), ptr(kv[1]), U, T, ptr(lens), W, D, H, ptr(ctx), n * D), alg)

if which in ("frontend", "all"):
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import espnet_b200

    B, L = 64, 480000
    fe = espnet_b200.DefaultFrontend().cuda()
    wave = 0.1 * torch.randn(B, L, device=dev)
    lens = torch.full((B,), L, dtype=torch.long)
    alg = B * (4 * L + 320 * (1 + L // 128))
    timeit("stft_logmel 64 x 30 s (algorithmic bytes: waveform read + log-mel write)", lambda: fe(wave, lens), alg)

if which in ("selfattn", "all"):
    U, W, H, D, L = 64, 10, 8, 512, 64
    n = U * W
    pos = 40
    qkv = torch.randn(n, 3 * D, device=dev)
    kc, vc = torch.randn(L, n, D, device=dev), torch.randn(L, n, D, device=dev)
    # ancestors stay inside the utterance's beam; older positions collapse onto few slots like a real beam
    g = torch.Generator(device="cpu").manual_seed(0)
    anc = torch.zeros(n, L, dtype=torch.int32)
    for j in range(L):
        spread = 1 + min(W - 1, max(0, j - (pos - 12)))
        anc[:, j] = (torch.arange(n) // W) * W + torch.randint(0, spread, (n,), generator=g)
    anc = anc.to(dev)
    ctx = torch.empty(2, n, D, device=dev)
    alg = n * 3 * D * 4 + 2 * n * D * 4 * 2
    timeit(f"dec_self_attn n{n} H8 pos{pos}", lambda: call("espb_dec_self_attn_f32", ptr(qkv), ptr(kc), ptr(vc), ptr(anc), L, n, D, H, pos, None, L, ptr(ctx), n * D), alg)

if which in ("ln", "all"):
    rows, D = 640, 512
    x = torch.randn(rows, D, device=dev)
    g, b = torch.randn(D, device=dev), torch.randn(D, device=dev)
    out = torch.empty(2, rows, D, device=dev)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        fn = lambda: call("espb_layernorm_f32", ptr(x), rows, D, ptr(g), ptr(b), 1e-12, None, ptr(out), rows * D)  # noqa: E731
        fn()
        s.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=s):
            for _ in range(100):
                fn()
        gr.replay()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        for _ in range(5):
            gr.replay()
        e1.record(s)
        s.synchronize()
    print(f"[kernel_microbench] layernorm {rows}x{D} in-graph back-to-back: {e0.elapsed_time(e1) * 1e3 / 500:6.2f} us/launch")

if which in ("ffn", "all"):
    from espnet_b200 import ops

    M, N, K = 59968, 2048, 512      # encoder feed-forward w_1 of the 64 x 30 s workload (Swish, hi/lo split output)
    a, b = ops.split_from(torch.randn(M, K, device=dev)), ops.split_from(torch.randn(N, K, device=dev) / K ** 0.5)
    bias = torch.randn(N, device=dev)
    out = torch.empty(2, M, N, device=dev)
    alg_bytes = (2 * M * K + 2 * N * K + 2 * M * N) * 4
    timeit(f"gemm_tf32x3 M{M} N{N} K{K} swish split ({2.0 * M * N * K / 1e12:.3f} TFLOP algorithmic)",
           lambda: ops.linear(a, b, out, bias=bias, act=ops.ACT_SWISH, split_out=True), alg_bytes)

if which in ("ac", "all"):
    from espnet_b200 import ops

    # q_u . k^T of the rel-pos attention (encoder.py): per (utterance, head) a T x T x 64 product, operands are head slices of [M][D] / [M][3D]
    B, H, T, D = 64, 8, 937, 512
    dk, Tp, M = D // H, 960, 64 * 937
    qu = ops.split_from(torch.randn(M, D, device=dev))
    qkv = ops.split_from(torch.randn(M, 3 * D, device=dev))
    ac = torch.empty(B * H * T, Tp, device=dev)
    alg = (2 * M * D * 2 + B * H * T * T) * 4        # hi/lo q and k read once, scores written once
    timeit(f"q_u.k^T GEMM T{T} x T{T} x {dk}, {B * H} problems ({2.0 * B * H * T * T * dk / 1e12:.3f} TFLOP algorithmic)",
           lambda: ops.gemm(T, T, dk, qu, M * D, D, qkv, M * 3 * D, 3 * D, ac, Tp, nbx=H, nby=B, sa=(dk, T * D), sb=(dk, T * 3 * D),
                            sc=(T * Tp, H * T * Tp), b_off=D), alg)

if which in ("logsoftmax", "all"):
    # decode-step shape (640 hypotheses x V 5000) and the encoder-side CTC posteriors (64 x 937 frames); ESPB_LOGSOFTMAX_3PASS=1 = the first kernel
    for rows in (640, 64 * 937):
        x = torch.randn(rows, 5000, device=dev)
        timeit(f"log_softmax_rows {rows} x 5000", lambda: call("espb_log_softmax_rows_f32", ptr(x), rows, 5000, 5000), 2 * rows * 5000 * 4)
        del x
