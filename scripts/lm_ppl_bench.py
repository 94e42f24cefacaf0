#!/usr/bin/env python
"""Throughput of LM perplexity (ESPnetLanguageModel.nll, what lm_calc_perplexity runs per batch) on the CUDA path (one JSON line on stdout).

    python scripts/lm_ppl_bench.py [--batch 64] [--steps 10] [--warmup 3]

Models, seeded random weights, V 5000:
  transformer  LibriSpeech's train_lm_transformer2.yaml: 16 layers, att_unit 512, 8 heads (d_k 64), unit 2048, embed_unit 128, pos_enc null
  lstm         2 x 650 LSTM (the recipes' train_lm.yaml shape)
Batch: --batch sentences of seeded random lengths 10..100 tokens (LibriSpeech test sets average about 35 BPE tokens a sentence).

Reported:
  tokens_per_s   scored tokens (sum of text_lengths + 1) / the median time of one nll call (CUDA events around work that ends in a sync)
  attention      per layer at the LM's shape (B = --batch, T = the padded length + 1, and T = 512), median kernel time of
                 espb_causal_flash_attn_f32 against the non-causal espb_flash_attn_f32 on the same inputs
  nll_kernel     espb_nll_rows_f32 over the LM's logits [B*T][5000]: median time and achieved TB/s (logit bytes + targets + output)
plus the card's name and power limit, read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

V = 5000


def gpu_identity():
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                           timeout=30)
        out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception:
        pass
    return out


def timed(fn, steps, warmup):
    """Median milliseconds of fn() over steps calls, after warmup calls."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return statistics.median(ts)


def build(kind):
    import espnet_b200

    torch.manual_seed(1)
    if kind == "transformer":
        lm = espnet_b200.TransformerLM(V, pos_enc=None, embed_unit=128, att_unit=512, head=8, unit=2048, layer=16)
    else:
        lm = espnet_b200.SequentialRNNLM(V, unit=650, nlayers=2)
    return espnet_b200.ESPnetLanguageModel(lm.cuda().eval(), V).eval()


def attention(B, T, steps, warmup):
    """Causal vs non-causal fused attention on one layer's q|k|v at B x T, 8 heads of 64."""
    from espnet_b200 import ops

    H, dk = 8, 64
    D, M, Tp = H * dk, B * T, (T + 31) // 32 * 32
    g = torch.Generator().manual_seed(0)
    qkv = ops.split_from(torch.randn(M, 3 * D, generator=g).cuda())
    tok = torch.randint(1, V, (B, T), generator=g, dtype=torch.int32).cuda()
    lens = torch.full((B,), T, dtype=torch.int32, device="cuda")
    vt = torch.empty(2, B, H, dk, Tp, device="cuda")
    ctx = torch.empty(2, M, D, device="cuda")
    ops.call("espb_v_transpose_f32", ops.ptr(qkv), M * 3 * D, B, T, D, H, ops.ptr(lens), ops.ptr(vt), B * H * dk * Tp, Tp)
    full = lambda: ops.flash_attn(qkv, 0, 3 * D, qkv, D, 3 * D, vt, Tp, None, 0, lens, B, H, T, dk, ctx)  # noqa: E731
    causal = lambda: ops.call("espb_causal_flash_attn_f32", ops.ptr(qkv), 0, M * 3 * D, 3 * D, ops.ptr(qkv), D, M * 3 * D, 3 * D,  # noqa: E731
                              ops.ptr(vt), B * H * dk * Tp, Tp, ops.ptr(tok), ops.ptr(lens), B, H, T, dk, ops.ptr(ctx), M * D, D)
    t_full, t_causal = timed(full, 5 * steps, warmup), timed(causal, 5 * steps, warmup)
    return dict(B=B, T=T, noncausal_ms=round(t_full, 4), causal_ms=round(t_causal, 4), causal_over_noncausal=round(t_causal / t_full, 3))


def nll_kernel(rows, steps, warmup):
    from espnet_b200 import ops

    g = torch.Generator().manual_seed(0)
    x = (torch.randn(rows, V, generator=g) * 4).cuda()
    tgt = torch.randint(0, V, (rows,), generator=g, dtype=torch.int32).cuda()
    out = torch.empty(rows, device="cuda")
    ms = timed(lambda: ops.call("espb_nll_rows_f32", ops.ptr(x), rows, V, V, ops.ptr(tgt), ops.ptr(out)), 10 * steps, warmup)
    nbytes = rows * V * 4 + rows * 8
    return dict(rows=rows, V=V, ms=round(ms, 4), tb_per_s=round(nbytes / ms / 1e9, 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "lm_ppl_bench measures the GPU: no CUDA device found"
    g = torch.Generator().manual_seed(0)
    lengths = torch.randint(10, 101, (args.batch,), generator=g)
    text = torch.randint(1, V - 1, (args.batch, int(lengths.max())), generator=g)
    ntok = int((lengths + 1).sum())
    res = dict(gpu=gpu_identity(), batch=args.batch, max_len=int(lengths.max()), scored_tokens=ntok)
    for kind in ("transformer", "lstm"):
        model = build(kind)
        nll, _ = model.nll(text, lengths)
        assert torch.isfinite(nll).all()
        ms = timed(lambda: model.nll(text, lengths), args.steps, args.warmup)
        res[kind] = dict(nll_ms=round(ms, 3), tokens_per_s=round(ntok / ms * 1e3, 1))
        del model
        torch.cuda.empty_cache()
    res["attention"] = [attention(args.batch, int(lengths.max()) + 1, args.steps, args.warmup), attention(args.batch, 512, args.steps, args.warmup)]
    res["nll_kernel"] = nll_kernel(args.batch * (int(lengths.max()) + 1), args.steps, args.warmup)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
