#!/usr/bin/env python
"""Throughput of the Branchformer encoder path (one JSON line on stdout).

    python scripts/branchformer_bench.py [--steps 3] [--warmup 1] [--batch 64] [--merge concat|learned_ave|fixed_ave]

Model: the LibriSpeech Branchformer recipe (egs2/librispeech/asr1/conf/tuning/train_asr_branchformer_hop_length160_e18_linear3072.yaml:
18 blocks, d 512, h 8, cgmlp 3072, kernel 31, concat merge; --merge picks another merge method at the same shape) + 6-layer Transformer
decoder (linear units 2048), V 5000, seeded random weights; 64 x 30-s synthetic waveforms; joint CTC/attention beam 10, ctc_weight 0.3,
maxlenratio -64, and the frontend of scripts/ebranchformer_bench.py (hop 128) -- the decode settings of bench.py's
conformer_large_joint_64x30s, so the utt/s figures of the three scripts compare directly.

Reported, in this order:
  parity      one utterance's encoder output against the CPU oracle (atol 1e-4); the script fails on a mismatch
  throughput  utterances/s, median of the timed steps (CUDA events, L2 flushed between steps), waveforms resident on the device
  encoder     encoder-only time per step and achieved TFLOP/s against the algorithmic operation count (flops_per_utt below)
  kernels     learned_ave pooling and branch-merge kernel time at B 64 x T 937 (CUDA events over repeated launches) and achieved TB/s
              against their algorithmic bytes
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
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")]

import refbuild  # noqa: E402
import refbuild_bf  # noqa: E402

CFG = dict(d_model=512, heads=8, ff=2048, enc_layers=18, dec_layers=6, vocab=5000, cgmlp=3072, cgmlp_kernel=31, merge=0, use_attn=1,
           use_cgmlp=1, encoder="branchformer")
SECONDS, BEAM, CTC_WEIGHT, MAXLENRATIO = 30, 10, 0.3, -64.0
HBM_TBS = 3.35   # H100 SXM data sheet


def flops_per_utt(T, Tf, cfg=CFG, n_mels=80):
    """Algorithmic multiply-add count x 2 of one utterance's encoder + CTC head (T encoder frames, Tf feature frames)."""
    D, U, V = cfg["d_model"], cfg["cgmlp"], cfg["vocab"]
    merge_k = 2 * D if cfg["merge"] == 0 else D          # merge_proj: Linear(2D, D) for concat, Linear(D, D) for the averages
    block = T * (4 * 2 * D * D + 2 * D * U + 2 * (U // 2) * D + 2 * merge_k * D) + 8 * T * T * D
    F2 = ((n_mels - 1) // 2 - 1) // 2
    conv2 = 2 * T * F2 * D * 9 * D
    embed_out = 2 * T * D * F2 * D
    ctc = 2 * T * D * V
    return cfg["enc_layers"] * block + conv2 + embed_out + ctc


def gpu_identity():
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                           timeout=30)
        out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception:
        pass
    return out


def time_ms(fn, reps, flush=None):
    """Median over `reps` of CUDA-event time of fn(); the L2 is flushed before each repetition when `flush` is given."""
    ts = []
    for _ in range(reps):
        if flush is not None:
            flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def kernel_numbers(B, T, flush):
    from espnet_b200.lib import call, ptr

    D = CFG["d_model"]
    M, nchunk = B * T, (T + 31) // 32
    g = torch.Generator(device="cuda").manual_seed(0)
    lens = torch.full((B,), T, dtype=torch.int32, device="cuda")
    cat = torch.randn(M, 2 * D, device="cuda", generator=g)
    pw, pb = torch.randn(2, D, device="cuda", generator=g), torch.randn(2, device="cuda", generator=g)
    ww, wb = torch.randn(2, D, device="cuda", generator=g) / D ** 0.5, torch.randn(2, device="cuda", generator=g)
    part, mw = torch.empty(B * 2 * nchunk * (D + 2), device="cuda"), torch.empty(B, 2, device="cuda")
    xb = torch.empty(2, M, D, device="cuda")
    pool = lambda: call("espb_branch_pool_f32", ptr(cat), ptr(cat[:, D:]), 2 * D, B, T, D, ptr(lens), ptr(pw), ptr(pb), ptr(ww), ptr(wb),  # noqa: E731
                        ptr(part), ptr(mw))
    merge = lambda: call("espb_branch_merge_f32", ptr(cat), ptr(cat[:, D:]), 2 * D, M, D, T, ptr(mw), 0.0, 0.0, ptr(xb), M * D)  # noqa: E731
    out = {}
    # pool: both branches read once, the partials written and read back; merge: both branches read, the split operand written
    for name, fn, nbytes in (("pool", pool, M * 2 * D * 4 + 2 * B * 2 * nchunk * (D + 2) * 4), ("merge", merge, M * 2 * D * 4 + 2 * M * D * 4)):
        for _ in range(3):
            fn()
        ms = time_ms(fn, 20, flush)
        out[name] = {"ms": round(ms, 4), "algorithmic_bytes": nbytes, "achieved_TBps": round(nbytes / ms / 1e9, 3),
                     "share_of_datasheet_hbm": round(nbytes / ms / 1e9 / HBM_TBS, 3)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--merge", choices=refbuild_bf.MERGES, default="concat")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "branchformer_bench.py measures on a CUDA device; there is no CPU fallback"
    CFG["merge"] = refbuild_bf.MERGES.index(args.merge)
    refbuild_bf.install()
    from gpu_util import random_weights, speech2text

    from oracle.branchformer import BranchformerSpeech2Text

    torch.cuda.set_device(0)
    card = gpu_identity()
    w = random_weights(CFG, seed=0)
    s2t = speech2text(CFG, w, beam_size=BEAM, ctc_weight=CTC_WEIGHT, maxlenratio=MAXLENRATIO, nbest=1)
    nsamp = SECONDS * 16000
    waves = torch.stack([refbuild.waveform(i, nsamp) for i in range(args.batch)])
    speech = waves.cuda()
    lens = torch.full((args.batch,), nsamp, dtype=torch.long)

    # ---- parity first: utterance 0 alone against the CPU oracle
    enc0, _ = s2t.asr_model.encode(speech[:1], lens[:1])
    torch.set_num_threads(min(16, torch.get_num_threads()))
    ref0 = BranchformerSpeech2Text(CFG, w).encode(waves[0])
    err = (enc0[0].double().cpu() - ref0.double()).abs().max().item()
    if not (enc0.shape[1] == ref0.shape[0] and err < 1e-4):
        print(json.dumps({"parity": "FAILED", "encoder_max_abs_err": err}))
        sys.exit(1)

    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")   # > 50 MB L2

    def step():
        enc, enc_lens = s2t.asr_model.encode(speech, lens)
        return s2t.beam_search.forward_batch(enc, enc_lens, s2t.asr_model.enc_split(enc), MAXLENRATIO, 0.0)

    def encode():
        s2t.asr_model.encode(speech, lens)

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    step_ms = time_ms(step, args.steps, flush)
    enc_ms = time_ms(encode, args.steps, flush)
    T = enc0.shape[1]
    Tf = 1 + nsamp // 128
    fl = flops_per_utt(T, Tf)
    line = {
        "metric": f"utterances/sec, Branchformer (LibriSpeech recipe, {args.merge} merge) + 6L decoder, joint CTC/attention beam 10, "
                  f"{args.batch} x 30 s",
        "value": round(args.batch / (step_ms / 1e3), 2), "unit": "utt/s", "step_ms_median": round(step_ms, 2), "steps": args.steps,
        "warmup": args.warmup, "batch": args.batch, "encoder_frames": T, "parity_encoder_max_abs_err": err,
        "encoder_ms_median": round(enc_ms, 2), "encoder_share_of_step": round(enc_ms / step_ms, 3),
        "encoder_gflop_per_utt_algorithmic": round(fl / 1e9, 1), "encoder_achieved_TFLOPs": round(fl * args.batch / (enc_ms / 1e3) / 1e12, 1),
        "kernels_B64xT937": kernel_numbers(64, T, flush), "card": card, "l2": "flushed before every timed repetition",
    }
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
