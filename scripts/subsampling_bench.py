#!/usr/bin/env python
"""The conv2d / conv2d2 / conv2d6 / conv2d8 input layers on the H100 (one JSON line on stdout).

    python scripts/subsampling_bench.py [--steps 3] [--warmup 1] [--batch 64]

Reported, in this order:
  parity      each input layer's subsampling output (Conformer-large weights, d 512) for two 5-s utterances, and the ReazonSpeech Conformer's
              encoder output for one 30-s utterance, against the CPU oracle (atol 1e-4); the script fails on a mismatch
  stacks      per input layer, the subsampling stack (conv1, the implicit-GEMM convs, the conv2d8 re-layout, embed.out) at B 64 x 30 s
              (T_f 3751, 80 mels), d 512: median time (CUDA events, L2 flushed), the algorithmic GFLOP from shapes (flops below) and the
              achieved TFLOP/s, plus the time of each launch of one extra run
  relayout    the conv2d8 re-layout kernel's time against the encoder time of a conv2d8 Conformer-large (12 blocks, d 512) on the same batch
  throughput  utterances/s of the ReazonSpeech Conformer (egs2/reazonspeech/asr1/conf/train_asr_conformer.yaml: 12 blocks, d 512, h 8,
              conv2d6) + 6-layer decoder, V 5000, joint CTC/attention beam 10 (ctc_weight 0.3, maxlenratio -64: bench.py's
              conformer_large_joint_64x30s decode settings) on 64 x 30 s, next to the same model with conv2d; waveforms resident on the device
plus the card's name and power limit, read in the same run.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")]

import refbuild  # noqa: E402
import refbuild_subsampling  # noqa: E402

LARGE = dict(d_model=512, heads=8, ff=2048, enc_layers=12, dec_layers=6, vocab=5000, kernel=31)
LAYERS = ("conv2d", "conv2d2", "conv2d6", "conv2d8")
SECONDS, BEAM, CTC_WEIGHT, MAXLENRATIO = 30, 10, 0.3, -64.0


def flops(input_layer, B, Tf, n_mels=80, C=512):
    """Algorithmic multiply-add count x 2 of the subsampling stack: conv1 (9 taps, 1 input channel), each k x k conv over C channels,
    embed.out over F_last * C inputs."""
    from espnet_b200.layers import SUBSAMPLING, subsampled_len

    Ts, Fs = subsampled_len(Tf, input_layer), subsampled_len(n_mels, input_layer)
    total = 2 * B * Ts[0] * Fs[0] * C * 9
    for i, (k, _) in enumerate(SUBSAMPLING[input_layer]):
        total += 2 * B * Ts[i + 1] * Fs[i + 1] * C * k * k * C
    return total + 2 * B * Ts[-1] * C * Fs[-1] * C


def gpu_identity():
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                           timeout=30)
        out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception:
        pass
    return out


def time_ms(fn, reps, flush):
    """Median over `reps` of CUDA-event time of fn(), the L2 flushed before each repetition."""
    ts = []
    for _ in range(reps):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def cfg_of(input_layer):
    return dict(LARGE, input_layer=input_layer)


def encoder_of(w, input_layer):
    import espnet_b200

    enc = espnet_b200.ConformerEncoder(80, output_size=512, attention_heads=8, linear_units=2048, num_blocks=12, input_layer=input_layer,
                                       macaron_style=True, rel_pos_type="latest", pos_enc_layer_type="rel_pos",
                                       selfattention_layer_type="rel_selfattn", use_cnn_module=True, cnn_module_kernel=31)
    enc.load_state_dict({k[len("encoder."):]: v for k, v in w.items() if k.startswith("encoder.")}, strict=True)
    return enc.cuda().eval()


def subsample(enc, xs):
    """The encoder's subsampling stack alone -> (B, T, D)."""
    B, Tf, _ = xs.shape
    from espnet_b200.layers import subsampled_len

    T = subsampled_len(Tf, enc.input_layer)[-1]
    x = enc._buf("x", (B * T, 512))
    enc._subsample(xs, x, math.sqrt(512))
    return x.view(B, T, 512)


def launches(fn):
    """(name [GEMM shape tag], ms) of every launch of one run of fn()."""
    from espnet_b200 import lib

    lib.profile = []
    fn()
    torch.cuda.synchronize()
    out = [(n + (f" [{t}]" if t else ""), round(a.elapsed_time(b), 3)) for n, t, a, b in lib.profile]
    lib.profile = None
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--batch", type=int, default=64)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "subsampling_bench.py measures on a CUDA device; there is no CPU fallback"
    from gpu_util import random_weights, speech2text

    from oracle import frontend as Fr
    from oracle.subsampling import SubsamplingSpeech2Text, conv2d_subsampling

    refbuild_subsampling.install()   # model yaml with cfg["input_layer"]

    torch.cuda.set_device(0)
    torch.set_num_threads(min(16, torch.get_num_threads()))
    line = {"metric": "input-layer subsampling stacks and ReazonSpeech-shape (conv2d6) Conformer throughput, 64 x 30 s", "card": gpu_identity()}
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")   # > 50 MB L2
    nsamp = SECONDS * 16000
    Tf = 1 + nsamp // 128
    B = args.batch
    g = torch.Generator().manual_seed(0)
    xs = torch.randn(B, Tf, 80, generator=g).cuda()
    short = [Fr.utterance_mvn(Fr.log_mel(Fr.stft_power(refbuild.waveform(100 + i, 80000)), Fr.slaney_mel_matrix())) for i in range(2)]

    # ---- subsampling stacks, with parity of each against the oracle
    line["parity"], line["stacks"] = {}, {}
    for il in LAYERS:
        w = random_weights(cfg_of(il), seed=0)
        enc = encoder_of(w, il)
        enc._pack()
        errs = []
        for f in short:
            got = subsample(enc, f[None].cuda())[0].cpu()
            ref = conv2d_subsampling(f, w, il)
            assert got.shape == ref.shape
            errs.append((got.double() - ref.double()).abs().max().item())
        line["parity"][f"{il}_subsampling_max_abs_err"] = max(errs)
        if max(errs) >= 1e-4:
            line["parity"]["result"] = "FAILED"
            print(json.dumps(line))
            sys.exit(1)
        for _ in range(args.warmup):
            subsample(enc, xs)
        ms = time_ms(lambda: subsample(enc, xs), max(3, args.steps), flush)
        fl = flops(il, B, Tf)
        line["stacks"][il] = {"ms_median": round(ms, 2), "gflop_algorithmic": round(fl / 1e9, 1), "achieved_TFLOPs": round(fl / ms / 1e9, 1),
                              "launches_ms": launches(lambda: subsample(enc, xs))}
        if il == "conv2d8":
            relayout = sum(ms_ for n, ms_ in line["stacks"][il]["launches_ms"] if n.startswith("espb_phase_split_f32"))
            for _ in range(args.warmup):
                enc(xs, torch.full((B,), Tf))
            enc_ms = time_ms(lambda: enc(xs, torch.full((B,), Tf)), args.steps, flush)
            line["relayout"] = {"phase_split_ms": round(relayout, 3), "conv2d8_conformer_large_encoder_ms": round(enc_ms, 2),
                                "share_of_encoder": round(relayout / enc_ms, 4)}
        del enc, w
        torch.cuda.empty_cache()
    del xs
    torch.cuda.empty_cache()

    # ---- end-to-end throughput: ReazonSpeech (conv2d6) next to conv2d
    waves = torch.stack([refbuild.waveform(i, nsamp) for i in range(B)])
    speech, lens = waves.cuda(), torch.full((B,), nsamp, dtype=torch.long)
    line["throughput_utt_per_s"] = {}
    for il in ("conv2d6", "conv2d"):
        cfg = cfg_of(il)
        w = random_weights(cfg, seed=0)
        s2t = speech2text(cfg, w, beam_size=BEAM, ctc_weight=CTC_WEIGHT, maxlenratio=MAXLENRATIO, nbest=1)
        if il == "conv2d6":
            enc0, _ = s2t.asr_model.encode(speech[:1], lens[:1])
            ref0 = SubsamplingSpeech2Text(cfg, w).encode(waves[0])
            err = (enc0[0].double().cpu() - ref0.double()).abs().max().item()
            line["parity"]["reazonspeech_encoder_max_abs_err"] = err
            if not (enc0.shape[1] == ref0.shape[0] and err < 1e-4):
                line["parity"]["result"] = "FAILED"
                print(json.dumps(line))
                sys.exit(1)

        def step():
            enc, enc_lens = s2t.asr_model.encode(speech, lens)
            return s2t.beam_search.forward_batch(enc, enc_lens, s2t.asr_model.enc_split(enc), MAXLENRATIO, 0.0)

        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        step_ms = time_ms(step, args.steps, flush)
        line["throughput_utt_per_s"][il] = {"value": round(B / (step_ms / 1e3), 2), "step_ms_median": round(step_ms, 2)}
        del s2t, w
        torch.cuda.empty_cache()
    line["parity"]["result"] = "ok"
    line.update(steps=args.steps, warmup=args.warmup, batch=B, l2="flushed before every timed repetition")
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
