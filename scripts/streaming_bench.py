#!/usr/bin/env python
"""Streaming decoding with the contextual-block Transformer encoder on the H100 (one JSON line on stdout).

    python scripts/streaming_bench.py [--streams 128] [--pushes 64] [--reps 3] [--utt-seconds 10]

Two recipe shapes of ``encoder: contextual_block_transformer`` (block 40, hop 16, look-ahead 16), random weights (seed 0), V 5000:
  aishell    egs2/aishell/asr1/conf/train_asr_streaming_transformer.yaml: 12 blocks, d 256, h 4, ff 2048, conv2d
  laborotv   egs2/laborotv/asr1 streaming Transformer: 18 blocks, d 512, h 8, ff 2048, conv2d6

Reported per shape:
  greedy  audio seconds per second of --streams lock-step streams, each pushing 40 ms (640 samples at 16 kHz) per call, CTC greedy
          (Speech2TextStreaming(greedy=True)): --reps timed windows of --pushes pushes each after --warmup pushes, CUDA events around each
          window, median / min / max.  The host -> device copy of each chunk and the device -> host copy of the new tokens are inside the
          window, as in a server.
  beam    per-push latency of one stream in beam-search mode with the AISHELL recipe's decode settings (beam 10, ctc_weight 0.6, lm_weight 0.3,
          disable_repetition_detection; 6-layer Transformer decoder, 2 x 650 LSTM LM, conf/train_lm.yaml): one --utt-seconds utterance pushed
          40 ms at a time, after one warm-up utterance; each push timed with CUDA events and a synchronise; median / p90 / max over the
          non-final pushes, and the final push alone.
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

SHAPES = {"aishell": dict(d_model=256, heads=4, ff=2048, layers=12, input_layer="conv2d"),
          "laborotv": dict(d_model=512, heads=8, ff=2048, layers=18, input_layer="conv2d6")}
PUSH = 640          # 40 ms at 16 kHz
VOCAB = 5000


def gpu_identity():
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                           timeout=30)
        out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception:
        pass
    return out


def build(shape, dec_layers):
    import espnet_b200

    s = SHAPES[shape]
    y = refbuild.model_yaml(dict(d_model=s["d_model"], heads=s["heads"], ff=s["ff"], enc_layers=s["layers"], dec_layers=max(dec_layers, 1),
                                 vocab=VOCAB))
    y.update(encoder="contextual_block_transformer", normalize=None, normalize_conf={},
             encoder_conf=dict(output_size=s["d_model"], attention_heads=s["heads"], linear_units=s["ff"], num_blocks=s["layers"],
                               input_layer=s["input_layer"], block_size=40, hop_size=16, look_ahead=16))
    if dec_layers == 0:
        y["decoder"] = None
    torch.manual_seed(0)
    return espnet_b200.build_model(argparse.Namespace(**y)).cuda().eval()


def greedy(shape, args):
    import espnet_b200

    model = build(shape, 0)
    s2t = espnet_b200.Speech2TextStreaming(model, n_streams=args.streams, device="cuda", greedy=True)
    host = (0.1 * torch.randn(args.streams, PUSH * (args.warmup + args.pushes * args.reps), generator=torch.Generator().manual_seed(1))).pin_memory()
    p = 0
    for _ in range(args.warmup):
        s2t(host[:, p * PUSH:(p + 1) * PUSH], is_final=False)
        p += 1
    rates = []
    for _ in range(args.reps):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.pushes):
            s2t(host[:, p * PUSH:(p + 1) * PUSH], is_final=False)
            p += 1
        e1.record()
        e1.synchronize()
        rates.append(args.streams * args.pushes * PUSH / 16000.0 / (e0.elapsed_time(e1) / 1000.0))
    return {"streams": args.streams, "pushes_per_window": args.pushes, "windows": args.reps, "audio_s_per_s_median": statistics.median(rates),
            "audio_s_per_s_min": min(rates), "audio_s_per_s_max": max(rates),
            "ms_per_push_median": args.streams * PUSH / 16000.0 / statistics.median(rates) * 1000.0}


def beam(shape, args):
    import espnet_b200

    model = build(shape, 6)
    torch.manual_seed(0)
    lm = espnet_b200.SequentialRNNLM(VOCAB, unit=650, nlayers=2, rnn_type="lstm")
    s2t = espnet_b200.Speech2TextStreaming(model, n_streams=1, device="cuda", beam_size=10, ctc_weight=0.6, lm_weight=0.3,
                                           disable_repetition_detection=True, lm=lm)
    n = args.utt_seconds * 16000 // PUSH * PUSH
    wave = refbuild.waveform(3, n)

    def utterance(timed):
        ms = []
        for p in range(0, n, PUSH):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            res = s2t(wave[p:p + PUSH], is_final=(p + PUSH >= n))
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        return ms, res

    utterance(False)
    ms, res = utterance(True)
    body = sorted(ms[:-1])
    return {"pushes": len(ms), "ms_per_push_median": statistics.median(body), "ms_per_push_p90": body[int(0.9 * (len(body) - 1))],
            "ms_per_push_max": body[-1], "ms_final_push": ms[-1], "final_tokens": len(res[0][2]) if res else 0}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--streams", type=int, default=128)
    ap.add_argument("--pushes", type=int, default=64, help="pushes per timed window")
    ap.add_argument("--reps", type=int, default=3, help="timed windows")
    ap.add_argument("--warmup", type=int, default=32, help="untimed pushes first")
    ap.add_argument("--utt-seconds", type=int, default=10, help="length of the beam-mode utterance")
    ap.add_argument("--shapes", default="aishell,laborotv")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("streaming_bench.py measures on a CUDA device; none found")
    out = {"gpu": gpu_identity(), "push_ms": 1000.0 * PUSH / 16000, "vocab": VOCAB}
    for shape in args.shapes.split(","):
        out[shape] = dict(SHAPES[shape], greedy=greedy(shape, args), beam=beam(shape, args))
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
