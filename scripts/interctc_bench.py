#!/usr/bin/env python
"""Cost of self-conditioned intermediate CTC on the CUDA path at the LibriSpeech-100 recipe shape
(egs2/librispeech_100/asr1/conf/tuning/train_conformer_scctc.yaml: Conformer 18 blocks, d 256, h 4, ff 1024, kernel 31, conv2d,
interctc_layer_idx [6, 12] with conditioning, no decoder, ctc_weight 1.0), random weights, V 5000, --utts utterances of --seconds s.

Reports, as one JSON line:
  * the encoder's time with and without the conditioning on the same weights (interctc_layer_idx emptied for the second run);
  * per conditioned layer, the time of the CTC logits GEMM, of espb_softmax_rows_split_f32 and of the conditioning GEMM (CUDA events over
    --reps launches at the encoder's own shape), and the softmax kernel's achieved bytes/s (V floats read and 2 x ldo floats written per
    row) against the H100 SXM data-sheet 3.35 TB/s;
  * utterances/s of Speech2Text.ctc_greedy and of the CTC-only beam search (Speech2Text.batch_decode, beam --beam);
  * peak device memory, and the card's name and power limit read in the same run.

    python scripts/interctc_bench.py [--utts 64] [--seconds 30] [--beam 10] [--maxlenratio -64]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def config(V):
    return dict(token_list=["<blank>", "<unk>"] + [f"t{i}" for i in range(V - 3)] + ["<sos/eos>"], frontend="default",
                frontend_conf=dict(n_fft=512, hop_length=160, n_mels=80), specaug=None, normalize="utterance_mvn", normalize_conf={},
                encoder="conformer",
                encoder_conf=dict(output_size=256, attention_heads=4, linear_units=1024, num_blocks=18, input_layer="conv2d", normalize_before=True,
                                  macaron_style=True, rel_pos_type="latest", pos_enc_layer_type="rel_pos", selfattention_layer_type="rel_selfattn",
                                  activation_type="swish", use_cnn_module=True, cnn_module_kernel=31, interctc_layer_idx=[6, 12],
                                  interctc_use_conditioning=True),
                model_conf=dict(ctc_weight=1.0, interctc_weight=0.66, lsm_weight=0.1, length_normalized_loss=False))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, pl = out.stdout.strip().splitlines()[0].split(", ")
        return dict(name=name, power_limit=pl)
    except Exception as e:   # the card's name from torch at least
        return dict(name=torch.cuda.get_device_name(0), power_limit=f"unknown ({e})")


def timed(fn, reps):
    """Mean ms of fn() over reps launches (CUDA events), after one warm-up call."""
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--utts", type=int, default=64)
    p.add_argument("--seconds", type=float, default=30.0)
    p.add_argument("--beam", type=int, default=10)
    p.add_argument("--vocab", type=int, default=5000)
    p.add_argument("--maxlenratio", type=float, default=-64.0)
    p.add_argument("--reps", type=int, default=10)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("interctc_bench.py measures on a CUDA device; none is available")
    import espnet_b200
    from espnet_b200 import Speech2Text, ops
    from espnet_b200.asr_inference import build_model
    from espnet_b200.layers import _pitch

    torch.manual_seed(0)
    model = build_model(argparse.Namespace(**config(a.vocab))).cuda().eval()
    enc, ctc = model.encoder, model.ctc
    g = torch.Generator().manual_seed(1)
    n_samp = int(a.seconds * 16000)
    waves = [0.1 * torch.randn(n_samp, generator=g) for _ in range(a.utts)]
    greedy = Speech2Text(asr_model=model, asr_train_args=None, device="cuda", ctc_weight=1.0, nbest=1)
    speech, lens = greedy._to_batch(waves)
    with torch.no_grad():
        feats, flens = model.frontend(speech, lens)
        feats, flens = model.normalize(feats, flens)

    # encoder with and without the conditioning, same weights
    def encode():
        with torch.no_grad():
            return enc(feats, flens, ctc=ctc)

    enc_ms = timed(encode, a.reps)
    idx = enc.interctc_layer_idx
    enc.interctc_layer_idx = []
    plain_ms = timed(encode, a.reps)
    enc.interctc_layer_idx = idx

    # the three launches of one conditioned layer, on the encoder's own buffers
    (out, _), olens, _ = encode()
    B, T, D = out.shape
    M, V, Vp = B * T, a.vocab, _pitch(a.vocab)
    ws = {k[0][1]: t for k, t in enc._ws.items()}
    hs, logits, probs, x = ws["ic_split"], ws["ic_logits"], ws["ic_probs"], ws["x"].clone()
    h = torch.empty(B, T, D, device="cuda")
    pk = enc._packed
    with torch.no_grad():
        logits_ms = timed(lambda: ctc.logits(h, hs, out=logits), a.reps)
        soft_ms = timed(lambda: ops.softmax_rows_split(logits, probs), a.reps)
        cond_ms = timed(lambda: ops.linear(probs, pk["cond_w"], x, bias=pk["cond_b"], residual=x), a.reps)
    soft_bytes = M * (V + 2 * Vp) * 4

    # decoding
    torch.cuda.synchronize()
    greedy.ctc_greedy(waves)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    greedy.ctc_greedy(waves)
    torch.cuda.synchronize()
    greedy_s = time.perf_counter() - t0
    beam = Speech2Text(asr_model=model, asr_train_args=None, device="cuda", beam_size=a.beam, ctc_weight=1.0, maxlenratio=a.maxlenratio, nbest=1)
    beam.batch_decode(waves)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    hyps = beam.batch_decode(waves)
    torch.cuda.synchronize()
    beam_s = time.perf_counter() - t0

    print(json.dumps(dict(
        metric="self-conditioned intermediate CTC, LibriSpeech-100 scctc Conformer (18 x d 256, layers [6, 12], V 5000)",
        utts=a.utts, seconds=a.seconds, frames=int(T), rows=M, vocab=V,
        encoder=dict(conditioned_ms=enc_ms, plain_ms=plain_ms, per_conditioned_layer_ms=(enc_ms - plain_ms) / len(idx)),
        per_layer=dict(logits_gemm_ms=logits_ms, softmax_split_ms=soft_ms, conditioning_gemm_ms=cond_ms,
                       softmax_split_gbytes=soft_bytes / 1e9, softmax_split_tb_per_s=soft_bytes / soft_ms / 1e9,
                       softmax_split_share_of_hbm_peak=soft_bytes / (soft_ms * 1e-3) / HBM_BYTES_PER_S),
        ctc_greedy_utt_per_s=a.utts / greedy_s, ctc_beam=dict(utt_per_s=a.utts / beam_s, beam=a.beam, maxlenratio=a.maxlenratio,
                                                              hyp_len_utt0=len(hyps[0][0][2]) if hyps[0] else 0),
        peak_mem_gb=torch.cuda.max_memory_allocated() / 2 ** 30, gpu=gpu_info(), espnet_b200=espnet_b200.__version__)))


if __name__ == "__main__":
    main()
