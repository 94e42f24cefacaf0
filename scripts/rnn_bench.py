#!/usr/bin/env python
"""Throughput of the RNN model family on the CUDA path at the CommonVoice recipe shape
(egs2/commonvoice/asr1/conf/tuning/train_asr_rnn.yaml: VGG + 4 x BLSTMP 1024, 2-layer LSTM decoder 1024, AttLoc adim 1024, 10 channels,
filters 100), random weights, V 5000, joint CTC / attention beam search (ctc_weight 0.5).

Reports, as one JSON line:
  * utterances/s of Speech2Text.batch_decode over --utts utterances of --seconds s (after one warm-up batch);
  * the encoder's time split into VGG2L, the LSTM recurrences (input GEMM + per-step GEMM and cell kernel) and the projections (CUDA events
    around each part, one synchronised encoder pass);
  * the decoder's time per search step (RNNDecoder.step for all utterances x beam slots, CUDA events over --dec-steps steps);
  * parity of the encoder with the float64 CPU oracle (oracle/rnn.py) on the first --parity-frames feature frames of one utterance;
  * the card's name and power limit, read in the same run.

    python scripts/rnn_bench.py [--utts 64] [--seconds 30] [--beam 10] [--maxlenratio -64]
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


def config(V):
    return dict(token_list=["<blank>", "<unk>"] + [f"t{i}" for i in range(V - 3)] + ["<sos/eos>"], frontend="default",
                frontend_conf=dict(n_fft=512, hop_length=160, n_mels=80), specaug=None, normalize="utterance_mvn", normalize_conf={}, encoder="vgg_rnn",
                encoder_conf=dict(rnn_type="lstm", bidirectional=True, use_projection=True, num_layers=4, hidden_size=1024, output_size=1024,
                                  dropout=0.2),
                decoder="rnn", decoder_conf=dict(num_layers=2, hidden_size=1024, sampling_probability=0.0, dropout=0.2,
                                                 att_conf=dict(atype="location", adim=1024, aconv_chans=10, aconv_filts=100)),
                model_conf=dict(ctc_weight=0.5, lsm_weight=0.1, length_normalized_loss=False))


class _Timer:
    """CUDA events around every call of a method (encoder parts)."""

    def __init__(self, obj, name):
        self.ev, fn = [], getattr(obj, name)

        def wrapped(*a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = fn(*a, **k)
            e1.record()
            self.ev.append((e0, e1))
            return r

        setattr(obj, name, wrapped)

    def ms(self):
        return sum(a.elapsed_time(b) for a, b in self.ev)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, pl = out.stdout.strip().splitlines()[0].split(", ")
        return dict(name=name, power_limit=pl)
    except Exception as e:   # the card's name from torch at least
        return dict(name=torch.cuda.get_device_name(0), power_limit=f"unknown ({e})")


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--utts", type=int, default=64)
    p.add_argument("--seconds", type=float, default=30.0)
    p.add_argument("--beam", type=int, default=10)
    p.add_argument("--vocab", type=int, default=5000)
    p.add_argument("--maxlenratio", type=float, default=-64.0)
    p.add_argument("--dec-steps", type=int, default=20)
    p.add_argument("--parity-frames", type=int, default=96)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rnn_bench.py measures on a CUDA device; none is available")
    import espnet_b200
    from espnet_b200 import Speech2Text, ops
    from espnet_b200.asr_inference import build_model
    from oracle import rnn as orn

    torch.manual_seed(0)
    model = build_model(argparse.Namespace(**config(a.vocab))).cuda().eval()
    s2t = Speech2Text(asr_model=model, asr_train_args=None, device="cuda", beam_size=a.beam, ctc_weight=0.5, maxlenratio=a.maxlenratio,
                      nbest=1)
    g = torch.Generator().manual_seed(1)
    n_samp = int(a.seconds * 16000)
    waves = [0.1 * torch.randn(n_samp, generator=g) for _ in range(a.utts)]

    s2t.batch_decode(waves)          # warm-up: every shape of the timed run
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    hyps = s2t.batch_decode(waves)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0

    # encoder split
    enc = model.encoder
    speech, lens = s2t._to_batch(waves)
    timers = {k: _Timer(enc, m) for k, m in (("vgg", "_vgg"), ("recurrence", "_lstm_layer"), ("projections", "_project"))}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.no_grad():
        feats, flens = model.frontend(speech, lens)
        feats, flens = model.normalize(feats, flens)
        torch.cuda.synchronize()
        e0.record()
        out, olens, _ = enc(feats, flens)
        e1.record()
    torch.cuda.synchronize()
    enc_ms = e0.elapsed_time(e1)
    split = {k: t.ms() for k, t in timers.items()}
    for k in timers:
        delattr(enc, {"vgg": "_vgg", "recurrence": "_lstm_layer", "projections": "_project"}[k])

    # decoder step time for U * beam slots
    dec = model.decoder
    U, Tmax = out.shape[0], out.shape[1]
    n = U * a.beam
    with torch.no_grad():
        st = dec.init_memory(ops.split_from(out.reshape(U * Tmax, -1)), U, Tmax, olens.to(device="cuda", dtype=torch.int32), n, a.dec_steps)
        anc = torch.arange(n, dtype=torch.int32, device="cuda").view(n, 1).repeat(1, a.dec_steps)
        tok = torch.randint(0, a.vocab, (n,), dtype=torch.int32, device="cuda")
        dec.step(st, 0, tok, anc)
        torch.cuda.synchronize()
        d0, d1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        d0.record()
        for pos in range(1, a.dec_steps):
            dec.step(st, pos, tok, anc)
        d1.record()
    torch.cuda.synchronize()
    dec_ms = d0.elapsed_time(d1) / (a.dec_steps - 1)

    # parity of the encoder with the float64 oracle on a prefix of utterance 0
    Tp = min(a.parity_frames, int(flens[0]))
    with torch.no_grad():
        got, golens, _ = enc(feats[:1, :Tp].contiguous(), torch.tensor([Tp]))
    w = {k: v.detach().double().cpu() for k, v in enc.state_dict().items()}
    ref, _ = orn.rnn_encoder(feats[0, :Tp].double().cpu(), w, dict(num_layers=4, bidirectional=True, use_projection=True), "vgg_rnn")
    parity = float((got[0].double().cpu() - ref).abs().max())

    print(json.dumps(dict(
        metric="utterances/s, RNN model family (VGG + 4 x BLSTMP 1024, 2 x LSTM 1024 decoder, AttLoc), joint CTC/attention beam search",
        value=a.utts / wall, unit="utterances/s", utts=a.utts, seconds=a.seconds, beam=a.beam, vocab=a.vocab, ctc_weight=0.5,
        maxlenratio=a.maxlenratio, wall_s=wall, hyp_len_utt0=len(hyps[0][0][2]) if hyps[0] else 0,
        encoder=dict(total_ms=enc_ms, vgg_ms=split["vgg"], recurrence_ms=split["recurrence"], projections_ms=split["projections"],
                     frames_after_vgg=int(Tmax)),
        decoder=dict(ms_per_step=dec_ms, slots=n),
        parity=dict(against="oracle/rnn.py float64", frames=Tp, max_abs_diff=parity),
        peak_mem_gb=torch.cuda.max_memory_allocated() / 2 ** 30, gpu=gpu_info(), espnet_b200=espnet_b200.__version__)))


if __name__ == "__main__":
    main()
