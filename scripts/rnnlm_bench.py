#!/usr/bin/env python
"""Throughput of LM shallow fusion with the LSTM LM (SequentialRNNLM, lm: seq_rnn) on the CUDA path (one JSON line on stdout).

    python scripts/rnnlm_bench.py [--unit 650|2024] [--steps 3] [--warmup 2]

Model and decode settings are those of bench.py's conformer_large_lm_beam60_16x30s (Conformer-large + 6-layer decoder, V 5000, 16 x 30-s
synthetic waveforms, beam 60, ctc_weight 0.3, lm_weight 0.6, maxlenratio -64), so the two utt/s figures compare directly; the LM is a seeded
random-init 2-layer LSTM LM of the recipes' shapes: 2 x 650 (train_lm.yaml of aishell, tedlium2, csj, ...) or 2 x 2024 (gigaspeech, ...).

Reported:
  parity      LM log-probs at n = 960 slots after 8 steps with random parents, against the CPU oracle on 32 slots (atol 1e-4); the script
              exits non-zero on a mismatch
  throughput  utterances/s, median of the timed steps (CUDA events, L2 flushed between steps), waveforms resident on the device
  lm_step     one lm.step at n = 960 replayed in a CUDA graph (median over replays, L2 flushed before each)
  lm_gemms    the step's GEMMs timed launch by launch, achieved TFLOP/s against the algorithmic count (unpadded K)
  lstm_cell   espb_lstm_cell_f32 at n = 960 (median of repeated launches), achieved TB/s against its algorithmic bytes
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
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

WORKLOAD = "conformer_large_lm_beam60_16x30s"
LM_WEIGHT, N_SLOTS, HBM_TBS = 0.6, 960, 3.35   # 16 utterances x beam 60; H100 SXM data sheet


def gpu_identity():
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                           timeout=30)
        out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception:
        pass
    return out


def build_lm(unit, V):
    import espnet_b200

    torch.manual_seed(1)
    lm = espnet_b200.SequentialRNNLM(V, unit=unit, nlayers=2)
    with torch.no_grad():
        lm.encoder.weight.normal_(0, 1.0)
    return lm.cuda().eval()


def parity(lm, n, steps=8, check=32):
    from oracle.rnn_lm import OracleRNNLM

    g = torch.Generator().manual_seed(0)
    lm.ws_tag = "parity"
    st = lm.init_cache(n, steps)
    anc = torch.zeros(n, steps + 1, dtype=torch.int32, device="cuda")
    prefix = None
    for pos in range(steps):
        tok = torch.randint(0, lm.vocab_size, (n,), generator=g)
        if pos == 0:
            prefix = tok.view(n, 1)
        else:
            par = torch.randint(0, n, (n,), generator=g)
            anc[:, pos - 1] = par.to(torch.int32).cuda()
            prefix = torch.cat([prefix[par], tok.view(n, 1)], dim=1)
        logp = lm.step(st, pos, tok.to(torch.int32).cuda(), anc, None)
    sl = torch.randperm(n, generator=g)[:check]
    ref = OracleRNNLM(dict(lm.state_dict()), lm.nlayers).batch_score(prefix[sl])
    return float((logp[sl.cuda()].cpu() - ref).abs().max())


def median_ms(fn, reps, flush=None):
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


def lm_numbers(lm, n, flush):
    from espnet_b200 import ops
    from espnet_b200.lib import call, ptr

    E, H, L, V = lm.unit, lm.nhid, lm.nlayers, lm.vocab_size
    lm.ws_tag = "bench"
    st = lm.init_cache(n, 64)
    g = torch.Generator(device="cuda").manual_seed(0)
    anc = torch.randint(0, n, (n, 65), generator=g, dtype=torch.int32, device="cuda")
    tok = torch.randint(0, V, (n,), generator=g, dtype=torch.int32, device="cuda")
    step_dev = torch.full((1,), 5, dtype=torch.int32, device="cuda")
    for _ in range(3):
        lm.step(st, 0, tok, anc, step_dev)
    torch.cuda.synchronize()
    graph, cs = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    cs.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(cs):
        graph.capture_begin()
        lm.step(st, 0, tok, anc, step_dev)
        graph.capture_end()
    torch.cuda.current_stream().wait_stream(cs)
    for _ in range(3):
        graph.replay()
    step_ms = median_ms(graph.replay, 30, flush)
    # GEMMs launch by launch (eager step, CUDA events around each tensor-core GEMM)
    ops.gemm_profile = []
    flush.zero_()
    lm.step(st, 0, tok, anc, step_dev)
    torch.cuda.synchronize()
    prof, ops.gemm_profile = ops.gemm_profile, None
    alg = [2.0 * n * 4 * H * ((E if k == 0 else H) + H) for k in range(L)] + [2.0 * n * V * H]
    gemm_ms = sum(e0.elapsed_time(e1) for _, e0, e1 in prof)
    # the cell kernel alone
    gates = torch.randn(n, 4 * H, device="cuda", generator=g)
    xo = torch.zeros(2, n, st["h"].shape[-1], device="cuda")
    cell = lambda: call("espb_lstm_cell_f32", ptr(gates), ptr(anc), 65, 0, ptr(step_dev), ptr(st["h"]), ptr(st["c"]), L - 1, L, n, H,  # noqa: E731
                        st["h"].shape[-1], ptr(xo), xo[0].numel(), xo.shape[2])
    for _ in range(3):
        cell()
    cell_ms = median_ms(cell, 50)
    cell_bytes = 4 * n * (4 * H + H + 2 * H + 2 * H) + 4 * n     # gates, parent c, h' and c' to the ring, split h', anc
    return dict(
        lm_step_graph_ms=round(step_ms, 4),
        lm_gemms=dict(launches=len(prof), ms=round(gemm_ms, 4), algorithmic_gflop=round(sum(alg) / 1e9, 3),
                      achieved_TFLOPs=round(sum(alg) / gemm_ms / 1e9, 2), all_on_tensor_cores=len(prof) == L + 1),
        lstm_cell=dict(ms=round(cell_ms, 5), algorithmic_bytes=cell_bytes, achieved_TBps=round(cell_bytes / cell_ms / 1e9, 3),
                       share_of_datasheet_hbm=round(cell_bytes / cell_ms / 1e9 / HBM_TBS, 3)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--unit", type=int, default=650, help="LSTM width (2 layers)")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "rnnlm_bench.py measures on a CUDA device; there is no CPU fallback"
    import bench
    from gpu_util import speech2text

    torch.cuda.set_device(0)
    card = gpu_identity()
    cfg, secs, batch, beam, ctcw, mlr = bench.WORKLOADS[WORKLOAD]
    lm = build_lm(args.unit, cfg["vocab"])
    err = parity(lm, N_SLOTS)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")   # > 50 MB L2
    nums = lm_numbers(lm, N_SLOTS, flush)
    s2t = speech2text(cfg, bench.model_weights(cfg), beam_size=beam, ctc_weight=ctcw, maxlenratio=mlr, nbest=1, lm=lm, lm_weight=LM_WEIGHT)
    nsamp = secs * 16000
    speech = bench.waveforms(batch, nsamp).cuda()
    lens = torch.full((batch,), nsamp, dtype=torch.long)

    def step():
        enc, enc_lens = s2t.asr_model.encode(speech, lens)
        return s2t.beam_search.forward_batch(enc, enc_lens, s2t.asr_model.enc_split(enc), mlr, 0.0)

    for _ in range(args.warmup):
        step()
    ms = median_ms(step, args.steps, flush)
    line = dict(script="rnnlm_bench", card=card, lm=dict(type="SequentialRNNLM", rnn_type="lstm", unit=args.unit, nlayers=2, weight=LM_WEIGHT),
                decode=dict(model=WORKLOAD.split("_lm")[0], utterances=batch, seconds=secs, beam=beam, ctc_weight=ctcw, maxlenratio=mlr,
                            vocab=cfg["vocab"]),
                parity_max_abs_logp_err=err, utt_per_s=round(batch / (ms / 1e3), 3), step_ms=round(ms, 2), n_slots=N_SLOTS, **nums)
    print(json.dumps(line), flush=True)
    if not err <= 1e-4:
        print(f"LM log-probs differ from the oracle by {err:.3g} (> 1e-4)", file=sys.stderr)
        sys.exit(1)


if __name__ == "__main__":
    main()
