"""LSTM LM shallow fusion: espnet_b200.SequentialRNNLM (lm: seq_rnn) as a full scorer of the device-resident search and of the streaming search,
against what the UNMODIFIED reference produced with its own SequentialRNNLM (tests/golden/rnnlm.npz from make_golden_rnnlm.py,
tests/golden/streaming_rnnlm.npz from make_golden_streaming_rnnlm.py).  CPU: the oracle, loading and refusals, and the host logic with the C-ABI
entry points emulated (tests/emu_rnnlm.py); -m gpu: the CUDA kernels, including the recipe shapes 2 x 650 and 2 x 2024.
Tolerance as test_lm_fusion.py: identical token sequences, total and per-scorer scores rtol 2e-4 (streaming also atol 2e-3)."""
import argparse
import json
import os

import numpy as np
import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SETTINGS = [("A", "joint_lm"), ("A", "att_lm"), ("A", "ctc_lm"), ("B", "joint_lm"), ("C", "joint_lm")]


def _z():
    return np.load(os.path.join(GOLDEN, "rnnlm.npz"))


def _lm_weights(z, name):
    p = f"{name}:w:"
    return {k[len(p):]: torch.from_numpy(z[k]) for k in z.files if k.startswith(p)}


def _lm(z, name, device="cpu"):
    import espnet_b200

    conf = json.loads(str(z["lms"]))[name]
    lm = espnet_b200.SequentialRNNLM(json.loads(str(z["cfg"]))["vocab"], rnn_type="lstm", dropout_rate=0.2, **conf)
    lm.load_state_dict(_lm_weights(z, name), strict=True)
    return lm.to(device).eval()


def _asr(device):
    import espnet_b200
    from gpu_util import refbuild

    z = _z()
    cfg = json.loads(str(z["cfg"]))
    t = np.load(os.path.join(GOLDEN, "tiny_lm.npz"))
    w = {k[2:]: torch.from_numpy(t[k]) for k in t.files if k.startswith("w:") and not k.startswith("w:lm.")}
    model = espnet_b200.build_model(argparse.Namespace(**refbuild.model_yaml(cfg)))
    model.load_state_dict(w, strict=True)
    return model.to(device).eval()


def _check(z, key, hyps):
    n = int(z[f"{key}:n"])
    assert len(hyps) >= n > 0
    for i in range(n):
        h = hyps[i]
        assert h.yseq.tolist() == z[f"{key}:{i}:yseq"].tolist(), (key, i)
        ref = float(z[f"{key}:{i}:score"])
        assert abs(float(h.score) - ref) <= 2e-4 * max(1.0, abs(ref)), (key, i, float(h.score), ref)
        for k, r in zip(("decoder", "ctc", "lm"), z[f"{key}:{i}:scores"].tolist()):
            if not np.isnan(r):
                assert abs(float(h.scores[k]) - r) <= 2e-4 * max(1.0, abs(r)), (key, k, float(h.scores[k]), r)


# ------------------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name", ["A", "B", "C"])
def test_oracle_logprobs_vs_reference_batch_score(name):
    from oracle.rnn_lm import OracleRNNLM

    z = _z()
    o = OracleRNNLM(_lm_weights(z, name), json.loads(str(z["lms"]))[name]["nlayers"])
    ys = torch.from_numpy(z["prefixes"])
    ref = z[f"{name}:prefix_logp"]
    for t in range(ys.shape[1]):
        assert np.abs(o.batch_score(ys[:, :t + 1]).numpy() - ref[t]).max() <= 1e-5, t


@pytest.mark.parametrize("name,dn", SETTINGS)
def test_oracle_nbest_vs_reference_fixture(name, dn):
    import oracle
    from oracle import encoder as OE
    from oracle.rnn_lm import OracleRNNLM
    from oracle.search import OracleDecoder, batch_beam_search

    z = _z()
    cfg = json.loads(str(z["cfg"]))
    t = np.load(os.path.join(GOLDEN, "tiny_lm.npz"))
    w = {k[2:]: torch.from_numpy(t[k]) for k in t.files if k.startswith("w:") and not k.startswith("w:lm.")}
    beam, cw, lw, mlr = z[f"{name}:{dn}:params"].tolist()
    o = oracle.OracleSpeech2Text(cfg, w, beam_size=int(beam), ctc_weight=cw, maxlenratio=mlr)
    enc = o.encode(torch.from_numpy(z["wave"]))
    logp = torch.log_softmax(OE.ctc_logits(enc, o.w), dim=-1)
    dec = OracleDecoder(o.w, cfg["heads"], cfg["dec_layers"]) if cw != 1.0 else None
    lm = OracleRNNLM(_lm_weights(z, name), json.loads(str(z["lms"]))[name]["nlayers"])
    res = batch_beam_search(enc, dec, logp, beam_size=int(beam), ctc_weight=cw, vocab=cfg["vocab"], sos=cfg["vocab"] - 1, eos=cfg["vocab"] - 1,
                            maxlenratio=mlr, lm=lm, lm_weight=lw)[:10]
    assert len(res) == int(z[f"{name}:{dn}:n"])
    _check(z, f"{name}:{dn}", res)


@pytest.mark.parametrize("name", ["A", "B", "C"])
def test_reference_state_dict_loads_strictly(name):
    z = _z()
    lm = _lm(z, name)
    assert sorted(lm.state_dict()) == sorted(_lm_weights(z, name))
    if name == "C":
        assert lm.decoder.weight is lm.encoder.weight
    assert not any(isinstance(m, torch.nn.LSTM) for m in lm.modules())


def test_refused_configurations():
    import espnet_b200

    for t in ("gru", "GRU", "rnn_tanh", "RNN_RELU"):
        with pytest.raises(NotImplementedError):
            espnet_b200.SequentialRNNLM(10, unit=8, rnn_type=t)
    with pytest.raises(ValueError):
        espnet_b200.SequentialRNNLM(10, unit=8, rnn_type="transformer")
    with pytest.raises(ValueError):
        espnet_b200.SequentialRNNLM(10, unit=8, nhid=12, tie_weights=True)
    assert espnet_b200.SequentialRNNLM(10, unit=8, rnn_type="LsTm", dropout_rate=0.5).nhid == 8


@pytest.mark.parametrize("with_key", [True, False])
def test_build_lm_from_file_seq_rnn(tmp_path, with_key):
    """``lm: seq_rnn`` and a config without an ``lm`` key (the reference's lm_choices default) both build SequentialRNNLM; the checkpoint's
    ``lm.`` prefix (ESPnetLanguageModel) is stripped."""
    import yaml

    from espnet_b200 import SequentialRNNLM, build_lm_from_file
    from gpu_util import refbuild

    z = _z()
    conf = dict(json.loads(str(z["lms"]))["B"], rnn_type="lstm")
    y = dict(token_list=refbuild.token_list(50), lm_conf=conf)
    if with_key:
        y["lm"] = "seq_rnn"
    (tmp_path / "lm.yaml").write_text(yaml.safe_dump(y))
    torch.save({"lm." + k: v for k, v in _lm_weights(z, "B").items()}, tmp_path / "lm.pth")
    lm, args = build_lm_from_file(str(tmp_path / "lm.yaml"), str(tmp_path / "lm.pth"), device="cpu")
    assert isinstance(lm, SequentialRNNLM) and lm.nlayers == 3 and lm.nhid == 44
    for k, v in _lm_weights(z, "B").items():
        assert torch.equal(lm.state_dict()[k], v), k


def _bs(model, lm, z, key):
    from espnet_b200.search import BatchBeamSearch

    beam, cw, lw, mlr = z[f"{key}:params"].tolist()
    scorers = dict(decoder=model.decoder if cw != 1.0 else None, ctc=model.ctc, lm=lm)
    weights = dict(decoder=1.0 - cw, ctc=cw, lm=lw, length_bonus=0.0)
    return BatchBeamSearch(scorers, weights, int(beam), model.vocab_size, model.sos, model.eos, token_list=model.token_list,
                           pre_beam_score_key=None if cw == 1.0 else "full"), mlr


@pytest.mark.parametrize("name,dn", SETTINGS)
def test_host_logic_vs_reference_fixture(name, dn, monkeypatch):
    import emu_backend
    import emu_rnnlm
    from oracle import frontend as OF

    emu_rnnlm.install(monkeypatch)
    z = _z()
    model, lm = _asr("cpu"), _lm(z, name)
    feats = OF.utterance_mvn(OF.frontend_forward(torch.from_numpy(z["wave"]), model.frontend.logmel.melmat))[None]
    enc, enc_lens, _ = model.encoder(feats, torch.tensor([feats.shape[1]]))
    bs, mlr = _bs(model, lm, z, f"{name}:{dn}")
    hyps = bs.forward_batch(enc, enc_lens, model.enc_split(enc), mlr, 0.0)[0]
    _check(z, f"{name}:{dn}", hyps)
    assert "espb_rnnlm_gather_f32" in emu_backend.calls and "espb_lstm_cell_f32" in emu_backend.calls


def _streaming(device, n_streams=1):
    import espnet_b200

    base = np.load(os.path.join(GOLDEN, "streaming_search.npz"))
    zs = np.load(os.path.join(GOLDEN, "streaming_rnnlm.npz"))
    y = json.loads(str(base["yaml"]))
    model = espnet_b200.build_model(argparse.Namespace(**y))
    model.load_state_dict({k[2:]: torch.from_numpy(base[k]) for k in base.files if k.startswith("w:")}, strict=True)
    model = model.to(device).eval()
    lm = espnet_b200.SequentialRNNLM(len(y["token_list"]), **json.loads(str(zs["lm_conf"])))
    lm.load_state_dict({k[3:]: torch.from_numpy(zs[k]) for k in zs.files if k.startswith("lm:")}, strict=True)
    wave, pushes = torch.from_numpy(base["wave"]), base["pushes"].tolist()
    for name, kw in json.loads(str(zs["settings"])).items():
        s2t = espnet_b200.Speech2TextStreaming(model, n_streams=n_streams, device=device, lm=lm.to(device).eval(), **kw)
        pos = 0
        for i, n in enumerate(pushes):
            chunk = wave[pos:pos + n]
            res = s2t(chunk if n_streams == 1 else chunk[None].repeat(n_streams, 1), is_final=(i == len(pushes) - 1))
            pos += n
            for per_stream in ([res] if n_streams == 1 else res):
                assert len(per_stream) == int(zs[f"{name}:{i}:n"]), (name, i, len(per_stream))
                for j, (_, _, token_int, hyp) in enumerate(per_stream):
                    key = f"{name}:{i}:{j}"
                    assert hyp.yseq.tolist() == zs[key + ":yseq"].tolist(), key
                    assert token_int == zs[key + ":token_int"].tolist(), key
                    ref = float(zs[key + ":score"])
                    assert abs(float(hyp.score) - ref) <= 2e-4 * abs(ref) + 2e-3, (key, float(hyp.score), ref)
                    for k, v in hyp.scores.items():
                        r = float(zs[f"{key}:score:{k}"])
                        assert abs(float(v) - r) <= 2e-4 * abs(r) + 2e-3, (key, k, float(v), r)


def test_streaming_host_logic_vs_reference_fixture(monkeypatch):
    import emu_backend
    import emu_rnnlm

    emu_rnnlm.install(monkeypatch)
    emu_backend.install_frontend(monkeypatch)
    _streaming("cpu")
    assert "espb_lstm_cell_f32" in emu_backend.calls


def test_reference_beam_search_drives_our_rnnlm(monkeypatch):
    """The reference's own BatchBeamSearch (unmodified, oracle/_ref) with our decoder, CTC prefix scorer and SequentialRNNLM.batch_score as
    scorers reproduces the reference Speech2Text's n-best with LM A (joint_lm)."""
    import emu_rnnlm
    from oracle import frontend as OF
    from test_scorer_interface import _reference

    _reference()
    from espnet2.legacy.nets.batch_beam_search import BatchBeamSearch
    from espnet2.legacy.nets.scorer_interface import BatchScorerInterface

    from espnet_b200 import SequentialRNNLM, integration

    emu_rnnlm.install(monkeypatch)
    z = _z()
    model, lm = _asr("cpu"), _lm(z, "A")
    lm.__class__ = type("SequentialRNNLM", (SequentialRNNLM, BatchScorerInterface), {})   # what the reference's BeamSearch type-checks
    feats = OF.utterance_mvn(OF.frontend_forward(torch.from_numpy(z["wave"]), model.frontend.logmel.melmat))[None]
    enc, _, _ = model.encoder(feats, torch.tensor([feats.shape[1]]))
    decoder = model.decoder
    decoder.__class__ = integration.register()["decoder"]["b200_transformer"]
    beam, cw, lw, mlr = z["A:joint_lm:params"].tolist()
    bs = BatchBeamSearch(beam_size=int(beam), weights=dict(decoder=1.0 - cw, ctc=cw, lm=lw, length_bonus=0.0),
                         scorers=dict(decoder=decoder, ctc=integration.ctc_prefix_scorer(model.ctc, model.eos), lm=lm),
                         sos=model.sos, eos=model.eos, vocab_size=model.vocab_size, token_list=model.token_list, pre_beam_score_key="full")
    hyps = bs(x=enc[0], maxlenratio=mlr, minlenratio=0.0)
    _check(z, "A:joint_lm", hyps[:10])


# ------------------------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["tc2", "simt"])
@pytest.mark.parametrize("name,dn", SETTINGS)
def test_speech2text_cuda_vs_reference_fixture(name, dn, mode):
    import espnet_b200
    from espnet_b200 import ops

    z = _z()
    model, lm = _asr("cuda"), _lm(z, name, "cuda")
    beam, cw, lw, mlr = z[f"{name}:{dn}:params"].tolist()
    prev = ops.gemm_mode()
    ops.set_gemm_mode(mode)
    try:
        s2t = espnet_b200.Speech2Text(asr_model=model, device="cuda", beam_size=int(beam), ctc_weight=cw, lm_weight=lw, maxlenratio=mlr, nbest=10,
                                      lm=lm)
        for _ in range(2):       # second call: cached state / CUDA graphs
            _check(z, f"{name}:{dn}", [r[3] for r in s2t(z["wave"])])
    finally:
        ops.set_gemm_mode(prev)


@pytest.mark.gpu
def test_ragged_batch_equals_single_cuda():
    import espnet_b200
    from gpu_util import refbuild

    z = _z()
    model, lm = _asr("cuda"), _lm(z, "A", "cuda")
    s2t = espnet_b200.Speech2Text(asr_model=model, device="cuda", beam_size=4, ctc_weight=0.3, lm_weight=0.6, maxlenratio=-10.0, nbest=4, lm=lm)
    waves = [refbuild.waveform(20 + i, n) for i, n in enumerate([12000, 8000, 15000])]
    batch = s2t.batch_decode(waves)
    for wv, got in zip(waves, batch):
        one = s2t(wv)
        assert [h[3].yseq.tolist() for h in got] == [h[3].yseq.tolist() for h in one]
        for a, b in zip(got, one):
            assert abs(a[3].score - b[3].score) <= 1e-5 * max(1.0, abs(b[3].score))


@pytest.mark.gpu
@pytest.mark.parametrize("n_streams", [1, 3])
def test_streaming_cuda_vs_reference_fixture(n_streams):
    _streaming("cuda", n_streams)


@pytest.mark.gpu
def test_lstm_cell_kernel_vs_torch():
    from espnet_b200.lib import call, ptr

    g = torch.Generator().manual_seed(3)
    n, H, Hp, L, layer, pos = 37, 50, 52, 2, 1, 3
    gates = (torch.randn(n, 4 * H, generator=g) * 3).cuda()
    h_ring, c_ring = torch.randn(2, L, n, Hp, generator=g).cuda(), torch.randn(2, L, n, Hp, generator=g).cuda()
    anc = torch.randint(0, n, (n, 6), generator=g, dtype=torch.int32).cuda()
    out = torch.zeros(2, n, 2 * Hp, device="cuda")
    step = torch.tensor([pos - 1], dtype=torch.int32, device="cuda")
    h0, c0 = h_ring.clone(), c_ring.clone()
    call("espb_lstm_cell_f32", ptr(gates), ptr(anc), 6, 1, ptr(step), ptr(h_ring), ptr(c_ring), layer, L, n, H, Hp, ptr(out), n * 2 * Hp, 2 * Hp)
    torch.cuda.synchronize()
    p = anc[:, pos - 1].long()
    i, f, gg, o = gates.chunk(4, dim=-1)
    c = torch.sigmoid(f) * c0[(pos - 1) & 1, layer][p][:, :H] + torch.sigmoid(i) * torch.tanh(gg)
    h = torch.sigmoid(o) * torch.tanh(c)
    assert (c_ring[pos & 1, layer, :, :H] - c).abs().max() <= 1e-6 * max(1.0, float(c.abs().max()))
    assert (h_ring[pos & 1, layer, :, :H] - h).abs().max() <= 1e-6
    hn = h_ring[pos & 1, layer, :, :H].contiguous()       # the split operand: tf32 hi plane and truncated remainder (common.cuh)
    hi = (hn.view(torch.int32) & -8192).view(torch.float32)
    assert torch.equal(out[0, :, :H], hi) and torch.equal(out[1, :, :H], ((hn - hi).view(torch.int32) & -8192).view(torch.float32))
    assert torch.equal(out[:, :, H:], torch.zeros_like(out[:, :, H:]))
    keep = torch.ones(2, L, dtype=torch.bool)
    keep[pos & 1, layer] = False
    assert torch.equal(h_ring[keep], h0[keep]) and torch.equal(c_ring[keep], c0[keep]) and torch.equal(h_ring[pos & 1, layer, :, H:], h0[pos & 1, layer, :, H:])


def _recipe_lm(unit, V=5000, seed=0):
    import espnet_b200

    torch.manual_seed(seed)
    lm = espnet_b200.SequentialRNNLM(V, unit=unit, nlayers=2)
    with torch.no_grad():
        lm.encoder.weight.normal_(0, 1.0)
    return lm


def run_recipe_steps(lm, n, steps, seed=0, check_slots=64):
    """``steps`` lm.step calls at n slots with random tokens and random parents written into anc (every other step with a device-side step
    counter).  Returns the max |log-prob - oracle| over ``check_slots`` slots at the last step and at the middle step, and the number of
    tensor-core GEMMs of one step."""
    from espnet_b200 import ops
    from oracle.rnn_lm import OracleRNNLM

    dev = lm.decoder.weight.device
    g = torch.Generator().manual_seed(seed)
    V = lm.vocab_size
    st = lm.init_cache(n, steps)
    anc = torch.zeros(n, steps + 1, dtype=torch.int32, device=dev)
    step_dev = torch.zeros(1, dtype=torch.int32, device=dev)
    prefix = None
    oracle = OracleRNNLM({k: v for k, v in lm.state_dict().items()}, lm.nlayers)
    errs, n_tc = [], None
    for pos in range(steps):
        tok = torch.randint(0, V, (n,), generator=g)
        if pos == 0:
            prefix = tok.view(n, 1)
        else:
            par = torch.randint(0, n, (n,), generator=g)
            anc[:, pos - 1] = par.to(torch.int32).to(dev)
            prefix = torch.cat([prefix[par], tok.view(n, 1)], dim=1)
        if pos == 1:
            ops.gemm_profile = []
        if pos & 1:
            step_dev.fill_(pos)
            logp = lm.step(st, 0, tok.to(torch.int32).to(dev), anc, step_dev)
        else:
            logp = lm.step(st, pos, tok.to(torch.int32).to(dev), anc, None)
        if pos == 1:
            torch.cuda.synchronize()
            n_tc, ops.gemm_profile = len(ops.gemm_profile), None
        if pos in (steps // 2, steps - 1):
            sl = torch.randperm(n, generator=g)[:check_slots]
            ref = oracle.batch_score(prefix[sl])
            errs.append(float((logp[sl.to(dev)].cpu() - ref).abs().max()))
    return max(errs), n_tc


@pytest.mark.gpu
@pytest.mark.parametrize("unit", [650, 2024])
def test_recipe_shape_steps_vs_oracle_on_tensor_cores(unit):
    """2 x 650 and 2 x 2024, V 5000, n = 960 slots (16 utterances x beam 60): 24 steps against the oracle; every LM GEMM on the tensor cores."""
    lm = _recipe_lm(unit).cuda().eval()
    err, n_tc = run_recipe_steps(lm, 960, 24)
    assert n_tc == lm.nlayers + 1
    assert err <= 1e-4, err
