"""LM shallow fusion (SURVEY.md 8f-3): espnet_b200.TransformerLM as a second full scorer of the device-resident search, against n-best lists the
UNMODIFIED reference Speech2Text produced with its own TransformerLM (tests/golden/tiny_lm.npz, made by tests/golden/make_golden_lm.py): joint
CTC/attention + LM, attention + LM, CTC-only + LM.  CPU: host logic with the C-ABI entry points emulated; -m gpu: the CUDA kernels.
Tolerance: identical token sequences, total and per-scorer scores rtol 2e-4."""
import argparse
import os

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tiny_lm.npz")
DECODES = ["joint_lm", "att_lm", "ctc_lm"]


def _load():
    z = np.load(GOLD)
    cfg = {k: int(v) for k, v in zip(z["cfg_keys"].tolist(), z["cfg_vals"].tolist())}
    lmc = {k: int(v) for k, v in zip(z["lm_keys"].tolist(), z["lm_vals"].tolist())}
    w = {k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("w:")}
    return z, cfg, lmc, w


def _build(device):
    import espnet_b200
    from gpu_util import refbuild

    z, cfg, lmc, w = _load()
    model = espnet_b200.build_model(argparse.Namespace(**refbuild.model_yaml(cfg)))
    model.load_state_dict({k: v for k, v in w.items() if not k.startswith("lm.")}, strict=True)
    lm = espnet_b200.TransformerLM(cfg["vocab"], pos_enc="sinusoidal", **lmc)
    lm.load_state_dict({k[3:]: v for k, v in w.items() if k.startswith("lm.")}, strict=True)
    return z, model.to(device).eval(), lm.to(device).eval()


def _check(z, dn, hyps):
    n = int(z[f"dec:{dn}:n"])
    assert len(hyps) >= n > 0
    for i in range(n):
        h = hyps[i]
        assert h.yseq.tolist() == z[f"dec:{dn}:{i}:yseq"].tolist(), (dn, i)
        ref = float(z[f"dec:{dn}:{i}:score"])
        assert abs(h.score - ref) <= 2e-4 * max(1.0, abs(ref))
        for k, r in zip(("decoder", "ctc", "lm"), z[f"dec:{dn}:{i}:scores"].tolist()):
            if not np.isnan(r):
                assert abs(h.scores[k] - r) <= 2e-4 * max(1.0, abs(r)), (dn, k, h.scores[k], r)


def _search(model, lm, z, dn):
    from espnet_b200.search import BatchBeamSearch

    beam, cw, lw, mlr = z[f"dec:{dn}:params"].tolist()
    scorers = dict(decoder=model.decoder if cw != 1.0 else None, ctc=model.ctc, lm=lm)
    weights = dict(decoder=1.0 - cw, ctc=cw, lm=lw, length_bonus=0.0)
    bs = BatchBeamSearch(scorers, weights, int(beam), model.vocab_size, model.sos, model.eos, token_list=model.token_list,
                         pre_beam_score_key=None if cw == 1.0 else "full")
    return bs, mlr


def test_refused_attention_head_size():
    """The decoder step's self-attention kernel covers heads of up to 128 dimensions: wider heads are refused at construction."""
    import espnet_b200

    with pytest.raises(NotImplementedError):
        espnet_b200.lm.TransformerLM(vocab_size=10, att_unit=512, head=2)
    with pytest.raises(NotImplementedError):
        espnet_b200.decoder.TransformerDecoder(vocab_size=10, encoder_output_size=512, attention_heads=2, num_blocks=1)
    espnet_b200.lm.TransformerLM(vocab_size=10, att_unit=512, head=4, layer=1)
    espnet_b200.decoder.TransformerDecoder(vocab_size=10, encoder_output_size=512, attention_heads=4, num_blocks=1)


@pytest.mark.parametrize("dn", DECODES)
def test_lm_fusion_host_logic_vs_reference_fixture(dn, monkeypatch):
    import emu_backend
    from oracle import frontend as OF

    emu_backend.install_search(monkeypatch)
    z, model, lm = _build("cpu")
    feats = OF.utterance_mvn(OF.frontend_forward(torch.from_numpy(z["wave"]), model.frontend.logmel.melmat))[None]
    enc, enc_lens, _ = model.encoder(feats, torch.tensor([feats.shape[1]]))
    bs, mlr = _search(model, lm, z, dn)
    hyps = bs.forward_batch(enc, enc_lens, model.enc_split(enc), mlr, 0.0)[0]
    _check(z, dn, hyps)
    assert "espb_track_scores_f32" in emu_backend.calls and "espb_gather_rows_split_f32" in emu_backend.calls


@pytest.mark.gpu
@pytest.mark.parametrize("dn", DECODES)
def test_lm_fusion_cuda_vs_reference_fixture(dn):
    import espnet_b200

    z, model, lm = _build("cuda")
    beam, cw, lw, mlr = z[f"dec:{dn}:params"].tolist()
    s2t = espnet_b200.Speech2Text(asr_model=model, device="cuda", beam_size=int(beam), ctc_weight=cw, lm_weight=lw, maxlenratio=mlr, nbest=10, lm=lm)
    for _ in range(2):       # second call: cached state / CUDA graphs
        res = s2t(z["wave"])
        _check(z, dn, [r[3] for r in res])


@pytest.mark.gpu
def test_lm_fusion_batch_vs_single_cuda():
    """Ragged batch with LM fusion == the same utterances decoded one by one."""
    import espnet_b200
    from gpu_util import refbuild

    z, model, lm = _build("cuda")
    s2t = espnet_b200.Speech2Text(asr_model=model, device="cuda", beam_size=4, ctc_weight=0.3, lm_weight=0.6, maxlenratio=-10.0, nbest=4, lm=lm)
    waves = [refbuild.waveform(20 + i, n) for i, n in enumerate([12000, 8000, 15000])]
    batch = s2t.batch_decode(waves)
    for wv, got in zip(waves, batch):
        one = s2t(wv)
        assert [h[3].yseq.tolist() for h in got] == [h[3].yseq.tolist() for h in one]
        for a, b in zip(got, one):
            assert abs(a[3].score - b[3].score) <= 1e-5 * max(1.0, abs(b[3].score))
