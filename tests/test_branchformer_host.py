"""Branchformer encoder on a CPU-only box: the oracle against the reference fixtures, and the host logic of espnet_b200.BranchformerEncoder
(weight packing per merge method and per branch set, the merge operand layouts, the attention-layer ordinals of the rel-pos tables, GEMM
descriptors, kernel order) with the C-ABI entry points replaced by their torch restatements (tests/emu_bf.py)."""
import argparse
import os
import sys

import numpy as np
import pytest
import torch
import yaml

import emu_backend
import emu_bf
from golden_util import DEC_NAMES, GOLDEN_DIR, decode_params, decode_results, load

sys.path.insert(0, GOLDEN_DIR)
import refbuild_bf  # noqa: E402

TAGS = ["A", "B", "C", "D", "E"]   # concat, learned_ave, fixed_ave [0, 0.3, 1], use_attn=False, use_cgmlp=False


def load_enc(tag):
    z = np.load(os.path.join(GOLDEN_DIR, "branchformer_enc.npz"))
    cfg = dict(zip(z[f"{tag}:cfg_keys"].tolist(), (int(v) for v in z[f"{tag}:cfg_vals"])))
    return z, cfg, z[f"{tag}:cgmlp_weight"].tolist(), refbuild_bf.fixture_weights(z, prefix=f"{tag}:")


def load_bf():
    z, cfg, _ = load("bf")
    return z, cfg, refbuild_bf.fixture_weights(z)


def build_encoder(cfg, cw, w=None):
    import espnet_b200

    enc = espnet_b200.BranchformerEncoder(80, **refbuild_bf.encoder_conf(cfg, cw))
    if w is not None:
        enc.load_state_dict({k[len("encoder."):]: v for k, v in w.items() if k.startswith("encoder.")}, strict=True)
    return enc.eval()


def _random_norms(enc, seed):
    """LayerNorm affines away from 1 / 0 and every bias non-zero; the learned_ave weight projections scaled up so that the two merge
    weights of an utterance are far from 0.5 / 0.5 (a swapped branch or a pooled padded row would show)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in enc.named_parameters():
            if "norm" in n or n.endswith("bias"):
                p.add_(0.2 * torch.randn(p.shape, generator=g))
            if "weight_proj" in n or "pooling_proj" in n:
                p.mul_(8.0)
    return {"encoder." + k: v.detach().clone() for k, v in enc.state_dict().items()}


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_vs_reference_encoder_fixture(tag):
    from oracle.branchformer import branchformer_encode

    z, cfg, cw, w = load_enc(tag)
    out, layers = branchformer_encode(torch.from_numpy(z[f"{tag}:feats"]), w, cfg["heads"], cfg["enc_layers"], cw, return_layers=True)
    assert out.shape[0] == int(z[f"{tag}:olens"][0])
    for i in range(1, cfg["enc_layers"] + 1):
        np.testing.assert_allclose(layers[i].numpy(), z[f"{tag}:layer{i}"], atol=1e-5, rtol=1e-5)
    np.testing.assert_allclose(out.numpy(), z[f"{tag}:out"], atol=1e-5, rtol=1e-5)


def test_oracle_vs_reference_speech2text_fixture():
    from oracle import ctc_logits
    from oracle.branchformer import BranchformerSpeech2Text

    z, cfg, w = load_bf()
    assert cfg["encoder"] == "branchformer"
    o = BranchformerSpeech2Text(cfg, w)
    enc = o.encode(torch.from_numpy(z["wave"]))
    np.testing.assert_allclose(enc.numpy(), z["enc"], atol=1e-5, rtol=1e-5)
    np.testing.assert_allclose(ctc_logits(enc, o.w).numpy(), z["ctc_logits"], atol=1e-4, rtol=1e-5)
    for dn in DEC_NAMES:
        res = BranchformerSpeech2Text(cfg, w, nbest=10, **decode_params(z, dn))(z["wave"])
        gold = decode_results(z, dn)
        assert len(res) == len(gold), dn
        for (_, _, _, h), (yseq, score, _) in zip(res, gold):
            assert h.yseq.tolist() == yseq, dn
            assert abs(float(h.score) - score) <= 1e-4 * max(1.0, abs(score)), dn


@pytest.mark.parametrize("tag", TAGS)
def test_encoder_host_logic_vs_reference_fixture(tag, monkeypatch):
    emu_bf.install(monkeypatch)
    z, cfg, cw, w = load_enc(tag)
    enc = build_encoder(cfg, cw, w)
    enc.trace = []
    feats = torch.from_numpy(z[f"{tag}:feats"])[None]
    out, olens, _ = enc(feats, torch.tensor([feats.shape[1]]))
    assert int(olens[0]) == int(z[f"{tag}:olens"][0])
    for i in range(1, cfg["enc_layers"] + 1):
        np.testing.assert_allclose(enc.trace[i][0].numpy(), z[f"{tag}:layer{i}"], atol=5e-5, rtol=1e-5)
    np.testing.assert_allclose(out[0].numpy(), z[f"{tag}:out"], atol=5e-5, rtol=1e-5)
    L, calls = cfg["enc_layers"], emu_backend.calls
    n_attn = sum(1 for lyr in enc.encoders if lyr.attn is not None)
    n_mlp = sum(1 for lyr in enc.encoders if lyr.cgmlp is not None)
    assert calls.count("espb_csgu_f32") == n_mlp and calls.count("espb_qu_qv_f32") == n_attn
    assert calls.count("espb_branch_pool_f32") == (L if tag == "B" else 0)
    assert calls.count("espb_branch_merge_f32") == {"B": L, "C": 1}.get(tag, 0)


RAGGED = {"A": [150, 47, 103, 7], "B": [31, 150, 7, 19, 88], "C": [7, 120, 61], "D": [95, 7, 40], "E": [60, 200, 7]}


@pytest.mark.parametrize("tag", TAGS)
def test_encoder_ragged_batch_host_logic(tag, monkeypatch):
    """Per-utterance semantics: own attention keys, own CSGU conv boundaries and, for learned_ave, pooling over the utterance's own frames
    only (7 feature frames give one encoder frame).  Padded output rows are 0."""
    from oracle.branchformer import branchformer_encode

    emu_bf.install(monkeypatch)
    _, cfg, cw, _ = load_enc(tag)
    torch.manual_seed(11)
    enc = build_encoder(cfg, cw)
    w = _random_norms(enc, 12)
    lens = RAGGED[tag]
    g = torch.Generator().manual_seed(13)
    feats = torch.randn(len(lens), max(lens), 80, generator=g)     # padded frames are garbage, not zeros
    out, olens, _ = enc(feats, torch.tensor(lens))
    for i, n in enumerate(lens):
        ref = branchformer_encode(feats[i, :n], w, cfg["heads"], cfg["enc_layers"], cw)
        T = ref.shape[0]
        assert int(olens[i]) == T
        np.testing.assert_allclose(out[i, :T].numpy(), ref.numpy(), atol=5e-5, rtol=1e-5)
        assert not out[i, T:].any()


def test_speech2text_host_logic_vs_reference_fixture(monkeypatch):
    """Waveform -> Branchformer encoder -> CTC head + decoder -> beam search, every kernel emulated, against the reference Speech2Text."""
    import espnet_b200
    from espnet_b200.search import BatchBeamSearch

    emu_backend.install_search(monkeypatch)
    emu_backend.install_frontend(monkeypatch)
    emu_bf.install(monkeypatch)
    z, cfg, w = load_bf()
    model = espnet_b200.build_model(argparse.Namespace(**refbuild_bf.model_yaml(cfg)))
    model.load_state_dict(w, strict=True)
    model.eval()
    wave = torch.from_numpy(z["wave"])
    enc, enc_lens = model.encode(wave[None], torch.tensor([wave.numel()]))
    np.testing.assert_allclose(enc[0].numpy(), z["enc"], atol=3e-4, rtol=1e-4)
    for dn in ("joint", "att", "ctc"):
        kw = decode_params(z, dn)
        cw = kw["ctc_weight"]
        scorers = dict(decoder=model.decoder if cw != 1.0 else None, ctc=model.ctc)
        weights = dict(decoder=1.0 - cw, ctc=cw, lm=1.0, ngram=0.9, length_bonus=kw["penalty"])
        bs = BatchBeamSearch(scorers, weights, kw["beam_size"], len(model.token_list), model.sos, model.eos, token_list=model.token_list,
                             pre_beam_score_key=None if cw == 1.0 else "full", normalize_length=kw["normalize_length"])
        hyps = bs.forward_batch(enc, enc_lens, model.enc_split(enc), kw["maxlenratio"], kw["minlenratio"])[0][:10]
        gold = decode_results(z, dn)
        assert len(hyps) == len(gold), dn
        for h, (yseq, score, _) in zip(hyps, gold):
            assert h.yseq.tolist() == yseq, dn
            assert abs(h.score - score) <= 3e-4 * max(1.0, abs(score)), dn


def test_state_dict_loads_strict_from_the_reference():
    """The reference's names and shapes per layer: concat merge_proj Linear(2D, D); learned_ave pooling / weight projections; fixed_ave
    layers with weight 0 / 1 without the dropped branch and its norm; Identity merge_proj (no parameters) with one branch."""
    import espnet_b200

    for tag in TAGS:
        z, cfg, cw, w = load_enc(tag)
        enc = build_encoder(cfg, cw, w)
        assert list(enc.state_dict()) == [k[len("encoder."):] for k in w]    # the reference's order too
    _, cfg, cw, _ = load_enc("C")
    enc = build_encoder(cfg, cw)
    assert enc.encoders[0].cgmlp is None and enc.encoders[0].norm_mlp is None and enc.encoders[0].merge_proj.weight.shape == (64, 64)
    assert enc.encoders[2].attn is None and enc.encoders[2].norm_mha is None
    z, cfg, w = load_bf()
    espnet_b200.build_model(argparse.Namespace(**refbuild_bf.model_yaml(cfg))).load_state_dict(w, strict=True)


@pytest.mark.parametrize("kw", [dict(input_layer="linear"), dict(input_layer="conv2d8"), dict(rel_pos_type="legacy"),
                                dict(pos_enc_layer_type="abs_pos"), dict(attention_layer_type="selfattn"),
                                dict(attention_layer_type="fast_selfattn", pos_enc_layer_type="abs_pos"), dict(use_linear_after_conv=True),
                                dict(gate_activation="tanh"), dict(cgmlp_conv_kernel=30), dict(cgmlp_linear_units=8194), dict(zero_triu=True),
                                dict(qk_norm=True), dict(output_size=80, attention_heads=4)])
def test_unsupported_options_are_refused(kw):
    import espnet_b200

    with pytest.raises(NotImplementedError):
        espnet_b200.BranchformerEncoder(80, **kw)


def test_reference_argument_errors():
    import espnet_b200

    with pytest.raises(ValueError):
        espnet_b200.BranchformerEncoder(80, output_size=64, merge_method="sum", num_blocks=1)
    with pytest.raises(ValueError):
        espnet_b200.BranchformerEncoder(80, output_size=64, cgmlp_weight=[0.5, 0.5], num_blocks=3)
    with pytest.raises(AssertionError):
        espnet_b200.BranchformerEncoder(80, output_size=64, use_attn=False, use_cgmlp=False, num_blocks=1)


def test_registries():
    import espnet_b200
    from espnet_b200 import integration

    assert espnet_b200.encoder_choices["branchformer"] is espnet_b200.BranchformerEncoder
    assert integration.NAMES["encoder"]["b200_branchformer"] == "BranchformerEncoder"
    # the reference's defaults build (concat, 12 blocks); training-only options are accepted
    enc = espnet_b200.BranchformerEncoder(80, stochastic_depth_rate=0.1, attn_branch_drop_rate=[0.1] * 12, use_flash_attn=False, dropout_rate=0.3)
    assert enc.output_size() == 256 and len(enc.encoders) == 12 and enc.encoders[0].merge_proj.weight.shape == (256, 512)


def test_build_model_accepts_specaug_of_a_recipe_config(tmp_path):
    """A recipe-written config.yaml names SpecAug (training-only, no parameters): it builds, and specaug_conf is ignored."""
    import espnet_b200

    z, cfg, w = load_bf()
    y = refbuild_bf.model_yaml(cfg)
    y["specaug"] = "specaug"
    y["specaug_conf"] = dict(apply_time_warp=True, time_warp_window=5, apply_freq_mask=True, freq_mask_width_range=[0, 27],
                             num_freq_mask=2, apply_time_mask=True, time_mask_width_ratio_range=[0.0, 0.05], num_time_mask=10)
    path = tmp_path / "config.yaml"
    path.write_text(yaml.safe_dump(y))
    with open(path) as f:
        args = argparse.Namespace(**yaml.safe_load(f))
    model = espnet_b200.build_model(args)
    model.load_state_dict(w, strict=True)
    assert isinstance(model.encoder, espnet_b200.BranchformerEncoder)
    y["specaug"] = "other"
    with pytest.raises(NotImplementedError):
        espnet_b200.build_model(argparse.Namespace(**y))
