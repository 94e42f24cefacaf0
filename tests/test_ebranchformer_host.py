"""E-Branchformer encoder on a CPU-only box: the oracle against the reference fixtures, and the host logic of
espnet_b200.EBranchformerEncoder (weight packing, the [M, 2D] concatenation buffer, GEMM descriptors, kernel order) with the C-ABI entry
points replaced by their torch restatements (tests/emu_ebf.py)."""
import argparse
import os
import sys

import numpy as np
import pytest
import torch

import emu_backend
import emu_ebf
from golden_util import DEC_NAMES, GOLDEN_DIR, decode_params, decode_results, load

sys.path.insert(0, GOLDEN_DIR)
import refbuild_ebf  # noqa: E402


def load_enc(tag):
    z = np.load(os.path.join(GOLDEN_DIR, "ebranchformer_enc.npz"))
    cfg = dict(zip(z[f"{tag}:cfg_keys"].tolist(), (int(v) for v in z[f"{tag}:cfg_vals"])))
    return z, cfg, refbuild_ebf.fixture_weights(z, prefix=f"{tag}:")


def load_ebf():
    z, cfg, _ = load("ebf")
    return z, cfg, refbuild_ebf.fixture_weights(z)


def build_encoder(cfg, w=None):
    import espnet_b200

    enc = espnet_b200.EBranchformerEncoder(80, **refbuild_ebf.encoder_conf(cfg))
    if w is not None:
        enc.load_state_dict({k[len("encoder."):]: v for k, v in w.items() if k.startswith("encoder.")}, strict=True)
    return enc.eval()


def _random_norms(enc, seed):
    """LayerNorm affines away from 1 / 0 (a normalised padded row is then beta, not 0) and every bias non-zero."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in enc.named_parameters():
            if "norm" in n or n.endswith("bias"):
                p.add_(0.2 * torch.randn(p.shape, generator=g))
    return {"encoder." + k: v.detach().clone() for k, v in enc.state_dict().items()}


@pytest.mark.parametrize("tag", ["A", "B"])
def test_oracle_vs_reference_encoder_fixture(tag):
    from oracle.e_branchformer import ebranchformer_encode

    z, cfg, w = load_enc(tag)
    out, layers = ebranchformer_encode(torch.from_numpy(z[f"{tag}:feats"]), w, cfg["heads"], cfg["enc_layers"], return_layers=True)
    assert out.shape[0] == int(z[f"{tag}:olens"][0])
    for i in range(1, cfg["enc_layers"] + 1):
        np.testing.assert_allclose(layers[i].numpy(), z[f"{tag}:layer{i}"], atol=1e-5, rtol=1e-5)
    np.testing.assert_allclose(out.numpy(), z[f"{tag}:out"], atol=1e-5, rtol=1e-5)


def test_oracle_vs_reference_speech2text_fixture():
    from oracle import ctc_logits
    from oracle.e_branchformer import EBranchformerSpeech2Text

    z, cfg, w = load_ebf()
    assert cfg["encoder"] == "e_branchformer"
    o = EBranchformerSpeech2Text(cfg, w)
    enc = o.encode(torch.from_numpy(z["wave"]))
    np.testing.assert_allclose(enc.numpy(), z["enc"], atol=1e-5, rtol=1e-5)
    np.testing.assert_allclose(ctc_logits(enc, o.w).numpy(), z["ctc_logits"], atol=1e-4, rtol=1e-5)
    for dn in DEC_NAMES:
        res = EBranchformerSpeech2Text(cfg, w, nbest=10, **decode_params(z, dn))(z["wave"])
        gold = decode_results(z, dn)
        assert len(res) == len(gold), dn
        for (_, _, _, h), (yseq, score, _) in zip(res, gold):
            assert h.yseq.tolist() == yseq, dn
            assert abs(float(h.score) - score) <= 1e-4 * max(1.0, abs(score)), dn


@pytest.mark.parametrize("tag", ["A", "B"])
def test_encoder_host_logic_vs_reference_fixture(tag, monkeypatch):
    emu_ebf.install(monkeypatch)
    z, cfg, w = load_enc(tag)
    enc = build_encoder(cfg, w)
    enc.trace = []
    feats = torch.from_numpy(z[f"{tag}:feats"])[None]
    out, olens, _ = enc(feats, torch.tensor([feats.shape[1]]))
    assert int(olens[0]) == int(z[f"{tag}:olens"][0])
    for i in range(1, cfg["enc_layers"] + 1):
        np.testing.assert_allclose(enc.trace[i][0].numpy(), z[f"{tag}:layer{i}"], atol=5e-5, rtol=1e-5)
    np.testing.assert_allclose(out[0].numpy(), z[f"{tag}:out"], atol=5e-5, rtol=1e-5)
    L = cfg["enc_layers"]
    assert emu_backend.calls.count("espb_csgu_f32") == L and emu_backend.calls.count("espb_merge_dwconv_f32") == L


@pytest.mark.parametrize("tag,lens", [("A", [150, 47, 103]), ("B", [31, 150, 19])])
def test_encoder_ragged_batch_host_logic(tag, lens, monkeypatch):
    """Per-utterance semantics: the conv halos of both depthwise convs reach past the end of the shorter utterances (T = 36, 11, 25 with
    kernels 31; T = 7, 36, 4 with kernels 15 / 3), which must see zeros there -- not the LayerNorm of a padded row.  Padded output rows
    are 0."""
    from oracle.e_branchformer import ebranchformer_encode

    emu_ebf.install(monkeypatch)
    _, cfg, _ = load_enc(tag)
    torch.manual_seed(11)
    enc = build_encoder(cfg)
    w = _random_norms(enc, 12)
    g = torch.Generator().manual_seed(13)
    feats = torch.randn(len(lens), max(lens), 80, generator=g)     # padded frames are garbage, not zeros
    out, olens, _ = enc(feats, torch.tensor(lens))
    for i, n in enumerate(lens):
        ref = ebranchformer_encode(feats[i, :n], w, cfg["heads"], cfg["enc_layers"])
        T = ref.shape[0]
        assert int(olens[i]) == T
        np.testing.assert_allclose(out[i, :T].numpy(), ref.numpy(), atol=5e-5, rtol=1e-5)
        assert not out[i, T:].any()


def test_speech2text_host_logic_vs_reference_fixture(monkeypatch):
    """Waveform -> E-Branchformer encoder -> CTC head + decoder -> beam search, every kernel emulated, against the reference Speech2Text."""
    import espnet_b200
    from espnet_b200.search import BatchBeamSearch

    emu_backend.install_search(monkeypatch)
    emu_backend.install_frontend(monkeypatch)
    emu_ebf.install(monkeypatch)
    z, cfg, w = load_ebf()
    model = espnet_b200.build_model(argparse.Namespace(**refbuild_ebf.model_yaml(cfg)))
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
    for tag in ("A", "B"):
        _, cfg, w = load_enc(tag)
        build_encoder(cfg, w)
    import espnet_b200

    z, cfg, w = load_ebf()
    espnet_b200.build_model(argparse.Namespace(**refbuild_ebf.model_yaml(cfg))).load_state_dict(w, strict=True)


@pytest.mark.parametrize("kw", [dict(input_layer="linear"), dict(rel_pos_type="legacy"), dict(pos_enc_layer_type="abs_pos"),
                                dict(attention_layer_type="selfattn"), dict(attention_layer_type="fast_selfattn"),
                                dict(use_linear_after_conv=True), dict(gate_activation="tanh"), dict(use_ffn=True, ffn_activation_type="tanh"),
                                dict(use_ffn=True, positionwise_layer_type="conv1d"), dict(cgmlp_conv_kernel=30), dict(merge_conv_kernel=129),
                                dict(zero_triu=True), dict(qk_norm=True), dict(interctc_layer_idx=[1]), dict(output_size=80, attention_heads=4)])
def test_unsupported_options_are_refused(kw):
    import espnet_b200

    with pytest.raises(NotImplementedError):
        espnet_b200.EBranchformerEncoder(80, **kw)


def test_registries():
    import espnet_b200
    from espnet_b200 import integration

    assert espnet_b200.encoder_choices["e_branchformer"] is espnet_b200.EBranchformerEncoder
    assert integration.NAMES["encoder"]["b200_e_branchformer"] == "EBranchformerEncoder"
    # the reference's own defaults build (no FFN, merge kernel 3); dropout / layer drop / flash / checkpointing options are accepted
    enc = espnet_b200.EBranchformerEncoder(80, layer_drop_rate=0.1, use_flash_attn=False, gradient_checkpoint_layers=[1], dropout_rate=0.3)
    assert enc.output_size() == 256 and enc.encoders[0].feed_forward is None and enc.merge_kernel == 3
