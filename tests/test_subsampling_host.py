"""The conv2d2 / conv2d6 / conv2d8 input layers on a CPU-only box: the oracle against the reference fixtures, strict loading of reference
state_dicts, the host logic of the shared subsampling (espnet_b200/layers.py) with the C-ABI entry points replaced by their torch restatements
(tests/emu_subsampling.py), check_short_utt's limits, and the encoders that keep refusing these input layers."""
import argparse

import numpy as np
import pytest
import torch

import emu_subsampling
from golden_util import load
from subsampling_fixture import PAIRS, build_encoder, feats, load_case, oracle_encode


@pytest.mark.parametrize("encoder,input_layer", PAIRS)
def test_oracle_vs_reference_fixture(encoder, input_layer):
    z, tag, cfg, w = load_case(encoder, input_layer)
    out, layers = oracle_encode(encoder, input_layer, cfg, w, feats(z, tag))
    assert out.shape[0] == int(z[f"{tag}olens"][0])
    for i in range(cfg["enc_layers"] + 1):
        np.testing.assert_allclose(layers[i].numpy(), z[f"{tag}layer{i}"], atol=1e-5, rtol=1e-5)
    np.testing.assert_allclose(out.numpy(), z[f"{tag}out"], atol=1e-5, rtol=1e-5)


@pytest.mark.parametrize("encoder,input_layer", PAIRS)
def test_reference_state_dict_loads_strictly(encoder, input_layer):
    z, tag, cfg, w = load_case(encoder, input_layer)
    enc = build_encoder(encoder, input_layer, cfg, w)   # load_state_dict(strict=True) of the reference's parameters and buffers
    assert {k: tuple(v.shape) for k, v in enc.state_dict().items()} == {k[len("encoder."):]: tuple(v.shape) for k, v in w.items()}


def test_recipe_config_model_loads_strictly(monkeypatch):
    """A whole model built from a config.yaml with a conv2d6 Conformer (the ReazonSpeech recipe's input layer) takes the reference
    Speech2Text's state_dict with strict=True."""
    import espnet_b200
    import refbuild_ebf
    import refbuild_subsampling
    from gpu_util import refbuild

    refbuild_subsampling.install(monkeypatch)
    z, cfg, _ = load("subsampling_s2t")
    weights = refbuild_ebf.fixture_weights(z)
    cfg["input_layer"] = str(z["input_layer"])
    model = espnet_b200.build_model(argparse.Namespace(**refbuild.model_yaml(cfg)))
    model.load_state_dict(weights, strict=True)
    assert model.encoder.input_layer == "conv2d6"


@pytest.mark.parametrize("encoder,input_layer", PAIRS)
def test_emulated_host_logic_vs_fixture(monkeypatch, encoder, input_layer):
    z, tag, cfg, w = load_case(encoder, input_layer)
    emu_subsampling.install(monkeypatch)
    enc = build_encoder(encoder, input_layer, cfg, w)
    enc.trace = []
    x = feats(z, tag)[None]
    out, olens, _ = enc(x, torch.tensor([x.shape[1]]))
    assert olens.tolist() == z[f"{tag}olens"].tolist()
    for i in range(cfg["enc_layers"] + 1):
        np.testing.assert_allclose(enc.trace[i][0].numpy(), z[f"{tag}layer{i}"], atol=5e-5, rtol=1e-5)
    np.testing.assert_allclose(out[0].numpy(), z[f"{tag}out"], atol=5e-5, rtol=1e-5)


@pytest.mark.parametrize("encoder,input_layer,lens", [("conformer", "conv2d6", [11, 40, 63, 58]), ("transformer", "conv2d8", [15, 71, 64, 33]),
                                                      ("e_branchformer", "conv2d2", [7, 30, 22]), ("conformer", "conv2d8", [16, 47, 23])])
def test_emulated_ragged_batch_equals_single_utterances(monkeypatch, encoder, input_layer, lens):
    """Every utterance of a ragged batch (one at the minimum length, the others with different residues modulo 6 and 8) gets what it gets
    alone; rows t >= olens[b] are padding."""
    from espnet_b200.layers import subsampled_len

    z, tag, cfg, w = load_case(encoder, input_layer)
    emu_subsampling.install(monkeypatch)
    enc = build_encoder(encoder, input_layer, cfg, w)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(len(lens), max(lens), 80, generator=g)
    out, olens, _ = enc(x, torch.tensor(lens))
    assert olens.tolist() == [subsampled_len(n, input_layer)[-1] for n in lens]
    for i, n in enumerate(lens):
        alone, ol, _ = enc(x[i:i + 1, :n], torch.tensor([n]))
        T = int(ol[0])
        assert T == int(olens[i]) and T >= 1
        np.testing.assert_allclose(out[i, :T].numpy(), alone[0].numpy(), atol=5e-5, rtol=1e-5)
        ref, _ = oracle_encode(encoder, input_layer, cfg, w, x[i, :n])
        np.testing.assert_allclose(out[i, :T].numpy(), ref.numpy(), atol=5e-5, rtol=1e-5)


@pytest.mark.parametrize("input_layer,n,limit", [("conv2d6", 10, 11), ("conv2d8", 14, 15), ("conv2d2", 6, 7)])
def test_too_short_utterance(monkeypatch, input_layer, n, limit):
    """check_short_utt (subsampling.py:31-48): the reference's message and limit, for the padded length and for one utterance of a batch."""
    from espnet_b200.errors import TooShortUttError
    from oracle.encoder import TooShortUttError as OracleTooShort
    from oracle.subsampling import conv2d_subsampling

    z, tag, cfg, w = load_case("conformer", input_layer)
    emu_subsampling.install(monkeypatch)
    enc = build_encoder("conformer", input_layer, cfg, w)
    msg = f"has {n} frames and is too short for subsampling (it needs more than {limit} frames), return empty results"
    with pytest.raises(TooShortUttError) as e:
        enc(torch.randn(1, n, 80), torch.tensor([n]))
    assert (e.value.actual_size, e.value.limit) == (n, limit) and str(e.value) == msg
    with pytest.raises(TooShortUttError) as e:
        enc(torch.randn(2, limit + 20, 80), torch.tensor([limit + 20, n]))
    assert (e.value.actual_size, e.value.limit) == (n, limit) and str(e.value).startswith(msg)
    with pytest.raises(OracleTooShort) as e:
        conv2d_subsampling(torch.randn(n, 80), w, input_layer)
    assert (e.value.actual_size, e.value.limit) == (n, limit) and str(e.value) == msg
    out, olens, _ = enc(torch.randn(1, limit, 80), torch.tensor([limit]))
    assert olens.tolist() == [1] and out.shape[1] == 1


def test_branchformer_and_streaming_refuse_new_input_layers():
    import espnet_b200

    for il in ("conv2d2", "conv2d6", "conv2d8"):
        with pytest.raises(NotImplementedError):
            espnet_b200.BranchformerEncoder(80, 64, input_layer=il)
        with pytest.raises(NotImplementedError):
            espnet_b200.ContextualBlockConformerEncoder(80, input_layer=il, macaron_style=True, use_cnn_module=True)


@pytest.mark.parametrize("cls", ["ConformerEncoder", "TransformerEncoder", "EBranchformerEncoder"])
def test_other_input_layers_still_refused(cls):
    import espnet_b200

    for il in ("conv2d1", "conv1d2", "linear", "embed"):
        with pytest.raises(NotImplementedError):
            getattr(espnet_b200, cls)(80, 64, input_layer=il)
