"""Intermediate and self-conditioned CTC (interctc_layer_idx / interctc_use_conditioning) on a CPU-only box: the float64 oracle against the
reference fixtures, the host logic of EncoderBase._interctc with the C-ABI entry points replaced by their torch restatements
(tests/emu_interctc.py), strict loading of recipe-shaped models, and the refusals."""
import argparse

import numpy as np
import pytest
import torch

import emu_backend
import emu_interctc
from espnet_b200.layers import _pitch
from gpu_util import refbuild
from interctc_fixture import CASES, build, feats, load_case, load_model_fixture, oracle
import refbuild_interctc  # noqa: E402  (tests/golden is on sys.path after interctc_fixture)

TOL = 2e-5   # float32 reference vs float64 oracle / emulation (the other fixtures' 1e-5 plus headroom for the softmax feedback)


@pytest.mark.parametrize("case", CASES)
def test_oracle_vs_reference_fixture(case):
    z, tag, cfg, idx, w = load_case(case)
    out, inter, blocks = oracle(cfg, w, idx, feats(z, tag))
    assert out.shape[0] == int(z[f"{tag}olens"][0])
    assert [li for li, _ in inter] == idx
    for i, x in enumerate(blocks):
        np.testing.assert_allclose(x.numpy(), z[f"{tag}layer{i + 1}"], atol=TOL, rtol=1e-5)
    for li, h in inter:
        np.testing.assert_allclose(h.numpy(), z[f"{tag}inter{li}"], atol=TOL, rtol=1e-5)
    np.testing.assert_allclose(out.numpy(), z[f"{tag}out"], atol=TOL, rtol=1e-5)


@pytest.mark.parametrize("case", ["conf64", "tfm64"])
def test_conditioning_moves_the_output(case):
    """The fixtures can tell a dropped conditioning GEMM apart: without it the output moves by far more than the tolerance."""
    z, tag, cfg, idx, w = load_case(case)
    out, _, _ = oracle(dict(cfg, ic_cond=0), w, idx, feats(z, tag))
    assert float((out - torch.from_numpy(z[f"{tag}out"]).double()).abs().max()) > 100 * TOL


@pytest.mark.parametrize("case", CASES)
def test_emulated_host_logic_vs_fixture(monkeypatch, case):
    z, tag, cfg, idx, w = load_case(case)
    emu_interctc.install(monkeypatch)
    enc, ctc = build(cfg, w)
    x = feats(z, tag)[None]
    (out, inter), olens, _ = enc(x, torch.tensor([x.shape[1]]), ctc=ctc)
    assert olens.tolist() == z[f"{tag}olens"].tolist()
    assert [li for li, _ in inter] == idx
    for li, h in inter:
        np.testing.assert_allclose(h[0].numpy(), z[f"{tag}inter{li}"], atol=TOL, rtol=1e-5)
    np.testing.assert_allclose(out[0].numpy(), z[f"{tag}out"], atol=TOL, rtol=1e-5)
    # one softmax per conditioned layer, between the CTC logits GEMM and the conditioning GEMM, into a K padded to a multiple of 32
    n_soft = emu_backend.calls.count("espb_softmax_rows_split_f32")
    assert n_soft == (len(idx) if cfg["ic_cond"] else 0)
    M = olens.item()
    probs = [t for (name, shape, _), t in enc._ws.items() if name[1] == "ic_probs"]
    if cfg["ic_cond"]:
        assert [tuple(p.shape) for p in probs] == [(2, M, _pitch(cfg["vocab"]))]
        assert bool((probs[0][:, :, cfg["vocab"]:] == 0).all())
        assert enc._packed["cond_w"].shape == (2, cfg["d_model"], _pitch(cfg["vocab"]))
    else:
        assert not probs


@pytest.mark.parametrize("case,lens", [("conf16", [161, 40, 97]), ("tfm64", [150, 63, 9])])
def test_emulated_ragged_batch_equals_single_utterances(monkeypatch, case, lens):
    """Every utterance of a ragged batch gets its per-utterance intermediate outputs and output; padding rows do not reach valid rows."""
    z, tag, cfg, idx, w = load_case(case)
    emu_interctc.install(monkeypatch)
    enc, ctc = build(cfg, w)
    g = torch.Generator().manual_seed(9)
    x = torch.randn(len(lens), max(lens), 80, generator=g)
    (out, inter), olens, _ = enc(x, torch.tensor(lens), ctc=ctc)
    for i, n in enumerate(lens):
        T = int(olens[i])
        ref, ref_inter, _ = oracle(cfg, w, idx, x[i, :n])
        assert ref.shape[0] == T
        assert torch.isfinite(out[i]).all()
        np.testing.assert_allclose(out[i, :T].numpy(), ref.numpy(), atol=5e-5, rtol=1e-5)
        for (li, h), (lr, hr) in zip(inter, ref_inter):
            assert li == lr
            np.testing.assert_allclose(h[i, :T].numpy(), hr.numpy(), atol=5e-5, rtol=1e-5)


def test_no_interctc_adds_no_launch_and_no_buffer(monkeypatch):
    z, tag, cfg, idx, w = load_case("noc")
    emu_interctc.install(monkeypatch)
    enc, ctc = build(dict(cfg, ic_a=0, ic_b=0), w)
    out, _, _ = enc(feats(z, tag)[None], torch.tensor([cfg["nframes"]]))
    assert isinstance(out, torch.Tensor)
    assert "espb_softmax_rows_split_f32" not in emu_backend.calls
    assert not [k for k in enc._ws if k[0][1].startswith("ic_")]
    assert "cond_w" not in enc._packed


def _model(name, monkeypatch):
    refbuild_interctc.install(monkeypatch)
    z, cfg, w = load_model_fixture(name)
    import espnet_b200

    model = espnet_b200.build_model(argparse.Namespace(**refbuild.model_yaml(cfg)))
    model.load_state_dict(w, strict=True)
    return z, cfg, model.eval()


@pytest.mark.parametrize("name", ["interctc_s2t", "interctc_ctconly"])
def test_model_fixture_loads_strictly_and_encodes(monkeypatch, name):
    """The reference Speech2Text's state_dict (encoder.conditioning_layer after after_norm) loads with strict=True; encode() passes the CTC
    head, drops the intermediate outputs, and its split copy is the one of the final LayerNorm (emulated kernels)."""
    z, cfg, model = _model(name, monkeypatch)
    keys = list(model.encoder.state_dict())
    assert keys[-4:] == ["after_norm.weight", "after_norm.bias", "conditioning_layer.weight", "conditioning_layer.bias"]
    assert (model.decoder is None) == bool(cfg.get("no_decoder", 0))
    emu_interctc.install(monkeypatch)
    emu_backend.install_frontend(monkeypatch)
    wave = torch.from_numpy(z["wave"])
    enc, lens = model.encode(wave[None], torch.tensor([wave.numel()]))
    assert isinstance(enc, torch.Tensor) and lens.tolist() == [z["enc"].shape[0]]
    np.testing.assert_allclose(enc[0].numpy(), z["enc"], atol=1e-4, rtol=1e-4)
    split = model.enc_split(enc)
    assert split is not None and split is model.encoder._ws[((0, "enc_split"), tuple(split.shape), torch.float32)]
    np.testing.assert_allclose((split[0] + split[1]).view_as(enc).numpy(), enc.numpy(), atol=1e-6)


def test_librispeech100_scctc_config_loads_strictly(tmp_path):
    """egs2/librispeech_100/asr1/conf/tuning/train_conformer_scctc.yaml (18 blocks, d 256, [6, 12], conditioning, no decoder, ctc_weight 1.0)
    with a 5000-token list: build_model_from_file loads a checkpoint of its own state_dict strictly."""
    import yaml

    import espnet_b200

    enc_conf = dict(output_size=256, attention_heads=4, linear_units=1024, num_blocks=18, dropout_rate=0.1, positional_dropout_rate=0.1,
                    attention_dropout_rate=0.1, input_layer="conv2d", normalize_before=True, macaron_style=True, rel_pos_type="latest",
                    pos_enc_layer_type="rel_pos", selfattention_layer_type="rel_selfattn", activation_type="swish", use_cnn_module=True,
                    cnn_module_kernel=31, interctc_layer_idx=[6, 12], interctc_use_conditioning=True)
    y = dict(token_list=refbuild.token_list(5000), frontend="default", frontend_conf=dict(n_fft=512, hop_length=160), specaug="specaug",
             specaug_conf=dict(apply_time_warp=True), encoder="conformer",
             encoder_conf=enc_conf, model_conf=dict(ctc_weight=1.0, interctc_weight=0.66, lsm_weight=0.1, length_normalized_loss=False))
    y["normalize"], y["normalize_conf"] = None, None   # the recipe's global_mvn needs its stats file
    args = argparse.Namespace(**y)
    model = espnet_b200.build_model(args)
    sd = model.state_dict()
    assert tuple(sd["encoder.conditioning_layer.weight"].shape) == (256, 5000) and model.decoder is None
    cfg, ckpt = tmp_path / "config.yaml", tmp_path / "model.pth"
    cfg.write_text(yaml.safe_dump(y))
    torch.save(sd, str(ckpt))
    loaded, _ = espnet_b200.asr_inference.build_model_from_file(str(cfg), None, device="cpu")
    loaded.load_state_dict(torch.load(str(ckpt)), strict=True)
    assert loaded.encoder.interctc_layer_idx == [6, 12] and loaded.encoder.interctc_use_conditioning


@pytest.mark.parametrize("cls", ["ConformerEncoder", "TransformerEncoder"])
def test_refusals(cls):
    import espnet_b200

    C = getattr(espnet_b200, cls)
    kw = dict(rel_pos_type="latest", macaron_style=True) if cls == "ConformerEncoder" else {}
    for bad in ([0, 2], [1, 3], [3]):   # 0 < min(idx) and max(idx) < num_blocks (conformer_encoder.py:318-319)
        with pytest.raises(AssertionError):
            C(80, 64, num_blocks=3, interctc_layer_idx=bad, **kw)
    enc = C(80, 64, num_blocks=3, interctc_layer_idx=[1], interctc_use_conditioning=True, **kw)
    with pytest.raises(ValueError, match="CTC head"):
        enc(torch.zeros(1, 30, 80), torch.tensor([30]))
    with pytest.raises(ValueError, match="conditioning_layer"):
        enc(torch.zeros(1, 30, 80), torch.tensor([30]), ctc=espnet_b200.CTC(10, 64))
    enc.conditioning_layer = torch.nn.Linear(11, 64)
    with pytest.raises(ValueError, match="posteriors"):
        enc(torch.zeros(1, 30, 80), torch.tensor([30]), ctc=espnet_b200.CTC(10, 64))
    if cls == "ConformerEncoder":
        with pytest.raises(NotImplementedError, match="ctc_trim"):
            C(80, 64, num_blocks=3, interctc_layer_idx=[1], ctc_trim=True, **kw)


def test_ebranchformer_still_refuses_interctc():
    import espnet_b200

    with pytest.raises(NotImplementedError):
        espnet_b200.EBranchformerEncoder(80, interctc_layer_idx=[1])
