"""CPU: the RNN model family (VGGRNNEncoder / RNNEncoder / RNNDecoder) -- the float64 oracle against the reference fixtures
(tests/golden/rnn.npz), strict loading of reference state_dicts, the refused configurations, the registries, a model built from a
recipe-style config.yaml and checkpoint, and the C-ABI bindings of the new entry points."""
import os
import re

import numpy as np
import pytest
import torch

import rnn_fixture as fx
from oracle import rnn as orn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("espb_vgg_conv1_relu_f32", "espb_vgg_pool_f32", "espb_lstm_rec_step_f32", "espb_rnn_proj_post_f32", "espb_att_loc_step_f32",
               "espb_drop_cand_i32")


@pytest.mark.parametrize("case", fx.ENC_CASES)
def test_oracle_encoder_vs_reference_fixture(case):
    z = fx.load()
    cls, conf, w, feats = fx.enc_case(case)
    out, trace = orn.rnn_encoder(feats[0].double(), orn.to(w), conf, cls)
    np.testing.assert_allclose(out.numpy(), z[f"{case}:out"][0], atol=1e-4, rtol=0)
    names = (["vgg"] if cls == "vgg_rnn" else []) + [f"layer{i}" for i in range(len(trace) - (cls == "vgg_rnn"))]
    for nm, t in zip(names, trace):
        np.testing.assert_allclose(t.numpy(), z[f"{case}:{nm}"].reshape(t.shape), atol=1e-4, rtol=0, err_msg=nm)
    assert out.shape[0] == int(z[f"{case}:olens"][0])


@pytest.mark.parametrize("case", fx.ENC_CASES)
def test_encoder_state_dict_loads_strictly(case):
    enc, _ = fx.build_encoder(case)
    _, _, w, _ = fx.enc_case(case)
    assert sorted(enc.state_dict()) == sorted(w)


@pytest.mark.parametrize("model", ["base", "ctxres"])
def test_model_from_recipe_config_and_checkpoint(tmp_path, model):
    """ASRTask.build_model_from_file path: config.yaml (encoder: vgg_rnn, decoder: rnn) + checkpoint -> every reference key loads."""
    from espnet_b200.asr_inference import build_model_from_file

    cfg, ckpt = fx.write_model_files(tmp_path, model)
    m, args = build_model_from_file(cfg, ckpt, device="cpu")
    w = fx.model_weights(model)
    sd = m.state_dict()
    assert sorted(k for k in sd if not k.startswith("frontend.")) == sorted(k for k in w if not k.startswith("frontend."))
    for k, v in w.items():
        if k in sd:
            assert torch.equal(sd[k], v), k
    assert type(m.encoder).__name__ == "VGGRNNEncoder" and type(m.decoder).__name__ == "RNNDecoder"
    assert m.decoder.context_residual == (model == "ctxres")


def test_registries():
    import espnet_b200
    from espnet_b200 import integration

    assert espnet_b200.encoder_choices["vgg_rnn"] is espnet_b200.VGGRNNEncoder
    assert espnet_b200.encoder_choices["rnn"] is espnet_b200.RNNEncoder
    assert espnet_b200.decoder_choices["rnn"] is espnet_b200.RNNDecoder
    assert integration.NAMES["encoder"]["b200_vgg_rnn"] == "VGGRNNEncoder"
    assert integration.NAMES["encoder"]["b200_rnn"] == "RNNEncoder"
    assert integration.NAMES["decoder"]["b200_rnn"] == "RNNDecoder"


def test_refused_configurations():
    import espnet_b200

    for cls in (espnet_b200.VGGRNNEncoder, espnet_b200.RNNEncoder):
        with pytest.raises(NotImplementedError):
            cls(80, rnn_type="gru")
        with pytest.raises(ValueError):
            cls(80, rnn_type="rnn_tanh")
    with pytest.raises(NotImplementedError):
        espnet_b200.VGGRNNEncoder(80, in_channel=3)
    dec = dict(vocab_size=10, encoder_output_size=8, hidden_size=8, att_conf=dict(adim=8, aconv_chans=2, aconv_filts=3))
    espnet_b200.RNNDecoder(**dec)
    bad = [dict(rnn_type="gru"), dict(replace_sos=True), dict(num_encs=2), dict(sampling_probability=0.1),
           dict(att_conf=dict(atype="dot")), dict(att_conf=dict(atype="location2d")), dict(att_conf=dict(han_mode=True)),
           dict(att_conf=dict(han_dim=16)), dict(att_conf=dict(num_att=2))]
    for kw in bad:
        with pytest.raises(NotImplementedError):
            espnet_b200.RNNDecoder(**dict(dec, **kw))
    with pytest.raises(ValueError):
        espnet_b200.RNNDecoder(**dict(dec, rnn_type="rnn"))
    with pytest.raises(TypeError):
        espnet_b200.RNNDecoder(**dict(dec, att_conf=dict(no_such_option=1)))


def test_decoder_parameter_names_match_reference():
    """The reference RNNDecoder's state_dict names (embed, decoder.{k}.*, output, att_list.0.*) as the fixture records them."""
    import espnet_b200

    cfg = fx.model_config("ctxres")
    dec = espnet_b200.RNNDecoder(vocab_size=len(cfg["token_list"]), encoder_output_size=cfg["encoder_conf"]["output_size"], **cfg["decoder_conf"])
    w = {k[len("decoder."):]: v for k, v in fx.model_weights("ctxres").items() if k.startswith("decoder.")}
    dec.load_state_dict(w, strict=True)


def test_oracle_decoder_step_properties():
    """The oracle decoder step: log-probabilities normalise, attention weights are a distribution, the first step uses uniform weights."""
    cfg = fx.model_config("base")
    w = orn.to({k[len("decoder."):]: v for k, v in fx.model_weights("base").items() if k.startswith("decoder.")})
    d = orn.OracleRNNDecoder(w, cfg["decoder_conf"]["num_layers"])
    enc = torch.randn(7, cfg["encoder_conf"]["output_size"], dtype=torch.float64)
    logp, st = d.score(len(cfg["token_list"]) - 1, None, enc)
    assert abs(float(logp.exp().sum()) - 1) < 1e-12 and abs(float(st[2].sum()) - 1) < 1e-12
    logp2, st2 = d.score(3, st, enc)
    assert abs(float(logp2.exp().sum()) - 1) < 1e-12 and not torch.equal(st2[2], st[2])


def test_new_entry_points_are_declared_and_bound():
    from espnet_b200 import lib

    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "espnet_b200.h")).read(), flags=re.S)
    for sym in NEW_SYMBOLS:
        assert sym in lib._SIGS and re.search(r"\bint\s+" + sym + r"\s*\(", src), sym
    assert len(lib._SIGS["espb_drop_cand_i32"]) == 5 and len(lib._SIGS["espb_att_loc_step_f32"]) == 28 and len(lib._SIGS["espb_lstm_rec_step_f32"]) == 16


# ------------------------------------------------------------------------------------------------ host logic through the kernel emulation
@pytest.mark.parametrize("case", fx.ENC_CASES)
def test_encoder_host_logic_vs_reference_fixture(case, monkeypatch):
    """VGGRNNEncoder / RNNEncoder.forward with the C-ABI entry points emulated (tests/emu_rnn.py): GEMM descriptors of the implicit-GEMM
    convs, the per-step recurrence GEMMs and the strided projection GEMMs, buffer pitches and layouts, against the reference fixture."""
    import emu_rnn

    emu_rnn.install(monkeypatch)
    z = fx.load()
    enc, feats = fx.build_encoder(case)
    enc.trace = []
    out, olens, _ = enc(feats, torch.tensor([feats.shape[1]]))
    np.testing.assert_allclose(out[0].numpy(), z[f"{case}:out"][0], atol=1e-4, rtol=0)
    assert int(olens[0]) == int(z[f"{case}:olens"][0])
    names = (["vgg"] if case.startswith("vgg") else []) + [k.split(":")[1] for k in sorted(z.files) if k.startswith(f"{case}:layer")]
    assert len(enc.trace) == len(names)
    for nm, t in zip(names, enc.trace):
        np.testing.assert_allclose(t[0].numpy(), z[f"{case}:{nm}"].reshape(t[0].shape), atol=1e-4, rtol=0, err_msg=nm)


@pytest.mark.parametrize("case", ["vgg_blstmp", "rnn_sub"])
def test_encoder_host_logic_ragged_batch_equals_single(case, monkeypatch):
    import emu_rnn

    emu_rnn.install(monkeypatch)
    enc, feats = fx.build_encoder(case)
    g = torch.Generator().manual_seed(9)
    T = feats.shape[1]
    lens = [T, T - 6, 3]
    xs = torch.randn(len(lens), T, 80, generator=g)
    out, olens, _ = enc(xs, torch.tensor(lens))
    out = out.clone()
    for i, L in enumerate(lens):
        o1, ol1, _ = enc(xs[i:i + 1, :L], torch.tensor([L]))
        assert int(olens[i]) == int(ol1[0])
        torch.testing.assert_close(out[i, :int(ol1[0])], o1[0], atol=1e-5, rtol=0)
        assert torch.all(out[i, int(ol1[0]):] == 0)


@pytest.mark.parametrize("context_residual", [False, True])
def test_decoder_host_logic_vs_oracle(context_residual, monkeypatch):
    """RNNDecoder.init_memory / step with the entry points emulated: 2 utterances (lengths 7, 3) x 2 slots over 4 positions with reordered
    ancestors, log-probabilities, h / c rings and attention weights against OracleRNNDecoder (float64); widths 10 / 14 exercise the padded
    operand columns."""
    import emu_rnn

    from espnet_b200 import RNNDecoder, ops

    emu_rnn.install(monkeypatch)
    torch.manual_seed(5)
    U, W, Tm, E, H, V, L, P = 2, 2, 7, 14, 10, 23, 2, 4
    n = U * W
    dec = RNNDecoder(V, E, num_layers=L, hidden_size=H, context_residual=context_residual,
                     att_conf=dict(adim=16, aconv_chans=3, aconv_filts=4)).eval()
    o = orn.OracleRNNDecoder(orn.to(dec.state_dict()), L, context_residual)
    lens = torch.tensor([7, 3])
    g = torch.Generator().manual_seed(6)
    enc = torch.randn(U, Tm, E, generator=g)
    st = dec.init_memory(ops.split_from(enc.view(U * Tm, E)), U, Tm, lens.to(torch.int32), n, P)
    anc = torch.zeros(n, P, dtype=torch.int32)
    prev = [None] * n
    for pos in range(P):
        tok = torch.randint(0, V, (n,), generator=g)
        if pos:
            anc[:, pos - 1] = torch.tensor([(s // W) * W + (s + pos) % W for s in range(n)], dtype=torch.int32)
        logp = dec.step(st, pos, tok.to(torch.int32), anc).double()
        cur = []
        for s in range(n):
            u, Lu = s // W, int(lens[s // W])
            lp, ns = o.score(int(tok[s]), prev[int(anc[s, pos - 1])] if pos else None, enc[u, :Lu].double())
            cur.append(ns)
            torch.testing.assert_close(logp[s], lp, atol=5e-5, rtol=0)
            for k in range(L):
                torch.testing.assert_close(st["h"][pos & 1, k, s, :H].double(), ns[0][k], atol=2e-5, rtol=0)
                torch.testing.assert_close(st["c"][pos & 1, k, s, :H].double(), ns[1][k], atol=2e-5, rtol=0)
            torch.testing.assert_close(st["a"][pos & 1, s, :Lu].double(), ns[2], atol=2e-5, rtol=0)
        prev = cur
