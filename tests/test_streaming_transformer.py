"""espnet_b200.ContextualBlockTransformerEncoder (encoder: contextual_block_transformer) against outputs of the UNMODIFIED reference
(tests/golden/streaming_tfm_enc.npz and streaming_tfm_search.npz, made by tests/golden/make_golden_streaming_transformer.py).

- encoder: ``forward_infer`` for the conv2d / conv2d6 / conv2d8 input layers, every push of uneven chunks, one whole-utterance call and a
  segment shorter than a block (atol 1e-4 on O(1) encoder outputs); N streams in lock step == one stream;
- Speech2TextStreaming with it: the n-best of every push for joint decoding and for the AISHELL streaming decode settings with an LSTM LM
  (identical token ids, total and per-scorer scores rtol 2e-4 + atol 2e-3, as test_streaming_search.py), ``greedy=True``, and the
  command-line tool.

CPU: the host logic with the kernels emulated (tests/emu_*.py); -m gpu: the CUDA kernels."""
import argparse
import json
import os
import sys

import numpy as np
import pytest
import torch
import yaml

from golden_util import GOLDEN_DIR

sys.path.insert(0, GOLDEN_DIR)
import refbuild  # noqa: E402
import refbuild_ebf  # noqa: E402

LAYERS = ["conv2d", "conv2d6", "conv2d8"]
ENC = os.path.join(GOLDEN_DIR, "streaming_tfm_enc.npz")
SEARCH = os.path.join(GOLDEN_DIR, "streaming_tfm_search.npz")


# ---------------------------------------------------------------- encoder
def _encoder(il, device):
    import espnet_b200

    z = np.load(ENC)
    cfg = {k: int(v) for k, v in zip(z["cfg_keys"].tolist(), z["cfg_vals"].tolist())}
    enc = espnet_b200.ContextualBlockTransformerEncoder(80, input_layer=il, **cfg)
    enc.load_state_dict(refbuild_ebf.fixture_weights(z, prefix=f"{il}:"), strict=True)
    return z, enc.to(device).eval()


def _close(y, ref, what):
    assert tuple(y.shape) == ref.shape, (what, tuple(y.shape), ref.shape)
    if ref.size:
        e = float((y.cpu() - torch.from_numpy(ref)).abs().max())
        assert e < 1e-4, (what, e)


def _run_encoder(il, device, n_streams=1):
    """Returns the outputs of every push (stream 0) after checking every stream against the fixture."""
    z, enc = _encoder(il, device)
    feats = torch.from_numpy(z["feats"]).float().to(device)[None].repeat(n_streams, 1, 1)
    pushes = z["pushes"].tolist()
    states, pos, outs = None, 0, []
    for i, n in enumerate(pushes):
        y, ylen, states = enc(feats[:, pos:pos + n], torch.full((n_streams,), n), states, is_final=(i == len(pushes) - 1), infer_mode=True)
        assert (ylen is None) == bool(z[f"{il}:stream:{i}:olens_none"]), (il, i)
        for s in range(n_streams):
            _close(y[s], z[f"{il}:stream:{i}:y"], (il, i, s))
        outs.append(y[0].cpu())
        pos += n
    assert states is None
    for name, n in (("whole", 700), ("short", 131)):
        y, ylen, st = enc(feats[:1, :n], torch.tensor([n]), None, is_final=True, infer_mode=True)
        assert st is None and (ylen is None) == bool(z[f"{il}:{name}:olens_none"])
        _close(y[0], z[f"{il}:{name}:y"], (il, name))
    return outs


@pytest.mark.parametrize("il", LAYERS)
def test_encoder_host_logic_vs_reference_fixture(monkeypatch, il):
    import emu_backend
    import emu_subsampling

    emu_subsampling.install(monkeypatch)
    _run_encoder(il, "cpu")
    for name in ("espb_cbe_build_chunks_f32", "espb_cbe_ctx_propagate_f32", "espb_zero_rows_f32", "espb_gather_rows_f32"):
        assert name in emu_backend.calls
    assert "espb_glu_dwconv_bn_swish_f32" not in emu_backend.calls


@pytest.mark.parametrize("il", LAYERS)
def test_reference_state_dict_loads_strictly(il):
    z, enc = _encoder(il, "cpu")
    assert {k: tuple(v.shape) for k, v in enc.state_dict().items()} == \
        {k[len(il) + 8:]: tuple(z[k].tolist()) for k in z.files if k.startswith(f"{il}:pshape:")}
    assert enc.subsample == {"conv2d": 4, "conv2d6": 6, "conv2d8": 8}[il]
    names = set(enc.state_dict())
    assert {"embed.out.weight", "after_norm.weight", "encoders.1.self_attn.linear_q.weight", "encoders.1.feed_forward.w_2.bias",
            "encoders.0.norm1.weight", "encoders.0.norm2.bias"} <= names
    assert ("embed.conv.4.weight" in names) == (il == "conv2d8")


@pytest.mark.parametrize("kw", [dict(input_layer="linear"), dict(input_layer="embed"), dict(input_layer=None), dict(concat_after=True),
                                dict(normalize_before=False), dict(positionwise_layer_type="conv1d"), dict(init_average=False),
                                dict(ctx_pos_enc=False), dict(output_size=80, attention_heads=4), dict(block_size=20, hop_size=16, look_ahead=16)])
def test_refused_configurations(kw):
    import espnet_b200

    with pytest.raises(NotImplementedError):
        espnet_b200.ContextualBlockTransformerEncoder(80, **kw)


def test_accepted_keywords_and_unknown_input_layer():
    import espnet_b200

    enc = espnet_b200.ContextualBlockTransformerEncoder(80, output_size=64, attention_heads=4, linear_units=96, num_blocks=1,
                                                        positionwise_conv_kernel_size=1, padding_idx=-1, pos_enc_class=None, dropout_rate=0.1)
    assert enc.output_size() == 64 and (enc.block_size, enc.hop_size, enc.look_ahead) == (40, 16, 16)
    with pytest.raises(ValueError):
        espnet_b200.ContextualBlockTransformerEncoder(80, input_layer="conv2d2")
    with pytest.raises(NotImplementedError):
        enc(torch.zeros(1, 64, 80), torch.tensor([64]), infer_mode=False)


def test_registries():
    import espnet_b200
    from espnet_b200 import integration

    assert espnet_b200.encoder_choices["contextual_block_transformer"] is espnet_b200.ContextualBlockTransformerEncoder
    assert espnet_b200.encoder_choices["contextual_block_conformer"] is espnet_b200.ContextualBlockConformerEncoder
    assert integration.NAMES["encoder"]["b200_contextual_block_transformer"] == "ContextualBlockTransformerEncoder"


# ---------------------------------------------------------------- Speech2TextStreaming
def _files(tmp_path):
    """The fixture's model and LM as a recipe's config.yaml / checkpoint pairs (seeded weights, nothing downloaded)."""
    z = np.load(SEARCH)
    y = json.loads(str(z["yaml"]))
    paths = {k: str(tmp_path / k) for k in ("config.yaml", "model.pth", "lm.yaml", "lm.pth")}
    with open(paths["config.yaml"], "w") as f:
        yaml.safe_dump(y, f)
    torch.save(refbuild_ebf.fixture_weights(z), paths["model.pth"])
    with open(paths["lm.yaml"], "w") as f:
        yaml.safe_dump(dict(token_list=y["token_list"], lm="seq_rnn", lm_conf=json.loads(str(z["lm_conf"])), model_conf={}, init=None,
                            use_preprocessor=False), f)
    torch.save({"lm." + k: v for k, v in refbuild_ebf.fixture_weights(z, prefix="lm:").items()}, paths["lm.pth"])   # LanguageModel keys
    return z, paths


def _s2t(z, paths, name, device, n_streams=1):
    import espnet_b200

    kw = json.loads(str(z["settings"]))[name]
    extra = dict(lm_train_config=paths["lm.yaml"], lm_file=paths["lm.pth"]) if "lm_weight" in kw else {}
    return espnet_b200.Speech2TextStreaming(asr_train_config=paths["config.yaml"], asr_model_file=paths["model.pth"], n_streams=n_streams,
                                            device=device, **kw, **extra)


def _check_nbest(z, key, per_stream):
    assert len(per_stream) == int(z[f"{key}:n"]), (key, len(per_stream))
    token_list = json.loads(str(z["yaml"]))["token_list"]
    for j, (_, token, token_int, hyp) in enumerate(per_stream):
        k = f"{key}:{j}"
        assert hyp.yseq.tolist() == z[k + ":yseq"].tolist(), (k, hyp.yseq.tolist(), z[k + ":yseq"].tolist())
        assert token_int == z[k + ":token_int"].tolist() and token == [token_list[t] for t in token_int], k
        ref = float(z[k + ":score"])
        assert abs(float(hyp.score) - ref) <= 2e-4 * abs(ref) + 2e-3, (k, float(hyp.score), ref)
        assert sorted(hyp.scores) == sorted(f[len(k) + 7:] for f in z.files if f.startswith(k + ":score:"))
        for sk, v in hyp.scores.items():
            r = float(z[f"{k}:score:{sk}"])
            assert abs(float(v) - r) <= 2e-4 * abs(r) + 2e-3, (k, sk, float(v), r)


def _run_search(tmp_path, name, device, n_streams=1):
    z, paths = _files(tmp_path)
    s2t = _s2t(z, paths, name, device, n_streams)
    assert type(s2t.asr_model.encoder).__name__ == "ContextualBlockTransformerEncoder"
    wave, pushes = refbuild.waveform(*z["wave"].tolist()), z["pushes"].tolist()
    pos = 0
    for i, n in enumerate(pushes):
        chunk = wave[pos:pos + n]
        res = s2t(chunk if n_streams == 1 else chunk[None].repeat(n_streams, 1), is_final=(i == len(pushes) - 1))
        pos += n
        for per_stream in ([res] if n_streams == 1 else res):
            _check_nbest(z, f"{name}:{i}", per_stream)


def test_recipe_config_builds_and_loads_strictly(tmp_path):
    import espnet_b200

    z, paths = _files(tmp_path)
    with open(paths["config.yaml"]) as f:
        args = argparse.Namespace(**yaml.safe_load(f))
    assert args.encoder == "contextual_block_transformer"
    model = espnet_b200.build_model(args)
    model.load_state_dict(torch.load(paths["model.pth"]), strict=True)
    assert isinstance(model.encoder, espnet_b200.ContextualBlockTransformerEncoder) and model.encoder.input_layer == "conv2d"


@pytest.mark.parametrize("name", ["joint", "aishell"])
def test_streaming_search_host_logic_vs_reference_fixture(monkeypatch, tmp_path, name):
    import emu_backend
    import emu_rnnlm

    emu_rnnlm.install(monkeypatch)
    emu_backend.install_frontend(monkeypatch)
    _run_search(tmp_path, name, "cpu")
    assert "espb_ctc_extend_state_f32" in emu_backend.calls and "espb_cbe_ctx_propagate_f32" in emu_backend.calls


def test_streaming_cli_sim_chunk_length_writes_result_dir(monkeypatch, tmp_path):
    """bin_asr_inference_streaming.inference with the AISHELL recipe's --sim_chunk_length 512: the final n-best equals the reference's for
    the same 512-sample chunks."""
    import emu_backend
    from espnet_b200.bin_asr_inference_streaming import inference

    emu_backend.install_search(monkeypatch)
    emu_backend.install_frontend(monkeypatch)
    z, paths = _files(tmp_path)
    s2t = _s2t(z, paths, "joint", "cpu")
    np.save(tmp_path / "utt1.npy", refbuild.waveform(*z["wave"].tolist()).numpy())
    (tmp_path / "wav.scp").write_text(f"utt1 {tmp_path / 'utt1.npy'}\n")
    nbest = json.loads(str(z["settings"]))["joint"]["nbest"]
    out = inference(str(tmp_path / "dec"), [(str(tmp_path / "wav.scp"), "speech", "sound")], nbest=nbest, sim_chunk_length=512, speech2text=s2t)
    _check_nbest(z, "sim512:joint", out["utt1"])
    lines = dict(ln.split(maxsplit=1) for ln in (tmp_path / "dec/1best_recog/token_int").read_text().splitlines())
    assert lines["utt1"].split() == [str(t) for t in z["sim512:joint:0:token_int"].tolist()]
    assert (tmp_path / f"dec/{nbest}best_recog/score").exists()


# ---------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("il", LAYERS)
def test_encoder_cuda_vs_reference_fixture(il):
    one = _run_encoder(il, "cuda", 1)
    five = _run_encoder(il, "cuda", 5)
    for a, b in zip(one, five):
        assert a.shape == b.shape and (a.numel() == 0 or float((a - b).abs().max()) < 1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["joint", "aishell"])
@pytest.mark.parametrize("n_streams", [1, 3])
def test_streaming_search_cuda_vs_reference_fixture(tmp_path, name, n_streams):
    _run_search(tmp_path, name, "cuda", n_streams)


@pytest.mark.gpu
def test_streaming_cli_from_files_cuda(tmp_path):
    """The whole command line: config.yaml / checkpoint / LM files, AISHELL decode settings, --sim_chunk_length 512."""
    from espnet_b200.bin_asr_inference_streaming import main

    z, paths = _files(tmp_path)
    np.save(tmp_path / "utt1.npy", refbuild.waveform(*z["wave"].tolist()).numpy())
    (tmp_path / "wav.scp").write_text(f"utt1 {tmp_path / 'utt1.npy'}\n")
    main(["--output_dir", str(tmp_path / "dec"), "--data_path_and_name_and_type", f"{tmp_path / 'wav.scp'},speech,sound",
          "--asr_train_config", paths["config.yaml"], "--asr_model_file", paths["model.pth"], "--lm_train_config", paths["lm.yaml"],
          "--lm_file", paths["lm.pth"], "--sim_chunk_length", "512", "--beam_size", "10", "--ctc_weight", "0.6", "--lm_weight", "0.3",
          "--disable_repetition_detection", "true", "--nbest", "3"])
    for j in range(int(z["sim512:aishell:n"])):
        lines = dict(ln.split(maxsplit=1) for ln in (tmp_path / f"dec/{j + 1}best_recog/token_int").read_text().splitlines())
        assert lines["utt1"].split() == [str(t) for t in z[f"sim512:aishell:{j}:token_int"].tolist()]


@pytest.mark.gpu
def test_streaming_speech2text_ctc_greedy_equals_whole_utterance_collapse(tmp_path):
    """40-ms pushes, greedy=True: the tokens emitted push by push equal argmax / collapse of the concatenated encoder frames, in every
    stream of the lock-step batch."""
    import espnet_b200

    z, paths = _files(tmp_path)
    n_streams = 4
    s2t = espnet_b200.Speech2TextStreaming(asr_train_config=paths["config.yaml"], asr_model_file=paths["model.pth"], n_streams=n_streams,
                                           device="cuda", greedy=True)
    model = s2t.asr_model
    frames = []
    orig = model.encoder.forward

    def spy(*a, **k):
        out = orig(*a, **k)
        frames.append(out[0][0].clone())
        return out
    model.encoder.forward = spy
    wave = refbuild.waveform(*z["wave"].tolist())
    emitted = [[] for _ in range(n_streams)]
    for p in range(0, wave.numel(), 640):
        new = s2t(wave[None, p:p + 640].repeat(n_streams, 1), is_final=(p + 640 >= wave.numel()))
        for s in range(n_streams):
            emitted[s] += new[s]
    am = model.ctc.argmax(torch.cat(frames, 0)[None])[0].cpu().tolist()
    ref = [t for i, t in enumerate(am) if t != 0 and (i == 0 or am[i - 1] != t)]
    assert emitted[0] == ref and len(ref) > 0
    assert all(e == emitted[0] for e in emitted)
    assert s2t.final_tokens[0] == ref


@pytest.mark.gpu
def test_offline_speech2text_refuses_the_streaming_encoder(tmp_path):
    import espnet_b200

    _, paths = _files(tmp_path)
    with pytest.raises(NotImplementedError):
        espnet_b200.Speech2Text(asr_train_config=paths["config.yaml"], asr_model_file=paths["model.pth"], device="cuda")
