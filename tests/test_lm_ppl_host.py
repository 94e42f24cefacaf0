"""LM perplexity (espnet_b200.ESPnetLanguageModel.nll / batchify_nll, espnet_b200.lm_calc_perplexity) on the host: loading reference
checkpoints, the sos / eos / padding logic of nll and the full-sequence forwards with the C-ABI entry points emulated (tests/emu_lm_ppl.py),
the files calc_perplexity writes, and the refusals.  Against tests/golden/lm_ppl.npz (make_golden_lm_ppl.py, the UNMODIFIED reference)."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch
import yaml

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LMS = ("tfm64", "tfm32", "lstm")


def _z():
    return np.load(os.path.join(GOLDEN, "lm_ppl.npz"))


def _weights(z, name):
    p = f"{name}:w:"
    return {k[len(p):]: torch.from_numpy(z[k]).float() for k in z.files if k.startswith(p)}   # stored as float16, exactly


def write_lm(z, name, root):
    """The LM's config.yaml and checkpoint as the reference's LM training writes them -> (config path, model path)."""
    kind, conf = json.loads(str(z["lms"]))[name]
    cfg, mdl = os.path.join(root, f"{name}.yaml"), os.path.join(root, f"{name}.pth")
    yaml.safe_dump(dict(token_list=json.loads(str(z["token_list"])), token_type="char", bpemodel=None, lm=kind, lm_conf=conf,
                        model_conf=dict(ignore_id=0), use_preprocessor=True, cleaner=None, g2p=None, non_linguistic_symbols=None, init=None),
                   open(cfg, "w"))
    torch.save(_weights(z, name), mdl)
    return cfg, mdl


def write_text(z, root):
    path = os.path.join(root, "text")
    with open(path, "w", encoding="utf-8") as f:
        for k, t in json.loads(str(z["texts"])):
            f.write(f"{k} {t}\n")
    return path


def check_ppl_files(z, name, tag, out_dir):
    """utt2ntokens and base as the reference wrote them, utt2ppl and ppl within rtol 1e-4, the same keys in the same order."""
    rd = lambda fn: open(os.path.join(out_dir, fn), encoding="utf-8").read()  # noqa: E731
    assert rd("utt2ntokens") == str(z[f"{name}:{tag}:utt2ntokens"])
    assert rd("base") == str(z[f"{name}:{tag}:base"])
    got = [ln.split() for ln in rd("utt2ppl").splitlines()]
    want = [ln.split() for ln in str(z[f"{name}:{tag}:utt2ppl"]).splitlines()]
    assert [g[0] for g in got] == [w[0] for w in want]
    np.testing.assert_allclose([float(g[1]) for g in got], [float(w[1]) for w in want], rtol=1e-4)
    np.testing.assert_allclose(float(rd("ppl")), float(str(z[f"{name}:{tag}:ppl"])), rtol=1e-4)


@pytest.mark.parametrize("name", LMS)
def test_reference_checkpoint_loads_strictly(name, tmp_path):
    import espnet_b200

    z = _z()
    cfg, mdl = write_lm(z, name, str(tmp_path))
    model, args = espnet_b200.build_espnet_lm_from_file(cfg, mdl, device="cpu")
    assert isinstance(model, espnet_b200.ESPnetLanguageModel)
    assert sorted(model.state_dict()) == sorted(_weights(z, name))
    model.load_state_dict(_weights(z, name), strict=True)
    assert model.sos == model.eos == int(z["V"]) - 1 and model.ignore_id == 0


@pytest.mark.parametrize("name", LMS)
def test_nll_host_logic_emulated(name, monkeypatch, tmp_path):
    """nll (sos / eos, padding, positions past text_lengths + 1 zeroed, a real token 0 masked as a key and scored as a target) and
    batchify_nll's max_length branch through the emulated kernels, against the reference's own values."""
    import emu_lm_ppl

    import espnet_b200

    emu_lm_ppl.install(monkeypatch)
    z = _z()
    model, _ = espnet_b200.build_espnet_lm_from_file(*write_lm(z, name, str(tmp_path)), device="cpu")
    text, lengths = torch.from_numpy(z["text"]), torch.from_numpy(z["lengths"])
    nll, xl = model.nll(text, lengths)
    assert nll.shape == z[f"{name}:nll"].shape and torch.equal(xl, torch.from_numpy(z[f"{name}:x_lengths"]))
    np.testing.assert_allclose(nll.numpy(), z[f"{name}:nll"], atol=1e-4, rtol=0)
    nll2, xl2 = model.batchify_nll(text, lengths, batch_size=2)
    np.testing.assert_allclose(nll2.numpy(), z[f"{name}:batchify_nll"], atol=1e-4, rtol=0)
    assert torch.equal(xl2, xl)
    logits, hidden = model.lm(text[:2, :8], None)
    assert hidden is None and logits.shape == (2, 8, int(z["V"]))


@pytest.mark.parametrize("log_base", [None, 10.0])
def test_calc_perplexity_files_emulated(log_base, monkeypatch, tmp_path):
    """The files and their format (utt2ppl, utt2ntokens, ppl, base) as the reference writes them, with log_base e and 10."""
    import emu_lm_ppl

    import espnet_b200.lm_calc_perplexity as lcp

    emu_lm_ppl.install(monkeypatch)
    build = lcp.build_espnet_lm_from_file
    monkeypatch.setattr(lcp, "build_espnet_lm_from_file", lambda c, m, device: build(c, m, device="cpu"))
    z = _z()
    cfg, mdl = write_lm(z, "lstm", str(tmp_path))
    out = str(tmp_path / "out")
    lcp.calc_perplexity(output_dir=out, batch_size=2, dtype="float32", ngpu=1, seed=0, num_workers=1, log_level="WARNING",
                        data_path_and_name_and_type=[(write_text(z, str(tmp_path)), "text", "text")], key_file=None, train_config=cfg,
                        model_file=mdl, log_base=log_base, allow_variable_data_keys=False)
    check_ppl_files(z, "lstm", "e" if log_base is None else "b10", out)


def test_refusals(tmp_path):
    import espnet_b200.lm_calc_perplexity as lcp
    from espnet_b200.bin_lm_calc_perplexity import get_parser

    z = _z()
    cfg, mdl = write_lm(z, "lstm", str(tmp_path))
    kw = dict(output_dir=str(tmp_path / "o"), batch_size=1, ngpu=1, seed=0, num_workers=1, log_level="WARNING",
              data_path_and_name_and_type=[(write_text(z, str(tmp_path)), "text", "text")], key_file=None, train_config=cfg, model_file=mdl,
              log_base=None, allow_variable_data_keys=False)
    for dtype in ("float16", "float64"):
        with pytest.raises(NotImplementedError):
            lcp.calc_perplexity(dtype=dtype, **kw)
    with pytest.raises(SystemExit):
        get_parser().parse_args(["--output_dir", "o", "--data_path_and_name_and_type", "t,text,text", "--dtype", "float16"])
    for token_type in ("phn", "hugging_face"):
        args = yaml.safe_load(open(cfg))
        with pytest.raises(NotImplementedError):
            lcp.text_to_ids(type("A", (), dict(args, token_type=token_type))())
    with pytest.raises(NotImplementedError):
        lcp.text_to_ids(type("A", (), dict(yaml.safe_load(open(cfg)), non_linguistic_symbols="nlsyms.txt"))())
    (tmp_path / "bad").write_text("utt1 hello\nutt2\n")
    with pytest.raises(RuntimeError):
        list(lcp.read_text(str(tmp_path / "bad")))
    a = get_parser().parse_args(["--output_dir", "o", "--data_path_and_name_and_type", "t,text,text", "--log_base", "none"])
    assert a.log_base is None and a.data_path_and_name_and_type == [("t", "text", "text")] and a.batch_size == 1


def test_tokenizers_text2tokens():
    from espnet_b200.text import build_tokenizer

    assert build_tokenizer("char").text2tokens("it's a") == ["i", "t", "'", "s", "<space>", "a"]
    assert build_tokenizer("word").text2tokens("hello  world") == ["hello", "world"]


def test_capi_entry_points_bound():
    from espnet_b200 import lib

    for name, n in (("espb_causal_flash_attn_f32", 21), ("espb_causal_softmax_f32", 11), ("espb_nll_rows_f32", 7)):
        assert len(lib._SIGS[name]) == n and name in lib.EXPORTED_SYMBOLS
    if os.path.exists(lib.LIB_PATH):
        handle = ctypes.CDLL(lib.LIB_PATH)
        for name in ("espb_causal_flash_attn_f32", "espb_causal_softmax_f32", "espb_nll_rows_f32"):
            assert hasattr(handle, name)
