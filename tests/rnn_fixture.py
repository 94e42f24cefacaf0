"""Shared helpers of the RNN model family tests: the fixture tests/golden/rnn.npz (make_golden_rnn.py) and the models built from it."""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import refbuild_ebf  # noqa: E402

ENC_CASES = ("vgg_blstmp", "vgg_blstm", "vgg_lstmp", "rnn_sub")
DECODES = ("ctc03", "ctc05", "ctc10", "ctxres", "lm", "tlm")   # decodes of the fixture waveform ("cli": its 16-bit PCM rounding)

_Z = None


def load():
    global _Z
    if _Z is None:
        _Z = np.load(os.path.join(HERE, "golden", "rnn.npz"))
    return _Z


def enc_case(case):
    """-> (cls name, constructor keywords, weights without the 'encoder.' prefix, feats (1, T, 80) float32)."""
    z = load()
    conf = json.loads(str(z[f"{case}:conf"]))
    cls = conf.pop("cls")
    w = {k[len("encoder."):]: v for k, v in refbuild_ebf.fixture_weights(z, f"{case}:").items()}
    return cls, conf, w, torch.from_numpy(z[f"{case}:feats"].astype(np.float32))


def build_encoder(case, device="cpu"):
    import espnet_b200

    cls, conf, w, feats = enc_case(case)
    enc = {"vgg_rnn": espnet_b200.VGGRNNEncoder, "rnn": espnet_b200.RNNEncoder}[cls](80, **conf)
    enc.load_state_dict(w, strict=True)
    return enc.to(device).eval(), feats


def model_config(model):
    return json.loads(str(load()[f"{model}:cfg"]))


def model_weights(model):
    return refbuild_ebf.fixture_weights(load(), f"{model}:")


def lm_config(name):
    return json.loads(str(load()[f"{name}:cfg"]))


def lm_weights(name):
    return refbuild_ebf.fixture_weights(load(), f"{name}:")


def decode(dn):
    """-> (model name, dict(beam_size, ctc_weight, lm_weight, maxlenratio), LM name ("lm" / "tlm") or "", [(yseq, score)])."""
    z = load()
    beam, cw, lw, mlr = z[f"{dn}:params"].tolist()
    kw = dict(beam_size=int(beam), ctc_weight=cw, maxlenratio=mlr, nbest=10)
    if lw:
        kw["lm_weight"] = lw
    hyps = [(z[f"{dn}:{i}:yseq"].tolist(), float(z[f"{dn}:{i}:score"])) for i in range(int(z[f"{dn}:n"]))]
    return str(z[f"{dn}:model"]), kw, str(z[f"{dn}:lm"]), hyps


def write_model_files(tmp_path, model):
    """Recipe-style exp dir: config.yaml + a checkpoint of the fixture weights -> (config path, checkpoint path)."""
    import yaml

    cfg = tmp_path / f"{model}_config.yaml"
    cfg.write_text(yaml.safe_dump(model_config(model)))
    ckpt = tmp_path / f"{model}.pth"
    torch.save(model_weights(model), str(ckpt))
    return str(cfg), str(ckpt)


def write_lm_files(tmp_path, name):
    import yaml

    cfg = tmp_path / f"{name}_config.yaml"
    cfg.write_text(yaml.safe_dump(lm_config(name)))
    ckpt = tmp_path / f"{name}.pth"
    torch.save({"lm." + k: v for k, v in lm_weights(name).items()}, str(ckpt))
    return str(cfg), str(ckpt)
