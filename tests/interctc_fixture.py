"""Readers of the intermediate-CTC fixtures (tests/golden/make_golden_interctc.py): the encoder cases of interctc_enc.npz with the CUDA-path
encoder and CTC head of each case built and loaded strictly, and the whole-model fixtures interctc_s2t.npz / interctc_ctconly.npz."""
import os
import sys

import numpy as np
import torch

from golden_util import GOLDEN_DIR

sys.path.insert(0, GOLDEN_DIR)
import refbuild_ebf  # noqa: E402
import refbuild_interctc  # noqa: E402

CASES = ["conf64", "conf16", "tfm64", "noc"]
_Z = {}


def _npz(name):
    if name not in _Z:
        _Z[name] = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    return _Z[name]


def load_case(case):
    """(fixture, tag, cfg, listed layers, weights with the reference's state_dict names: encoder.* and ctc.*)."""
    z, tag = _npz("interctc_enc"), case + ":"
    cfg = dict(zip(z[f"{tag}cfg_keys"].tolist(), (int(v) for v in z[f"{tag}cfg_vals"])))
    return z, tag, cfg, z[f"{tag}idx"].tolist(), refbuild_ebf.fixture_weights(z, tag)


def feats(z, tag):
    return torch.from_numpy(z[f"{tag}feats"]).float()


def encoder_kwargs(cfg):
    common = dict(output_size=cfg["d_model"], attention_heads=cfg["heads"], linear_units=cfg["ff"], num_blocks=cfg["enc_layers"],
                  input_layer="conv2d", normalize_before=True, **refbuild_interctc.interctc_conf(cfg))
    if cfg["tfm"]:
        return common
    return dict(common, macaron_style=True, rel_pos_type="latest", pos_enc_layer_type="rel_pos", selfattention_layer_type="rel_selfattn",
                activation_type="swish", use_cnn_module=True, cnn_module_kernel=cfg["kernel"])


def build(cfg, w, device="cpu"):
    """(encoder, CTC head) of a case, as ESPnetASRModel builds them (conditioning_layer = Linear(vocab, d)), loaded with strict=True."""
    import espnet_b200

    enc = (espnet_b200.TransformerEncoder if cfg["tfm"] else espnet_b200.ConformerEncoder)(80, **encoder_kwargs(cfg))
    if enc.interctc_use_conditioning:
        enc.conditioning_layer = torch.nn.Linear(cfg["vocab"], cfg["d_model"])
    enc.load_state_dict({k[len("encoder."):]: v for k, v in w.items() if k.startswith("encoder.")}, strict=True)
    ctc = espnet_b200.CTC(cfg["vocab"], cfg["d_model"])
    ctc.load_state_dict({k[len("ctc."):]: v for k, v in w.items() if k.startswith("ctc.")}, strict=True)
    return enc.to(device).eval(), ctc.to(device).eval()


def oracle(cfg, w, idx, x):
    """(output, [(layer, intermediate output)], block outputs) of one utterance, float64."""
    from oracle.interctc import encode

    return encode(x, w, cfg["heads"], cfg["enc_layers"], idx, bool(cfg["ic_cond"]), transformer=bool(cfg["tfm"]))


def load_model_fixture(name):
    """interctc_s2t / interctc_ctconly -> (fixture, cfg, weights of the whole model)."""
    z = _npz(name)
    cfg = {k: int(v) for k, v in zip(z["cfg_keys"].tolist(), z["cfg_vals"].tolist())}
    return z, cfg, refbuild_ebf.fixture_weights(z)
