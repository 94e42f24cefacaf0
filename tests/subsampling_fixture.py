"""Readers of tests/golden/subsampling_enc.npz (tests/golden/make_golden_subsampling.py): the nine (encoder, input layer) cases, the CUDA-path
encoder of each case built and loaded strictly, and the oracle that computes it."""
import os
import sys

import numpy as np
import torch

from golden_util import GOLDEN_DIR

sys.path.insert(0, GOLDEN_DIR)
import refbuild_ebf  # noqa: E402

PAIRS = [(e, il) for e in ("conformer", "transformer", "e_branchformer") for il in ("conv2d2", "conv2d6", "conv2d8")]
_Z = None


def load_case(encoder, input_layer):
    """(fixture, tag, cfg, weights with the reference's state_dict names: the seeded parameters plus the stored buffers)."""
    global _Z
    if _Z is None:
        _Z = np.load(os.path.join(GOLDEN_DIR, "subsampling_enc.npz"))
    tag = f"{encoder}:{input_layer}:"
    cfg = dict(zip(_Z[f"{tag}cfg_keys"].tolist(), (int(v) for v in _Z[f"{tag}cfg_vals"])))
    shapes = {k: [v for v in shp if v >= 0] for k, shp in zip(_Z[f"{tag}pnames"].tolist(), _Z[f"{tag}pshapes"].tolist())}
    w = refbuild_ebf.seeded_weights(shapes, int(_Z[f"{tag}wseed"]))
    w.update({k[len(tag) + 2:]: torch.from_numpy(_Z[k]) for k in _Z.files if k.startswith(f"{tag}w:")})
    return _Z, tag, cfg, w


def feats(z, tag):
    """The case's input features (stored as float16, exactly the float32 values the reference saw)."""
    return torch.from_numpy(z[f"{tag}feats"]).float()


def encoder_kwargs(encoder, input_layer, cfg):
    """Constructor arguments of the espnet_b200 encoder, as the fixture's reference encoder was built (make_golden_subsampling.encoder_conf)."""
    if encoder == "e_branchformer":
        return dict(refbuild_ebf.encoder_conf(cfg), input_layer=input_layer)
    common = dict(output_size=cfg["d_model"], attention_heads=cfg["heads"], linear_units=cfg["ff"], num_blocks=cfg["enc_layers"],
                  input_layer=input_layer, normalize_before=True)
    if encoder == "transformer":
        return common
    return dict(common, macaron_style=True, rel_pos_type="latest", pos_enc_layer_type="rel_pos", selfattention_layer_type="rel_selfattn",
                activation_type="swish", use_cnn_module=True, cnn_module_kernel=cfg["kernel"])


def build_encoder(encoder, input_layer, cfg, w):
    import espnet_b200

    cls = {"conformer": espnet_b200.ConformerEncoder, "transformer": espnet_b200.TransformerEncoder,
           "e_branchformer": espnet_b200.EBranchformerEncoder}[encoder]
    enc = cls(80, **encoder_kwargs(encoder, input_layer, cfg))
    enc.load_state_dict({k[len("encoder."):]: v for k, v in w.items()}, strict=True)
    return enc.eval()


def oracle_encode(encoder, input_layer, cfg, w, x):
    """(output, [embed output, block 1, ...]) of one utterance."""
    from oracle.subsampling import encode

    return encode(encoder, input_layer, x, w, cfg["heads"], cfg["enc_layers"], return_layers=True)
