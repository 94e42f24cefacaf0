"""refbuild.model_yaml extended with the E-Branchformer encoder (cfg["encoder"] == "e_branchformer").  Test infrastructure.

cfg keys of that encoder (ints, as fixtures store cfg as int64): d_model, heads, enc_layers, cgmlp (cgmlp_linear_units), cgmlp_kernel,
merge_kernel, use_ffn, macaron, ff (FFN and decoder linear units).  Every other model setting is refbuild's.

The E-Branchformer fixtures do not store their random weights: every parameter is a function of (seed, name, shape), computed by
seeded_weights() below the same way when the fixture is made and when it is read, and the fixture records the seed and each parameter's
name and shape (f"{prefix}pshape:{name}").  Non-parameter state (the mel matrix) is stored as before (f"{prefix}w:{name}").
"""
import math
import zlib

import numpy as np
import torch

import refbuild

_base_model_yaml = refbuild.model_yaml


def encoder_conf(cfg):
    return dict(output_size=cfg["d_model"], attention_heads=cfg["heads"], attention_layer_type="rel_selfattn", pos_enc_layer_type="rel_pos",
                rel_pos_type="latest", cgmlp_linear_units=cfg["cgmlp"], cgmlp_conv_kernel=cfg["cgmlp_kernel"], use_linear_after_conv=False,
                gate_activation="identity", num_blocks=cfg["enc_layers"], dropout_rate=0.1, positional_dropout_rate=0.1,
                attention_dropout_rate=0.0, input_layer="conv2d", use_ffn=bool(cfg["use_ffn"]), macaron_ffn=bool(cfg["macaron"]),
                ffn_activation_type="swish", linear_units=cfg["ff"], positionwise_layer_type="linear", merge_conv_kernel=cfg["merge_kernel"],
                use_flash_attn=False)


def model_yaml(cfg):
    y = _base_model_yaml(cfg)
    if cfg.get("encoder") == "e_branchformer":
        y["encoder"], y["encoder_conf"] = "e_branchformer", encoder_conf(cfg)
    return y


def seeded_weights(shapes, seed):
    """{name: shape} -> {name: float32 tensor}, identical on every machine: integers drawn from torch's CPU generator (seeded per name), divided
    by a power of two, then one IEEE-rounded scaling -- no transcendental functions, so no dependence on the host's math library or vector
    width.  Ranges follow PyTorch's default initialisation: weights of rank >= 2 uniform in +-1/sqrt(fan_in); LayerNorm weights 1 +- 0.2
    and biases +-0.2 (away from 1 / 0, so that a normalised padded row -- beta, not 0 -- is visible); other biases +-0.1."""
    out = {}
    for name, shape in shapes.items():
        shape = tuple(int(v) for v in shape)
        g = torch.Generator().manual_seed(seed * 1000003 + zlib.crc32(name.encode()))
        u = torch.randint(-32768, 32768, shape, generator=g, dtype=torch.int64).to(torch.float32) / 32768.0
        if len(shape) >= 2:
            w = u * (1.0 / math.sqrt(math.prod(shape[1:])))
        elif "norm" in name and name.endswith("weight"):
            w = 1.0 + 0.2 * u
        elif "norm" in name:
            w = 0.2 * u
        else:
            w = 0.1 * u
        out[name] = w.contiguous()
    return out


def seeded_state(named_params, seed):
    """Overwrite parameters in place with seeded_weights; returns the {name: shape} record the fixture stores."""
    named_params = list(named_params)
    shapes = {k: tuple(p.shape) for k, p in named_params}
    w = seeded_weights(shapes, seed)
    params = dict(named_params)
    with torch.no_grad():
        for k, p in params.items():
            p.copy_(w[k])
    return shapes


def fixture_weights(z, prefix=""):
    """All weights of a fixture written this way: the seeded parameters plus the stored non-parameter entries."""
    seed = int(z[f"{prefix}wseed"])
    shapes = {k[len(prefix) + 7:]: z[k].tolist() for k in z.files if k.startswith(f"{prefix}pshape:")}
    w = seeded_weights(shapes, seed)
    w.update({k[len(prefix) + 2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith(f"{prefix}w:")})
    return w


def shape_record(shapes, seed, prefix=""):
    z = {f"{prefix}pshape:{k}": np.array(v, dtype=np.int64) for k, v in shapes.items()}
    z[f"{prefix}wseed"] = np.array(seed, dtype=np.int64)
    return z


def install():
    """Route refbuild.model_yaml (and with it refbuild.build_reference, gpu_util.speech2text) through model_yaml above."""
    refbuild.model_yaml = model_yaml
