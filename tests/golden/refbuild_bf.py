"""refbuild.model_yaml extended with the Branchformer encoder (cfg["encoder"] == "branchformer").  Test infrastructure.

cfg keys of that encoder (ints, as fixtures store cfg as int64): d_model, heads, enc_layers, cgmlp (cgmlp_linear_units), cgmlp_kernel,
merge (index into MERGES), use_attn, use_cgmlp, ff (decoder linear units).  fixed_ave's per-layer cgmlp_weight is a float list kept beside
the cfg.  Every other model setting is refbuild's.

The fixtures do not store their random weights: they are rebuilt with refbuild_ebf.seeded_weights from the recorded seed and the reference's
parameter names and shapes (refbuild_ebf.fixture_weights).
"""
import refbuild
from refbuild_ebf import fixture_weights, seeded_state, seeded_weights, shape_record  # noqa: F401

MERGES = ("concat", "learned_ave", "fixed_ave")

_base_model_yaml = refbuild.model_yaml


def encoder_conf(cfg, cgmlp_weight=0.5):
    return dict(output_size=cfg["d_model"], use_attn=bool(cfg.get("use_attn", 1)), attention_heads=cfg["heads"],
                attention_layer_type="rel_selfattn", pos_enc_layer_type="rel_pos", rel_pos_type="latest", use_cgmlp=bool(cfg.get("use_cgmlp", 1)),
                cgmlp_linear_units=cfg["cgmlp"], cgmlp_conv_kernel=cfg["cgmlp_kernel"], use_linear_after_conv=False, gate_activation="identity",
                merge_method=MERGES[cfg.get("merge", 0)],
                cgmlp_weight=[float(v) for v in cgmlp_weight] if isinstance(cgmlp_weight, (list, tuple)) else float(cgmlp_weight),
                attn_branch_drop_rate=0.0, num_blocks=cfg["enc_layers"], dropout_rate=0.1, positional_dropout_rate=0.1, attention_dropout_rate=0.0,
                input_layer="conv2d", stochastic_depth_rate=0.0, use_flash_attn=False)


def model_yaml(cfg):
    y = _base_model_yaml(cfg)
    if cfg.get("encoder") == "branchformer":
        y["encoder"], y["encoder_conf"] = "branchformer", encoder_conf(cfg)
    return y


def install():
    """Route refbuild.model_yaml (and with it refbuild.build_reference, gpu_util.speech2text) through model_yaml above."""
    refbuild.model_yaml = model_yaml
