"""Generate the input-layer fixtures from the UNMODIFIED reference (build container only).

    python tests/golden/make_golden_subsampling.py

subsampling_enc.npz: the reference ConformerEncoder, TransformerEncoder and EBranchformerEncoder with input_layer conv2d2, conv2d6 and
  conv2d8 (Conv2dSubsampling2/6/8, espnet2/legacy/nets/pytorch_backend/transformer/subsampling.py:590-860) on seeded features, one
  utterance per call: nine cases under the prefix "{encoder}:{input_layer}:", each with feats, the embed output ("layer0"), every block
  output ("layer1".."layerL"), the output and olens.
  One case per encoder has d_k 64 (the fused attention kernel), the others d_k 16 (the materialised attention).  The features are drawn,
  rounded to float16 and fed to the reference as float32, so storing them as float16 loses nothing.
subsampling_s2t.npz: the reference Speech2Text with a conv2d6 Conformer encoder, 2 decoder layers, V 50 (the five decode settings of
  make_golden.py); its input layer under "input_layer".
Weights are not stored: parameters come from refbuild_ebf.seeded_weights (the fixtures record the seed and each parameter's name and
shape: "{prefix}pnames" / "{prefix}pshapes" in subsampling_enc.npz, "pshape:{name}" in subsampling_s2t.npz); the non-parameter state (BatchNorm running statistics, drawn from a seeded generator for the encoder cases; the mel matrix) is
stored ("w:").
"""
import logging
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import refshim  # noqa: E402
import refbuild  # noqa: E402
import refbuild_ebf  # noqa: E402
import refbuild_subsampling  # noqa: E402

logging.disable(logging.WARNING)
refshim.install()
import make_golden  # noqa: E402
from espnet2.asr.encoder.conformer_encoder import ConformerEncoder  # noqa: E402
from espnet2.asr.encoder.e_branchformer_encoder import EBranchformerEncoder  # noqa: E402
from espnet2.asr.encoder.transformer_encoder import TransformerEncoder  # noqa: E402

# (encoder, input_layer) -> cfg; d_model / heads = 128 / 2 is the d_k 64 case of each encoder.  Frame counts have different residues
# modulo 6 and 8.
ENC_CASES = {
    ("conformer", "conv2d2"): dict(d_model=64, heads=4, ff=128, kernel=15, enc_layers=2, nframes=81),
    ("conformer", "conv2d6"): dict(d_model=128, heads=2, ff=256, kernel=31, enc_layers=2, nframes=119),
    ("conformer", "conv2d8"): dict(d_model=64, heads=4, ff=128, kernel=15, enc_layers=2, nframes=131),
    ("transformer", "conv2d2"): dict(d_model=64, heads=4, ff=128, enc_layers=2, nframes=75),
    ("transformer", "conv2d6"): dict(d_model=64, heads=4, ff=128, enc_layers=2, nframes=106),
    ("transformer", "conv2d8"): dict(d_model=128, heads=2, ff=256, enc_layers=2, nframes=141),
    ("e_branchformer", "conv2d2"): dict(d_model=64, heads=4, cgmlp=192, cgmlp_kernel=15, merge_kernel=3, use_ffn=1, macaron=1, ff=128,
                                        enc_layers=2, nframes=85),
    ("e_branchformer", "conv2d6"): dict(d_model=64, heads=4, cgmlp=192, cgmlp_kernel=15, merge_kernel=3, use_ffn=0, macaron=0, ff=2048,
                                        enc_layers=2, nframes=125),
    ("e_branchformer", "conv2d8"): dict(d_model=128, heads=2, cgmlp=256, cgmlp_kernel=31, merge_kernel=31, use_ffn=1, macaron=1, ff=192,
                                        enc_layers=2, nframes=118),
}
S2T = dict(cfg=dict(d_model=64, heads=4, ff=128, enc_layers=2, dec_layers=2, vocab=50, kernel=15), nsamples=16000, wave_id=11)
S2T_INPUT_LAYER = "conv2d6"
S2T_SEED = 13


def encoder_conf(encoder, input_layer, cfg):
    """Keyword arguments of the reference encoder class for a fixture cfg."""
    d, h = cfg["d_model"], cfg["heads"]
    if encoder == "e_branchformer":
        return dict(refbuild_ebf.encoder_conf(cfg), input_layer=input_layer)
    common = dict(output_size=d, attention_heads=h, linear_units=cfg["ff"], num_blocks=cfg["enc_layers"], dropout_rate=0.1,
                  positional_dropout_rate=0.1, attention_dropout_rate=0.0, input_layer=input_layer, normalize_before=True,
                  use_flash_attn=False)
    if encoder == "transformer":
        return common
    return dict(common, macaron_style=True, rel_pos_type="latest", pos_enc_layer_type="rel_pos", selfattention_layer_type="rel_selfattn",
                activation_type="swish", use_cnn_module=True, cnn_module_kernel=cfg["kernel"])


ENCODERS = {"conformer": ConformerEncoder, "transformer": TransformerEncoder, "e_branchformer": EBranchformerEncoder}


def encoder_case(encoder, input_layer, cfg, seed):
    tag = f"{encoder}:{input_layer}:"
    enc = ENCODERS[encoder](80, **encoder_conf(encoder, input_layer, cfg)).eval()
    shapes = refbuild_ebf.seeded_state([("encoder." + k, p) for k, p in enc.named_parameters()], seed)
    g = torch.Generator().manual_seed(200 + seed)
    z = {}
    with torch.no_grad():
        for m in enc.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.running_mean.copy_(0.1 * torch.randn(m.running_mean.shape, generator=g))
                m.running_var.copy_(0.5 + torch.rand(m.running_var.shape, generator=g))
        for k, v in enc.named_buffers():
            z[f"{tag}w:encoder.{k}"] = v.numpy().copy()
        feats = torch.randn(1, cfg["nframes"], 80, generator=g).half().float()
        layers = []

        def first(o):   # conformer / e-branchformer modules return ((x, pos_emb), mask), transformer modules (x, mask)
            x = o[0]
            return (x[0] if isinstance(x, tuple) else x)[0].clone()

        hooks = [enc.embed.register_forward_hook(lambda m, i, o: layers.append(first(o)))]
        hooks += [lyr.register_forward_hook(lambda m, i, o: layers.append(first(o))) for lyr in enc.encoders]
        out, olens, _ = enc(feats, torch.tensor([cfg["nframes"]]))
        for h in hooks:
            h.remove()
    assert len(layers) == cfg["enc_layers"] + 1
    z.update({f"{tag}cfg_keys": np.array(list(cfg.keys())), f"{tag}cfg_vals": np.array(list(cfg.values()), dtype=np.int64),
              f"{tag}feats": feats[0].half().numpy(), f"{tag}out": out[0].numpy(), f"{tag}olens": olens.numpy()})
    for i, t in enumerate(layers):
        z[f"{tag}layer{i}"] = t.numpy()
    z.update(shape_record(shapes, seed, tag))
    return z


def shape_record(shapes, seed, tag):
    """{name: shape} of the seeded parameters as two arrays: the names, and the shapes padded to rank 4 with -1."""
    assert max(len(v) for v in shapes.values()) <= 4
    return {f"{tag}pnames": np.array(list(shapes)), f"{tag}wseed": np.array(seed, dtype=np.int64),
            f"{tag}pshapes": np.array([list(v) + [-1] * (4 - len(v)) for v in shapes.values()], dtype=np.int64)}


if __name__ == "__main__":
    z = {}
    for i, ((encoder, input_layer), cfg) in enumerate(ENC_CASES.items()):
        z.update(encoder_case(encoder, input_layer, cfg, i + 21))
    path = os.path.join(HERE, "subsampling_enc.npz")
    np.savez_compressed(path, **z)
    print("subsampling_enc.npz", os.path.getsize(path) // 1024, "KiB")

    refbuild_subsampling.install()
    build_reference = refbuild.build_reference

    def build_seeded(cfg, seed=0, **kw):
        """refbuild.build_reference with the conv2d6 input layer and every parameter replaced by refbuild_ebf.seeded_weights(S2T_SEED)."""
        s2t = build_reference(dict(cfg, input_layer=S2T_INPUT_LAYER), seed=seed, **kw)
        refbuild_ebf.seeded_state(s2t.asr_model.named_parameters(), S2T_SEED)
        return s2t

    refbuild.build_reference = build_seeded
    make_golden.run_case("subsampling_s2t", S2T)
    # keep the non-parameter state and replace the stored parameters by their seed / shape record
    path = os.path.join(HERE, "subsampling_s2t.npz")
    z = dict(np.load(path))
    params = dict(build_seeded(S2T["cfg"]).asr_model.named_parameters())
    for k in params:
        assert np.array_equal(z.pop("w:" + k), params[k].detach().numpy()), k
    z.update(refbuild_ebf.shape_record({k: tuple(p.shape) for k, p in params.items()}, S2T_SEED))
    z["input_layer"] = np.array(S2T_INPUT_LAYER)
    np.savez_compressed(path, **z)
    print("subsampling_s2t.npz", os.path.getsize(path) // 1024, "KiB; stored weights:", sorted(k for k in z if k.startswith("w:")))
