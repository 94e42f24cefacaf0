"""Generate the intermediate-CTC fixtures from the UNMODIFIED reference (build container only).

    python tests/golden/make_golden_interctc.py

interctc_enc.npz: the reference ConformerEncoder / TransformerEncoder with interctc_layer_idx (conformer_encoder.py:317-321,375-426,
  transformer_encoder.py:210-214,268-299), called as ESPnetASRModel.encode calls them (espnet_model.py:412-425): encoder(feats, lens,
  ctc=ctc) with a reference CTC head and encoder.conditioning_layer = Linear(vocab, d) (espnet_model.py:104-107).  Cases under the prefix
  "{case}:" (ENC_CASES): d_k 64 (fused attention) and d_k 16 (materialised attention) Conformers and a d_k 64 Transformer, each with two
  conditioned layers, and a Conformer with one listed layer and no conditioning.  Each case stores feats (float16-exact), every block output
  ("layer1".."layerL", before the conditioning is added), every intermediate output ("inter{l}"), the output and olens, "idx" (the listed
  layers), and the BatchNorm running statistics (drawn from a seeded generator).
interctc_s2t.npz: the reference Speech2Text with a self-conditioned Conformer (layers 1 and 2 of 3), V 50: the encoder output and the
  intermediate outputs, CTC greedy ids, and the n-best of the five decode settings of make_golden.py ("dec:{name}:...").
interctc_ctconly.npz: the same encoder in a model without a decoder (ctc_weight 1.0, as the LibriSpeech-100 train_conformer_scctc.yaml
  recipe), decoded CTC-only with beam 4 and beam 10.
Weights are not stored: parameters come from refbuild_ebf.seeded_weights (the fixtures record the seed and each parameter's name and
shape); the non-parameter state is stored ("w:").
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
import refbuild_interctc  # noqa: E402

logging.disable(logging.WARNING)
refshim.install()
import make_golden  # noqa: E402
from espnet2.asr.ctc import CTC  # noqa: E402
from espnet2.asr.encoder.conformer_encoder import ConformerEncoder  # noqa: E402
from espnet2.asr.encoder.transformer_encoder import TransformerEncoder  # noqa: E402

# tfm = 1: TransformerEncoder; ic_a / ic_b: listed layers (0 = none); ic_cond: self-conditioning
ENC_CASES = {
    "conf64": dict(tfm=0, d_model=128, heads=2, ff=256, kernel=15, enc_layers=4, vocab=37, ic_a=1, ic_b=3, ic_cond=1, nframes=203),
    "conf16": dict(tfm=0, d_model=64, heads=4, ff=128, kernel=15, enc_layers=3, vocab=50, ic_a=1, ic_b=2, ic_cond=1, nframes=161),
    "tfm64": dict(tfm=1, d_model=128, heads=2, ff=256, kernel=0, enc_layers=3, vocab=41, ic_a=1, ic_b=2, ic_cond=1, nframes=150),
    "noc": dict(tfm=0, d_model=64, heads=4, ff=128, kernel=15, enc_layers=3, vocab=50, ic_a=2, ic_b=0, ic_cond=0, nframes=120),
}
S2T = dict(cfg=dict(d_model=64, heads=4, ff=128, enc_layers=3, dec_layers=2, vocab=50, kernel=15, ic_a=1, ic_b=2, ic_cond=1),
           nsamples=16000, wave_id=17)
CTCONLY = dict(cfg=dict(d_model=64, heads=4, ff=128, enc_layers=3, dec_layers=0, vocab=50, kernel=15, ic_a=1, ic_b=2, ic_cond=1, no_decoder=1),
               nsamples=20000, wave_id=19)
CTCONLY_DECODES = [("ctc4", 4, 1.0, -5.0, 0.0, 0.0, False), ("ctc10", 10, 1.0, 0.0, 0.0, 0.0, False)]
S2T_SEED = 31


def encoder_conf(cfg):
    """Keyword arguments of the reference encoder class for an encoder case."""
    common = dict(output_size=cfg["d_model"], attention_heads=cfg["heads"], linear_units=cfg["ff"], num_blocks=cfg["enc_layers"],
                  dropout_rate=0.1, positional_dropout_rate=0.1, attention_dropout_rate=0.0, input_layer="conv2d", normalize_before=True,
                  use_flash_attn=False, **refbuild_interctc.interctc_conf(cfg))
    if cfg["tfm"]:
        return common
    return dict(common, macaron_style=True, rel_pos_type="latest", pos_enc_layer_type="rel_pos", selfattention_layer_type="rel_selfattn",
                activation_type="swish", use_cnn_module=True, cnn_module_kernel=cfg["kernel"])


def encoder_case(tag, cfg, seed):
    enc = (TransformerEncoder if cfg["tfm"] else ConformerEncoder)(80, **encoder_conf(cfg)).eval()
    ctc = CTC(odim=cfg["vocab"], encoder_output_size=cfg["d_model"]).eval()
    if cfg["ic_cond"]:
        enc.conditioning_layer = torch.nn.Linear(cfg["vocab"], cfg["d_model"])
    named = [("encoder." + k, p) for k, p in enc.named_parameters()] + [("ctc." + k, p) for k, p in ctc.named_parameters()]
    shapes = refbuild_ebf.seeded_state(named, seed)
    g = torch.Generator().manual_seed(300 + seed)
    z = {}
    with torch.no_grad():
        for m in enc.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.running_mean.copy_(0.1 * torch.randn(m.running_mean.shape, generator=g))
                m.running_var.copy_(0.5 + torch.rand(m.running_var.shape, generator=g))
        for k, v in enc.named_buffers():
            z[f"{tag}:w:encoder.{k}"] = v.numpy().copy()
        feats = torch.randn(1, cfg["nframes"], 80, generator=g).half().float()
        layers = []

        def first(o):   # conformer layers return ((x, pos_emb), mask), transformer layers (x, mask)
            x = o[0]
            return (x[0] if isinstance(x, tuple) else x)[0].clone()

        hooks = [lyr.register_forward_hook(lambda m, i, o: layers.append(first(o))) for lyr in enc.encoders]
        (out, inter), olens, _ = enc(feats, torch.tensor([cfg["nframes"]]), ctc=ctc)
        for h in hooks:
            h.remove()
    assert len(layers) == cfg["enc_layers"]
    idx = refbuild_interctc.interctc_conf(cfg)["interctc_layer_idx"]
    assert [li for li, _ in inter] == idx
    z.update({f"{tag}:cfg_keys": np.array(list(cfg.keys())), f"{tag}:cfg_vals": np.array(list(cfg.values()), dtype=np.int64),
              f"{tag}:idx": np.array(idx, dtype=np.int64), f"{tag}:feats": feats[0].half().numpy(), f"{tag}:out": out[0].numpy(),
              f"{tag}:olens": olens.numpy()})
    for i, t in enumerate(layers):
        z[f"{tag}:layer{i + 1}"] = t.numpy()
    for li, h in inter:
        z[f"{tag}:inter{li}"] = h[0].numpy()
    z.update(refbuild_ebf.shape_record(shapes, seed, prefix=f"{tag}:"))
    return z


def build_seeded(cfg, **kw):
    """The reference Speech2Text of cfg with every parameter replaced by refbuild_ebf.seeded_weights(S2T_SEED)."""
    s2t = refbuild.build_reference(cfg, seed=0, **kw)
    refbuild_ebf.seeded_state(s2t.asr_model.named_parameters(), S2T_SEED)
    return s2t


def s2t_case(name, spec, decodes):
    cfg = spec["cfg"]
    z = {"cfg_keys": np.array(list(cfg.keys())), "cfg_vals": np.array(list(cfg.values()), dtype=np.int64)}
    wave = refbuild.waveform(spec["wave_id"], spec["nsamples"])
    z["wave"] = wave.numpy()
    s2t = build_seeded(cfg, beam_size=4, ctc_weight=1.0 if cfg.get("no_decoder") else 0.3, maxlenratio=-8.0, nbest=10)
    model = s2t.asr_model
    assert model.encoder.conditioning_layer is not None
    for k, v in model.named_buffers():
        z["w:" + k] = v.numpy().copy()
    with torch.no_grad():
        (enc, inter), _ = model.encode(wave[None], torch.tensor([wave.numel()]))
        z["enc"] = enc[0].numpy()
        for li, h in inter:
            z[f"inter{li}"] = h[0].numpy()
        am = model.ctc.argmax(enc)[0]
        ids = torch.unique_consecutive(am)
        z["ctc_greedy"] = ids[ids != 0].numpy()
    for (dn, beam, cw, mlr, minr, pen, nl) in decodes:
        res, _ = build_seeded(cfg, beam_size=beam, ctc_weight=cw, maxlenratio=mlr, minlenratio=minr, penalty=pen, normalize_length=nl,
                              nbest=10)(wave)   # (n-best, intermediate CTC greedy tokens) (asr_inference.py:557-560)
        z[f"dec:{dn}:params"] = np.array([beam, cw, mlr, minr, pen, float(nl)], dtype=np.float64)
        z[f"dec:{dn}:n"] = np.array(len(res))
        for j, (_, _, _, hyp) in enumerate(res):
            z[f"dec:{dn}:{j}:yseq"] = hyp.yseq.numpy()
            z[f"dec:{dn}:{j}:score"] = np.array(float(hyp.score))
            z[f"dec:{dn}:{j}:scores"] = np.array([float(hyp.scores.get(k, np.nan)) for k in ("decoder", "ctc", "length_bonus")])
    z.update(refbuild_ebf.shape_record({k: tuple(p.shape) for k, p in model.named_parameters()}, S2T_SEED))
    path = os.path.join(HERE, f"{name}.npz")
    np.savez_compressed(path, **z)
    print(name, os.path.getsize(path) // 1024, "KiB; stored weights:", sorted(k for k in z if k.startswith("w:")))


if __name__ == "__main__":
    z = {}
    for i, (tag, cfg) in enumerate(ENC_CASES.items()):
        z.update(encoder_case(tag, cfg, i + 41))
    path = os.path.join(HERE, "interctc_enc.npz")
    np.savez_compressed(path, **z)
    print("interctc_enc.npz", os.path.getsize(path) // 1024, "KiB")
    refbuild_interctc.install()
    s2t_case("interctc_s2t", S2T, make_golden.DECODES)
    s2t_case("interctc_ctconly", CTCONLY, CTCONLY_DECODES)
