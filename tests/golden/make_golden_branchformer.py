"""Generate the Branchformer fixtures from the UNMODIFIED reference (build container only).

    python tests/golden/make_golden_branchformer.py

branchformer_enc.npz: espnet2/asr/encoder/branchformer_encoder.py:BranchformerEncoder on seeded features, five configurations (prefix "A:" ..):
  A: concat, d 128, h 2 (d_k 64: fused attention), cgmlp 256, kernel 31, 3 blocks (the recipes' merge);
  B: learned_ave, d 64, h 4 (d_k 16: materialised attention), cgmlp 192, kernel 15, 2 blocks;
  C: fixed_ave with cgmlp_weight [0.0, 0.3, 1.0]: an attention-only, a two-branch and a cgMLP-only layer, each with merge_proj;
  D: use_attn=False (Identity merge_proj);
  E: use_cgmlp=False (Identity merge_proj), d_k 64;
  each with feats, every block output (forward hooks) and the output; per-layer cgmlp_weight under "{tag}:cgmlp_weight".
bf.npz: the reference Speech2Text with the configuration-A encoder, 2 decoder layers, V 50 (the five decode settings of make_golden.py).
The weights are not stored: the reference modules are loaded with refbuild_ebf.seeded_weights, and the fixtures record the seed and the
name and shape of every parameter, so readers rebuild identical weights.
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
import refbuild_bf  # noqa: E402

logging.disable(logging.WARNING)
refshim.install()
refbuild_bf.install()
import make_golden  # noqa: E402
from espnet2.asr.encoder.branchformer_encoder import BranchformerEncoder  # noqa: E402

ENC_CASES = {
    "A": (dict(d_model=128, heads=2, cgmlp=256, cgmlp_kernel=31, merge=0, use_attn=1, use_cgmlp=1, enc_layers=3, nframes=403), 0.5),
    "B": (dict(d_model=64, heads=4, cgmlp=192, cgmlp_kernel=15, merge=1, use_attn=1, use_cgmlp=1, enc_layers=2, nframes=141), 0.5),
    "C": (dict(d_model=64, heads=4, cgmlp=128, cgmlp_kernel=31, merge=2, use_attn=1, use_cgmlp=1, enc_layers=3, nframes=211), [0.0, 0.3, 1.0]),
    "D": (dict(d_model=64, heads=4, cgmlp=128, cgmlp_kernel=15, merge=0, use_attn=0, use_cgmlp=1, enc_layers=2, nframes=97), 0.5),
    "E": (dict(d_model=128, heads=2, cgmlp=256, cgmlp_kernel=31, merge=0, use_attn=1, use_cgmlp=0, enc_layers=2, nframes=187), 0.5),
}
BF = dict(cfg=dict(d_model=128, heads=2, ff=192, enc_layers=3, dec_layers=2, vocab=50, cgmlp=256, cgmlp_kernel=31, merge=0, use_attn=1,
                   use_cgmlp=1), encoder="branchformer", nsamples=16000, wave_id=9)
BF_SEED = 11


def encoder_case(tag, cfg, cw, seed):
    enc = BranchformerEncoder(80, **refbuild_bf.encoder_conf(cfg, cw)).eval()
    assert not list(enc.buffers())
    shapes = refbuild_bf.seeded_state([("encoder." + k, p) for k, p in enc.named_parameters()], seed)
    g = torch.Generator().manual_seed(100 + seed)
    layers = []
    hooks = [lyr.register_forward_hook(lambda m, i, o: layers.append(o[0][0][0].clone())) for lyr in enc.encoders]
    with torch.no_grad():
        feats = torch.randn(1, cfg["nframes"], 80, generator=g)
        out, olens, _ = enc(feats, torch.tensor([cfg["nframes"]]))
    for h in hooks:
        h.remove()
    L = cfg["enc_layers"]
    z = {f"{tag}:cfg_keys": np.array(list(cfg.keys())), f"{tag}:cfg_vals": np.array(list(cfg.values()), dtype=np.int64),
         f"{tag}:cgmlp_weight": np.array(cw if isinstance(cw, list) else [cw] * L, dtype=np.float64),
         f"{tag}:feats": feats[0].numpy(), f"{tag}:out": out[0].numpy(), f"{tag}:olens": olens.numpy()}
    assert len(layers) == L
    for i, h in enumerate(layers):
        z[f"{tag}:layer{i + 1}"] = h.numpy()
    z.update(refbuild_bf.shape_record(shapes, seed, prefix=f"{tag}:"))
    return z


def _build_seeded(cfg, seed=0, **kw):
    """refbuild.build_reference with every parameter of the model replaced by refbuild_ebf.seeded_weights(BF_SEED)."""
    s2t = _build_reference(cfg, seed=seed, **kw)
    refbuild_bf.seeded_state(s2t.asr_model.named_parameters(), BF_SEED)
    return s2t


if __name__ == "__main__":
    z = {}
    for i, (tag, (cfg, cw)) in enumerate(ENC_CASES.items()):
        z.update(encoder_case(tag, cfg, cw, i + 1))
    path = os.path.join(HERE, "branchformer_enc.npz")
    np.savez_compressed(path, **z)
    print("branchformer_enc.npz", os.path.getsize(path) // 1024, "KiB")
    _build_reference = refbuild.build_reference
    refbuild.build_reference = _build_seeded
    make_golden.run_case("bf", BF)
    # keep the non-parameter state (the mel matrix) and replace the stored parameters by their seed / shape record
    path = os.path.join(HERE, "bf.npz")
    z = dict(np.load(path))
    s2t = _build_seeded(dict(BF["cfg"], encoder=BF["encoder"]))
    params = dict(s2t.asr_model.named_parameters())
    for k in params:
        assert np.array_equal(z.pop("w:" + k), params[k].detach().numpy()), k
    z.update(refbuild_bf.shape_record({k: tuple(p.shape) for k, p in params.items()}, BF_SEED))
    np.savez_compressed(path, **z)
    print("bf.npz", os.path.getsize(path) // 1024, "KiB; stored weights:", sorted(k for k in z if k.startswith("w:")))
