"""Generate the E-Branchformer fixtures from the UNMODIFIED reference (build container only).

    python tests/golden/make_golden_ebranchformer.py

ebranchformer_enc.npz: espnet2/asr/encoder/e_branchformer_encoder.py:EBranchformerEncoder on seeded features, two configurations
  A (prefix "A:"): recipe-like -- d 128, h 2 (d_k 64), cgmlp 256, macaron FFN 192, cgmlp / merge kernels 31 / 31, 3 blocks;
  B (prefix "B:"): the reference defaults -- d 64, h 4 (d_k 16), no FFN, cgmlp kernel 15, merge kernel 3, 2 blocks;
  each with feats, every block output (return_all_hs) and the output.
ebf.npz: the reference Speech2Text with the configuration-A encoder, 2 decoder layers, V 50 (same contents as make_golden.py's cases).
The weights are not stored: the reference modules are loaded with refbuild_ebf.seeded_weights, and the fixtures record the seed and the
name and shape of every parameter (the reference's state_dict surface, which the tests load strictly), so readers rebuild identical weights.
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

logging.disable(logging.WARNING)
refshim.install()
refbuild_ebf.install()
import make_golden  # noqa: E402
from espnet2.asr.encoder.e_branchformer_encoder import EBranchformerEncoder  # noqa: E402

ENC_CASES = {
    "A": dict(d_model=128, heads=2, cgmlp=256, cgmlp_kernel=31, merge_kernel=31, use_ffn=1, macaron=1, ff=192, enc_layers=3, nframes=403),
    "B": dict(d_model=64, heads=4, cgmlp=192, cgmlp_kernel=15, merge_kernel=3, use_ffn=0, macaron=0, ff=2048, enc_layers=2, nframes=141),
}
EBF = dict(cfg=dict(d_model=128, heads=2, ff=192, enc_layers=3, dec_layers=2, vocab=50, cgmlp=256, cgmlp_kernel=31, merge_kernel=31,
                    use_ffn=1, macaron=1), encoder="e_branchformer", nsamples=16000, wave_id=7)
EBF_SEED = 7


def encoder_case(tag, cfg, seed):
    enc = EBranchformerEncoder(80, **refbuild_ebf.encoder_conf(cfg)).eval()
    assert not list(enc.buffers())
    shapes = refbuild_ebf.seeded_state([("encoder." + k, p) for k, p in enc.named_parameters()], seed)
    g = torch.Generator().manual_seed(100 + seed)
    with torch.no_grad():
        feats = torch.randn(1, cfg["nframes"], 80, generator=g)
        out, olens, _ = enc(feats, torch.tensor([cfg["nframes"]]), return_all_hs=True)
    out, inter = out
    z = {f"{tag}:cfg_keys": np.array(list(cfg.keys())), f"{tag}:cfg_vals": np.array(list(cfg.values()), dtype=np.int64),
         f"{tag}:feats": feats[0].numpy(), f"{tag}:out": out[0].numpy(), f"{tag}:olens": olens.numpy()}
    for i, h in enumerate(inter):
        z[f"{tag}:layer{i + 1}"] = h[0].numpy()
    z.update(refbuild_ebf.shape_record(shapes, seed, prefix=f"{tag}:"))
    return z


def _build_seeded(cfg, seed=0, **kw):
    """refbuild.build_reference with every parameter of the model replaced by refbuild_ebf.seeded_weights(EBF_SEED)."""
    s2t = _build_reference(cfg, seed=seed, **kw)
    refbuild_ebf.seeded_state(s2t.asr_model.named_parameters(), EBF_SEED)
    return s2t


if __name__ == "__main__":
    z = {}
    for i, (tag, cfg) in enumerate(ENC_CASES.items()):
        z.update(encoder_case(tag, cfg, i + 1))
    np.savez_compressed(os.path.join(HERE, "ebranchformer_enc.npz"), **z)
    print("wrote ebranchformer_enc.npz", sorted(k for k in z if ":pshape:" not in k))
    _build_reference = refbuild.build_reference
    refbuild.build_reference = _build_seeded
    make_golden.run_case("ebf", EBF)
    # keep the non-parameter state (the mel matrix) and replace the stored parameters by their seed / shape record
    path = os.path.join(HERE, "ebf.npz")
    z = dict(np.load(path))
    s2t = _build_seeded(dict(EBF["cfg"], encoder=EBF["encoder"]))
    params = dict(s2t.asr_model.named_parameters())
    for k in params:
        assert np.array_equal(z.pop("w:" + k), params[k].detach().numpy()), k
    z.update(refbuild_ebf.shape_record({k: tuple(p.shape) for k, p in params.items()}, EBF_SEED))
    np.savez_compressed(path, **z)
    print("ebf.npz", os.path.getsize(path) // 1024, "KiB; stored weights:", sorted(k for k in z if k.startswith("w:")))
