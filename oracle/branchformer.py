"""Oracle: BranchformerEncoder (conv2d input layer, rel_pos "latest", identity-gated cgMLP; concat, learned_ave and fixed_ave merging, and
layers with one branch), one utterance at a time.  TEST INFRASTRUCTURE.

Reference: espnet2/asr/encoder/branchformer_encoder.py:138-293 (block), 528-576 (forward), espnet2/asr/layers/cgmlp.py:57-124.
Weights: flat dict with the reference's state_dict names.  Which branches and merge parameters a layer has follows the weights; fixed_ave's
cgmlp_weight (a float or one per layer) is the only setting the weights do not carry.
"""
import numpy as np
import torch

from . import frontend as Fr
from .e_branchformer import cgmlp
from .encoder import _lin, _ln, conv2d_subsampling, rel_positional_encoding, rel_self_attention
from .pipeline import OracleSpeech2Text


def _pool_weight(x, w, pool, proj):
    """Attention pooling of one branch over its frames, then the Linear(D, 1) weight (branchformer_encoder.py:222-238)."""
    score = torch.softmax(_lin(x, w, pool).t() / x.shape[-1] ** 0.5, dim=-1)   # (1, T)
    return _lin((score @ x).squeeze(0), w, proj)                                 # (1,)


def branchformer_layer(x, pos_emb, w, pfx, heads, cgmlp_weight=0.5):
    """BranchformerEncoderLayer.forward (branchformer_encoder.py:138-293) in eval mode."""
    x1 = rel_self_attention(_ln(x, w, pfx + ".norm_mha"), pos_emb, w, pfx + ".attn", heads) if pfx + ".attn.linear_q.weight" in w else None
    x2 = cgmlp(_ln(x, w, pfx + ".norm_mlp"), w, pfx + ".cgmlp") if pfx + ".cgmlp.channel_proj1.0.weight" in w else None
    mp = pfx + ".merge_proj"
    if x1 is not None and x2 is not None:
        if pfx + ".pooling_proj1.weight" in w:                                       # learned_ave
            mw = torch.softmax(torch.cat([_pool_weight(x1, w, pfx + ".pooling_proj1", pfx + ".weight_proj1"),
                                          _pool_weight(x2, w, pfx + ".pooling_proj2", pfx + ".weight_proj2")]), dim=-1)
            y = mw[0] * x1 + mw[1] * x2
        elif w[mp + ".weight"].shape[1] == 2 * x.shape[-1]:                          # concat
            y = torch.cat([x1, x2], dim=-1)
        else:                                                                         # fixed_ave
            y = (1.0 - cgmlp_weight) * x1 + cgmlp_weight * x2
        x = x + _lin(y, w, mp)
    else:
        y = x1 if x1 is not None else x2
        x = x + (_lin(y, w, mp) if mp + ".weight" in w else y)                      # Identity merge_proj without a second branch
    return _ln(x, w, pfx + ".norm_final")


def branchformer_encode(feats, w, heads, num_blocks, cgmlp_weight=0.5, return_layers=False):
    """BranchformerEncoder.forward for one utterance.  feats (T_f, 80) normalised log-mel -> (T, d); layers = [embed, block 1, ...]."""
    cw = list(cgmlp_weight) if isinstance(cgmlp_weight, (list, tuple, np.ndarray)) else [cgmlp_weight] * num_blocks
    x = conv2d_subsampling(feats, w)
    pos_emb = rel_positional_encoding(x.shape[0], x.shape[1])
    layers = [x]
    for i in range(num_blocks):
        x = branchformer_layer(x, pos_emb, w, f"encoder.encoders.{i}", heads, float(cw[i]))
        layers.append(x)
    x = _ln(x, w, "encoder.after_norm")
    return (x, layers) if return_layers else x


class BranchformerSpeech2Text(OracleSpeech2Text):
    """OracleSpeech2Text with the Branchformer encoder (cfg: d_model, heads, enc_layers, dec_layers, vocab, ...)."""

    def __init__(self, cfg, weights, cgmlp_weight=0.5, **kw):
        super().__init__(cfg, weights, **kw)
        self.cgmlp_weight = cgmlp_weight

    @torch.no_grad()
    def encode(self, speech):
        if isinstance(speech, np.ndarray):
            speech = torch.tensor(speech)
        feats = Fr.utterance_mvn(Fr.log_mel(Fr.stft_power(speech.float()), self.melmat))
        return branchformer_encode(feats, self.w, self.cfg["heads"], self.cfg["enc_layers"], self.cgmlp_weight)
