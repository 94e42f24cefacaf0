"""Oracle: EBranchformerEncoder (conv2d input layer, rel_pos "latest", identity-gated cgMLP, optional / macaron FFN), one utterance at a
time.  TEST INFRASTRUCTURE.

Reference: espnet2/asr/encoder/e_branchformer_encoder.py:110-183 (block), 453-563 (forward), espnet2/asr/layers/cgmlp.py:57-124 (cgMLP,
CSGU with gate_activation "identity", no linear after the conv), layer_norm.py (eps 1e-12), nets_utils.py:571-584 (FFN activations).
Weights: flat dict with the reference's state_dict names.
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import frontend as Fr
from .encoder import _lin, _ln, conv2d_subsampling, rel_positional_encoding, rel_self_attention
from .pipeline import OracleSpeech2Text


def _dwconv(x, w, b):
    """Depthwise Conv1d over time with 'same' zero padding: x (T, C), w (C, 1, K)."""
    return F.conv1d(x.t().unsqueeze(0), w, b, padding=(w.shape[-1] - 1) // 2, groups=w.shape[0]).squeeze(0).t()


def cgmlp(x, w, pfx):
    """ConvolutionalGatingMLP.forward (cgmlp.py:110-124): channel_proj1 (Linear + exact GELU) -> CSGU -> channel_proj2."""
    h = F.gelu(_lin(x, w, pfx + ".channel_proj1.0"))
    x_r, x_g = h.chunk(2, dim=-1)
    x_g = _ln(x_g, w, pfx + ".csgu.norm")
    x_g = _dwconv(x_g, w[pfx + ".csgu.conv.weight"], w[pfx + ".csgu.conv.bias"])
    return _lin(x_r * x_g, w, pfx + ".channel_proj2")


def _ffn(x, w, pfx, act):
    h = _lin(x, w, pfx + ".w_1")
    h = h * torch.sigmoid(h) if act == "swish" else torch.relu(h)
    return _lin(h, w, pfx + ".w_2")


def ebranchformer_layer(x, pos_emb, w, pfx, heads, ffn_act="swish"):
    """EBranchformerEncoderLayer.forward (e_branchformer_encoder.py:110-183); which FFNs exist follows the weights."""
    macaron = pfx + ".feed_forward_macaron.w_1.weight" in w
    ff_scale = 0.5 if macaron else 1.0
    if macaron:
        x = x + ff_scale * _ffn(_ln(x, w, pfx + ".norm_ff_macaron"), w, pfx + ".feed_forward_macaron", ffn_act)
    x_att = rel_self_attention(_ln(x, w, pfx + ".norm_mha"), pos_emb, w, pfx + ".attn", heads)
    x_mlp = cgmlp(_ln(x, w, pfx + ".norm_mlp"), w, pfx + ".cgmlp")
    cat = torch.cat([x_att, x_mlp], dim=-1)
    cat = cat + _dwconv(cat, w[pfx + ".depthwise_conv_fusion.weight"], w[pfx + ".depthwise_conv_fusion.bias"])
    x = x + _lin(cat, w, pfx + ".merge_proj")
    if pfx + ".feed_forward.w_1.weight" in w:
        x = x + ff_scale * _ffn(_ln(x, w, pfx + ".norm_ff"), w, pfx + ".feed_forward", ffn_act)
    return _ln(x, w, pfx + ".norm_final")


def ebranchformer_encode(feats, w, heads, num_blocks, ffn_act="swish", return_layers=False):
    """EBranchformerEncoder.forward for one utterance.  feats (T_f, 80) normalised log-mel -> (T, d); layers = [embed, block 1, ...]."""
    x = conv2d_subsampling(feats, w)
    pos_emb = rel_positional_encoding(x.shape[0], x.shape[1])
    layers = [x]
    for i in range(num_blocks):
        x = ebranchformer_layer(x, pos_emb, w, f"encoder.encoders.{i}", heads, ffn_act)
        layers.append(x)
    x = _ln(x, w, "encoder.after_norm")
    return (x, layers) if return_layers else x


class EBranchformerSpeech2Text(OracleSpeech2Text):
    """OracleSpeech2Text with the E-Branchformer encoder (cfg: d_model, heads, enc_layers, dec_layers, vocab, ...)."""

    @torch.no_grad()
    def encode(self, speech):
        if isinstance(speech, np.ndarray):
            speech = torch.tensor(speech)
        feats = Fr.utterance_mvn(Fr.log_mel(Fr.stft_power(speech.float()), self.melmat))
        return ebranchformer_encode(feats, self.w, self.cfg["heads"], self.cfg["enc_layers"])
