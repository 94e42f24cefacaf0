"""Oracle: the conv2d2 / conv2d6 / conv2d8 input layers (Conv2dSubsampling2/6/8) and the Conformer, Transformer and E-Branchformer
encoders behind them, one utterance at a time.  TEST INFRASTRUCTURE.

Reference: espnet2/legacy/nets/pytorch_backend/transformer/subsampling.py:31-48 (check_short_utt), 590-860 (Conv2dSubsampling2/6/8);
the encoder blocks are the ones of oracle/encoder.py, oracle/transformer_encoder.py and oracle/e_branchformer.py.  With input_layer
"conv2d" every function here computes what those modules compute.
Weights: flat dict with the reference's state_dict names.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from . import e_branchformer as EB
from . import encoder as E
from . import frontend as Fr
from . import transformer_encoder as TE
from .pipeline import OracleSpeech2Text

# input_layer -> (kernel, stride) of the convs after the first 3x3/stride-2 one, and check_short_utt's limit (subsampling.py:31-48)
SUBSAMPLING = {"conv2d": (((3, 2),), 7), "conv2d2": (((3, 1),), 7), "conv2d6": (((5, 3),), 11), "conv2d8": (((3, 2), (3, 2)), 15)}


def conv2d_subsampling(feats, w, input_layer, pfx="encoder.embed"):
    """Conv2dSubsampling{,2,6,8}.forward (subsampling.py:432-474, 625-649, 730-754, 838-862): a 3x3/stride-2 conv and the input layer's
    further convs, each + ReLU, flatten as feature index c*F'+f, Linear, then x*sqrt(d) (embedding.py:329)."""
    convs, limit = SUBSAMPLING[input_layer]
    if feats.shape[0] < limit:
        raise E.TooShortUttError(f"has {feats.shape[0]} frames and is too short for subsampling "
                                 f"(it needs more than {limit} frames), return empty results", feats.shape[0], limit)
    x = F.relu(F.conv2d(feats.unsqueeze(0).unsqueeze(0), w[pfx + ".conv.0.weight"], w[pfx + ".conv.0.bias"], stride=2))
    for i, (_, s) in enumerate(convs):
        x = F.relu(F.conv2d(x, w[pfx + f".conv.{2 * i + 2}.weight"], w[pfx + f".conv.{2 * i + 2}.bias"], stride=s))
    _, c, t, f = x.shape
    x = E._lin(x.transpose(1, 2).contiguous().view(t, c * f), w, pfx + ".out")
    return x * math.sqrt(x.shape[-1])


def encode(encoder, input_layer, feats, w, heads, num_blocks, return_layers=False):
    """ConformerEncoder / TransformerEncoder / EBranchformerEncoder.forward for one utterance with the given input layer.
    feats (T_f, 80) normalised log-mel -> (T, d); layers = [embed output, block 1, ...]."""
    x = conv2d_subsampling(feats, w, input_layer)
    T, d = x.shape
    if encoder == "transformer":
        x = x + TE.positional_encoding(T, d)
        layer = lambda x, pfx: TE.encoder_layer(x, w, pfx, heads)  # noqa: E731
    else:
        pos_emb = E.rel_positional_encoding(T, d)
        fn = E.encoder_layer if encoder == "conformer" else EB.ebranchformer_layer
        layer = lambda x, pfx: fn(x, pos_emb, w, pfx, heads)  # noqa: E731
    layers = [x]
    for i in range(num_blocks):
        x = layer(x, f"encoder.encoders.{i}")
        layers.append(x)
    x = E._ln(x, w, "encoder.after_norm")
    return (x, layers) if return_layers else x


class SubsamplingSpeech2Text(OracleSpeech2Text):
    """OracleSpeech2Text whose encoder takes cfg["input_layer"] (cfg["encoder"]: "conformer" (default), "transformer" or
    "e_branchformer")."""

    @torch.no_grad()
    def encode(self, speech):
        if isinstance(speech, np.ndarray):
            speech = torch.tensor(speech)
        feats = Fr.utterance_mvn(Fr.log_mel(Fr.stft_power(speech.float()), self.melmat))
        return encode(self.cfg.get("encoder", "conformer"), self.cfg["input_layer"], feats, self.w, self.cfg["heads"], self.cfg["enc_layers"])
