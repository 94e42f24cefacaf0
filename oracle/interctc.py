"""Oracle: intermediate CTC with self-conditioning in the Conformer and Transformer encoders (conv2d input layer), one utterance at a time,
in float64.  TEST INFRASTRUCTURE.

Reference: espnet2/asr/encoder/conformer_encoder.py:317-321,375-426 and transformer_encoder.py:210-214,268-299 (the encoder loop),
espnet2/asr/espnet_model.py:104-107 (conditioning_layer = Linear(vocab, d)), espnet2/asr/ctc.py:187-195 (CTC.softmax).  After block l
(1-based) when l is listed: h = after_norm(x) is the intermediate output and, with conditioning, x = x + conditioning_layer(softmax(ctc_lo(h))).
The blocks are the ones of oracle/encoder.py and oracle/transformer_encoder.py.
Weights: flat dict with the reference's state_dict names (encoder.*, ctc.ctc_lo.*).
"""
import torch

from . import encoder as E
from . import transformer_encoder as TE


def encode(feats, w, heads, num_blocks, layer_idx, use_conditioning, transformer=False):
    """feats (T_f, 80) -> (output (T, d), [(l, intermediate output (T, d)), ...], [block outputs before the conditioning]), all float64."""
    w = {k: (v.double() if v.is_floating_point() else v) for k, v in w.items()}
    x = E.conv2d_subsampling(feats.double(), w)
    T, d = x.shape
    if transformer:
        x = x + TE.positional_encoding(T, d).double()
    else:
        pos_emb = E.rel_positional_encoding(T, d).double()
    inter, blocks = [], []
    for i in range(num_blocks):
        pfx = f"encoder.encoders.{i}"
        x = TE.encoder_layer(x, w, pfx, heads) if transformer else E.encoder_layer(x, pos_emb, w, pfx, heads)
        blocks.append(x)
        if i + 1 in layer_idx:
            h = E._ln(x, w, "encoder.after_norm")
            inter.append((i + 1, h))
            if use_conditioning:
                x = x + E._lin(torch.softmax(E._lin(h, w, "ctc.ctc_lo"), dim=-1), w, "encoder.conditioning_layer")
    return E._ln(x, w, "encoder.after_norm"), inter, blocks
