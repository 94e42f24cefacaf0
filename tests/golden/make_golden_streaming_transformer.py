"""Generate tests/golden/streaming_tfm_enc.npz and tests/golden/streaming_tfm_search.npz from the UNMODIFIED reference
ContextualBlockTransformerEncoder (espnet2/asr/encoder/contextual_block_transformer_encoder.py) and Speech2TextStreaming
(espnet2/bin/asr_inference_streaming.py) with that encoder.  Build container only.

    python tests/golden/make_golden_streaming_transformer.py

streaming_tfm_enc.npz, for each of the conv2d / conv2d6 / conv2d8 input layers (key prefix "<input_layer>:"): ``forward_infer`` on seeded
features pushed in uneven chunks (outputs of every push, and whether olens came back as None), one whole-utterance ``is_final`` call and a
segment shorter than a block.

streaming_tfm_search.npz: the n-best of every push of one waveform for joint CTC/attention decoding and for the AISHELL streaming decode
settings (egs2/aishell/asr1/conf/decode_asr_streaming.yaml: beam 10, ctc_weight 0.6, lm_weight 0.3, disable_repetition_detection) with an
LSTM ``seq_rnn`` LM, the LM type of that recipe's conf/train_lm.yaml; and for both settings the final n-best of the same waveform pushed in
chunks of the recipe's sim_chunk_length, 512 samples, as the reference's inference() pushes them (key prefix "sim512:").

Weights are not stored: every parameter is refbuild_ebf.seeded_weights of (seed, name, shape), and the fixtures record the seed and each
parameter's name and shape; non-parameter state (the mel matrix) is stored as it is.  Input features are stored as float16 and the reference
is run on the float16-rounded values, so nothing is lost."""
import json
import logging
import os
import sys
import tempfile

import numpy as np
import torch
import yaml

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import refbuild  # noqa: E402
import refbuild_ebf  # noqa: E402
import refshim  # noqa: E402

logging.disable(logging.WARNING)
refshim.install()
from espnet2.asr.encoder.contextual_block_transformer_encoder import ContextualBlockTransformerEncoder  # noqa: E402
from espnet2.bin.asr_inference_streaming import Speech2TextStreaming  # noqa: E402

# ---------------------------------------------------------------- encoder
CFG = dict(output_size=64, attention_heads=4, linear_units=96, num_blocks=2, block_size=40, hop_size=16, look_ahead=16)
LAYERS = ("conv2d", "conv2d6", "conv2d8")
PUSHES = [64, 64, 37, 100, 64, 150, 221, 200]
out = {"cfg_keys": np.array(list(CFG.keys())), "cfg_vals": np.array(list(CFG.values()), dtype=np.int64), "pushes": np.array(PUSHES)}
g = torch.Generator().manual_seed(11)
feats16 = torch.randn(1, sum(PUSHES), 80, generator=g).to(torch.float16)
out["feats"] = feats16[0].numpy()
feats = feats16.float()
for li, il in enumerate(LAYERS):
    enc = ContextualBlockTransformerEncoder(80, input_layer=il, normalize_before=True, **CFG).eval()
    shapes = refbuild_ebf.seeded_state(enc.named_parameters(), 100 + li)
    out.update(refbuild_ebf.shape_record(shapes, 100 + li, prefix=f"{il}:"))
    for k, v in enc.state_dict().items():
        if k not in shapes:
            out[f"{il}:w:{k}"] = v.numpy()
    with torch.no_grad():
        states, pos = None, 0
        for i, n in enumerate(PUSHES):
            y, ylen, states = enc(feats[:, pos:pos + n], torch.tensor([n]), states, is_final=(i == len(PUSHES) - 1), infer_mode=True)
            out[f"{il}:stream:{i}:y"] = y[0].numpy()
            out[f"{il}:stream:{i}:olens_none"] = np.array(ylen is None)
            pos += n
        y, ylen, _ = enc(feats[:, :700], torch.tensor([700]), None, is_final=True, infer_mode=True)
        out[f"{il}:whole:y"], out[f"{il}:whole:olens_none"] = y[0].numpy(), np.array(ylen is None)
        y, ylen, _ = enc(feats[:, :131], torch.tensor([131]), None, is_final=True, infer_mode=True)   # fewer frames than a block
        out[f"{il}:short:y"], out[f"{il}:short:olens_none"] = y.reshape(-1, y.shape[-1]).numpy(), np.array(ylen is None)
    print(il, {k: v.shape for k, v in out.items() if k.startswith(il) and ":y" in k})
path = os.path.join(HERE, "streaming_tfm_enc.npz")
np.savez_compressed(path, **out)
print("wrote", path, os.path.getsize(path) // 1024, "KiB")

# ---------------------------------------------------------------- Speech2TextStreaming
MCFG = dict(d_model=64, heads=4, ff=96, enc_layers=2, dec_layers=1, vocab=30)
y = refbuild.model_yaml(MCFG)
y.update(encoder="contextual_block_transformer", normalize=None, normalize_conf={},
         encoder_conf=dict(output_size=64, attention_heads=4, linear_units=96, num_blocks=2, block_size=40, hop_size=16, look_ahead=16,
                           input_layer="conv2d", normalize_before=True, init_average=True, ctx_pos_enc=True, dropout_rate=0.0,
                           positional_dropout_rate=0.0, attention_dropout_rate=0.0))
tmp = tempfile.mkdtemp(prefix="espref_stream_tfm_")
cfg_path, lm_path = os.path.join(tmp, "config.yaml"), os.path.join(tmp, "lm.yaml")
with open(cfg_path, "w") as f:
    yaml.safe_dump(y, f)
LM = dict(rnn_type="lstm", unit=64, nlayers=2)
with open(lm_path, "w") as f:
    yaml.safe_dump(dict(token_list=y["token_list"], lm="seq_rnn", lm_conf=LM, model_conf={}, init=None, use_preprocessor=False), f)
SETTINGS = {
    "joint": dict(beam_size=3, ctc_weight=0.3, nbest=2),
    "aishell": dict(beam_size=10, ctc_weight=0.6, lm_weight=0.3, penalty=0.0, maxlenratio=0.0, minlenratio=0.0,
                    disable_repetition_detection=True, nbest=3),
}
WAVE = (9, 52000)   # refbuild.waveform(*WAVE): rebuilt from its seed, not stored
wave = refbuild.waveform(*WAVE)
pushes = [8000, 640, 640, 9000, 12000, 3000, 18720]
assert sum(pushes) == wave.numel()
out = {"lm_conf": np.array(json.dumps(LM)), "yaml": np.array(json.dumps(y)), "wave": np.array(WAVE), "pushes": np.array(pushes),
       "settings": np.array(json.dumps(SETTINGS))}
for name, kw in SETTINGS.items():
    extra = dict(lm_train_config=lm_path, lm_file=None) if "lm_weight" in kw else {}
    s2t = Speech2TextStreaming(asr_train_config=cfg_path, asr_model_file=None, device="cpu", **kw, **extra)
    params = dict(s2t.asr_model.named_parameters())
    shapes = refbuild_ebf.seeded_state(params.items(), 7)
    if "wseed" not in out:
        out.update(refbuild_ebf.shape_record(shapes, 7))
        for k, v in s2t.asr_model.state_dict().items():
            if k not in params:
                out["w:" + k] = v.numpy()
    if extra:
        lm = s2t.beam_search.full_scorers["lm"]
        out.update(refbuild_ebf.shape_record(refbuild_ebf.seeded_state(lm.named_parameters(), 8), 8, prefix="lm:"))

    def record(key, res):
        out[f"{key}:n"] = np.array(len(res))
        for j, (_, _, token_int, hyp) in enumerate(res):
            out[f"{key}:{j}:yseq"] = np.array(hyp.yseq.tolist(), dtype=np.int64)
            out[f"{key}:{j}:token_int"] = np.array(token_int, dtype=np.int64)
            out[f"{key}:{j}:score"] = np.array(float(hyp.score), dtype=np.float64)
            for k, v in hyp.scores.items():
                out[f"{key}:{j}:score:{k}"] = np.array(float(v), dtype=np.float64)

    pos = 0
    for i, n in enumerate(pushes):
        with torch.no_grad():
            res = s2t(wave[pos:pos + n], is_final=(i == len(pushes) - 1))
        pos += n
        record(f"{name}:{i}", res)
    with torch.no_grad():   # espnet2/bin/asr_inference_streaming.py inference(): full chunks, then the remainder as the final push
        n_full = wave.numel() // 512
        for i in range(n_full):
            s2t(wave[i * 512:(i + 1) * 512], is_final=False)
        record(f"sim512:{name}", s2t(wave[n_full * 512:], is_final=True))
    last = len(pushes) - 1
    print(name, "pushes with output:", sum(int(out[f"{name}:{i}:n"]) > 0 for i in range(len(pushes))),
          "final:", [out[f"{name}:{last}:{j}:yseq"].tolist() for j in range(int(out[f"{name}:{last}:n"]))])
path = os.path.join(HERE, "streaming_tfm_search.npz")
np.savez_compressed(path, **out)
print("wrote", path, os.path.getsize(path) // 1024, "KiB")
