"""Generate tests/golden/rnn.npz from the UNMODIFIED reference (build container only): the RNN model family.

    python tests/golden/make_golden_rnn.py

Encoder cases (one utterance per call, seeded features rounded to float16 and fed as float32), under the prefix "{case}:":
  vgg_blstmp  VGGRNNEncoder, bidirectional, use_projection                     (vgg_rnn_encoder.py, encoders.py VGG2L + RNNP)
  vgg_blstm   VGGRNNEncoder, bidirectional, use_projection false               (VGG2L + RNN: one stacked LSTM, then l_last + tanh)
  vgg_lstmp   VGGRNNEncoder, unidirectional, use_projection
  rnn_sub     RNNEncoder, bidirectional, use_projection, subsample 2_2_1_1    (rnn_encoder.py)
each with feats, the VGG2L output ("vgg", VGG encoders), every projection output after its tanh ("layer0".., RNNP), the output and olens.
Frame counts are odd after each pool.

Speech2Text cases: a small VGG-BLSTMP encoder + 2-layer RNN decoder (AttLoc) model, V 50, decoded by the reference's own Speech2Text (its
non-batch BeamSearch: RNNDecoder is not a BatchScorerInterface) under "{dn}:": ctc_weight 0.3 / 0.5 / 1.0, the context_residual variant
("ctxres" model), LM shallow fusion with an LSTM LM ("lm", LM weights "lm:") and a Transformer LM ("tlm", LM weights "tlm:"), and the
waveform rounded to 16-bit PCM ("cli": what bin_asr_inference reads from a wav file).

Weights are not stored: parameters come from refbuild_ebf.seeded_weights ("{prefix}wseed" and "{prefix}pshape:{name}"), the non-parameter
state (the frontend's buffers) is stored as "{prefix}w:{name}".
"""
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
import refshim  # noqa: E402
import refbuild  # noqa: E402
import refbuild_ebf  # noqa: E402

logging.disable(logging.WARNING)
refshim.install()
from espnet2.asr.encoder.rnn_encoder import RNNEncoder  # noqa: E402
from espnet2.asr.encoder.vgg_rnn_encoder import VGGRNNEncoder  # noqa: E402
from espnet2.bin.asr_inference import Speech2Text  # noqa: E402

ENC_CASES = {
    "vgg_blstmp": dict(cls="vgg_rnn", conf=dict(rnn_type="lstm", bidirectional=True, use_projection=True, num_layers=3, hidden_size=50,
                                                 output_size=36), nframes=41, seed=1),
    "vgg_blstm": dict(cls="vgg_rnn", conf=dict(rnn_type="lstm", bidirectional=True, use_projection=False, num_layers=2, hidden_size=40,
                                                output_size=44), nframes=73, seed=2),
    "vgg_lstmp": dict(cls="vgg_rnn", conf=dict(rnn_type="lstm", bidirectional=False, use_projection=True, num_layers=2, hidden_size=48,
                                                output_size=32), nframes=41, seed=3),
    "rnn_sub": dict(cls="rnn", conf=dict(rnn_type="lstm", bidirectional=True, use_projection=True, num_layers=4, hidden_size=36,
                                          output_size=28, subsample=[2, 2, 1, 1]), nframes=59, seed=4),
}
V = 50
DEC_CONF = dict(rnn_type="lstm", num_layers=2, hidden_size=40, dropout=0.0, att_conf=dict(atype="location", adim=32, aconv_chans=4,
                                                                                          aconv_filts=6))
ENC_CONF = dict(rnn_type="lstm", bidirectional=True, use_projection=True, num_layers=2, hidden_size=48, output_size=40)
LM_CONFS = {"lm": ("seq_rnn", dict(unit=36, nlayers=2, rnn_type="lstm", dropout_rate=0.0)),
            "tlm": ("transformer", dict(pos_enc=None, embed_unit=16, att_unit=32, head=2, unit=48, layer=2))}
# name -> (model, beam, ctc_weight, LM (a LM_CONFS key or None), maxlenratio)
DECODES = {"ctc03": ("base", 4, 0.3, None, 0.0), "ctc05": ("base", 4, 0.5, None, 0.0), "ctc10": ("base", 3, 1.0, None, 0.0),
           "ctxres": ("ctxres", 4, 0.5, None, 0.0), "lm": ("base", 4, 0.5, "lm", 0.0), "tlm": ("base", 4, 0.3, "tlm", 0.0),
           "cli": ("base", 4, 0.5, None, 0.0)}
S2T_SEED, LM_SEED = 21, 22
ENC_CLASSES = {"vgg_rnn": VGGRNNEncoder, "rnn": RNNEncoder}


def model_yaml(context_residual):
    y = refbuild.model_yaml(dict(d_model=40, heads=2, ff=64, enc_layers=1, dec_layers=1, vocab=V))
    y["encoder"], y["encoder_conf"] = "vgg_rnn", dict(ENC_CONF)
    y["decoder"], y["decoder_conf"] = "rnn", dict(DEC_CONF, context_residual=context_residual)
    y["model_conf"] = dict(ctc_weight=0.5, lsm_weight=0.1, length_normalized_loss=False)
    return y


def lm_yaml(name):
    kind, conf = LM_CONFS[name]
    return dict(token_list=refbuild.token_list(V), lm=kind, lm_conf=dict(conf), model_conf={}, init=None, use_preprocessor=False)


def encoder_case(name, c):
    tag = f"{name}:"
    enc = ENC_CLASSES[c["cls"]](80, **c["conf"]).eval()
    shapes = refbuild_ebf.seeded_state([("encoder." + k, p) for k, p in enc.named_parameters()], c["seed"])
    g = torch.Generator().manual_seed(300 + c["seed"])
    feats = torch.randn(1, c["nframes"], 80, generator=g).to(torch.float16).to(torch.float32)
    trace = []
    rnn = enc.enc[-1]
    hooks = []
    if hasattr(rnn, "elayers"):     # RNNP: projection outputs (tanh applied below for all but the last)
        for i in range(rnn.elayers):
            hooks.append(getattr(rnn, f"bt{i}").register_forward_hook(lambda m, inp, out: trace.append(out.detach().clone())))
    if c["cls"] == "vgg_rnn":
        hooks.append(enc.enc[0].register_forward_hook(lambda m, inp, out: out and trace.insert(0, out[0].detach().clone())))
    with torch.no_grad():
        out, olens, _ = enc(feats, torch.tensor([c["nframes"]]))
    for h in hooks:
        h.remove()
    z = {tag + "conf": np.array(json.dumps(dict(cls=c["cls"], **c["conf"]))), tag + "feats": feats.numpy().astype(np.float16),
         tag + "out": out.numpy(), tag + "olens": np.asarray(olens, dtype=np.int64)}
    k = 0
    if c["cls"] == "vgg_rnn":
        z[tag + "vgg"] = trace[0].numpy()
        k = 1
    projs = trace[k:]
    for i, p in enumerate(projs):
        z[f"{tag}layer{i}"] = (torch.tanh(p) if i + 1 < len(projs) else p).view(1, -1, p.shape[-1]).numpy()
    z.update(refbuild_ebf.shape_record(shapes, c["seed"], prefix=tag))
    print(name, out.shape, [v.shape for v in projs])
    return z


def s2t_cases():
    tmp = tempfile.mkdtemp(prefix="espref_rnn_")
    out = {}
    wave = refbuild.waveform(7, 12000)
    out["s2t:wave"] = wave.numpy()
    pcm = (wave.clamp(-1, 1) * 32767).round().to(torch.int16)
    out["cli:pcm"] = pcm.numpy()
    done = set()
    for dn, (model, beam, cw, use_lm, mlr) in DECODES.items():
        path = os.path.join(tmp, f"{model}.yaml")
        yaml.safe_dump(model_yaml(model == "ctxres"), open(path, "w"))
        kw = {}
        if use_lm:
            lm_path = os.path.join(tmp, f"{use_lm}.yaml")
            yaml.safe_dump(lm_yaml(use_lm), open(lm_path, "w"))
            kw = dict(lm_train_config=lm_path, lm_file=None, lm_weight=0.5)
        torch.manual_seed(0)
        s2t = Speech2Text(asr_train_config=path, asr_model_file=None, device="cpu", dtype="float32", beam_size=beam, ctc_weight=cw,
                          maxlenratio=mlr, nbest=10, **kw)
        assert cw == 1.0 or type(s2t.beam_search).__name__ == "BeamSearch", type(s2t.beam_search)
        m = s2t.asr_model
        shapes = refbuild_ebf.seeded_state(list(m.named_parameters()), S2T_SEED)
        if model not in done:
            out[f"{model}:cfg"] = np.array(json.dumps(model_yaml(model == "ctxres")))
            out.update(refbuild_ebf.shape_record(shapes, S2T_SEED, prefix=f"{model}:"))
            pnames = set(shapes)
            for k, v in m.state_dict().items():
                if k not in pnames:
                    out[f"{model}:w:{k}"] = v.numpy()
            done.add(model)
        if use_lm:
            lm = s2t.beam_search.full_scorers["lm"]
            assert type(lm).__name__ == {"lm": "SequentialRNNLM", "tlm": "TransformerLM"}[use_lm]
            lshapes = refbuild_ebf.seeded_state(list(lm.named_parameters()), LM_SEED)
            out[f"{use_lm}:cfg"] = np.array(json.dumps(lm_yaml(use_lm)))
            out.update(refbuild_ebf.shape_record(lshapes, LM_SEED, prefix=f"{use_lm}:"))
        with torch.no_grad():
            res = s2t(pcm.to(torch.float32) / 32768.0 if dn == "cli" else wave)
        out[f"{dn}:params"] = np.array([beam, cw, 0.5 if use_lm else 0.0, mlr], dtype=np.float64)
        out[f"{dn}:lm"] = np.array(use_lm or "")
        out[f"{dn}:model"] = np.array(model)
        out[f"{dn}:n"] = np.array(len(res))
        for i, (_, _, ids, hyp) in enumerate(res):
            out[f"{dn}:{i}:yseq"] = hyp.yseq.numpy()
            out[f"{dn}:{i}:score"] = np.array(float(hyp.score))
        print(dn, len(res), res[0][3].yseq.tolist(), float(res[0][3].score))
    return out


if __name__ == "__main__":
    z = {}
    for name, c in ENC_CASES.items():
        z.update(encoder_case(name, c))
    z.update(s2t_cases())
    path = os.path.join(HERE, "rnn.npz")
    np.savez_compressed(path, **z)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")
