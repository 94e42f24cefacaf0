"""Generate tests/golden/rnnlm.npz from the UNMODIFIED reference Speech2Text with a SequentialRNNLM (lm: seq_rnn, LSTM) scorer (LM shallow
fusion, espnet2/bin/asr_inference.py:178-191, espnet2/lm/seq_rnn_lm.py).  Build container only.

    python tests/golden/make_golden_rnnlm.py

Same tiny ASR model (and seed) as tiny_lm.npz: its weights are not stored again, only checked to be those of tiny_lm.npz.  Three LMs, their
weights stored as they are (small):
  A: unit 50, 2 layers (50 is not a multiple of 4: the padded GEMM operands)   -- decode settings joint_lm, att_lm, ctc_lm
  B: unit 36, nhid 44, 3 layers (nhid != unit)                                  -- joint_lm
  C: unit 48, tie_weights, 1 layer                                              -- joint_lm
For each LM also the reference's own batch_score log-probabilities on fixed prefixes, fed one token at a time from the zero state.
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
import refbuild  # noqa: E402
import refshim  # noqa: E402

logging.disable(logging.WARNING)
refshim.install()
from espnet2.bin.asr_inference import Speech2Text  # noqa: E402

CFG = dict(d_model=64, heads=4, ff=128, enc_layers=2, dec_layers=2, vocab=50, kernel=15)   # tiny_lm.npz's ASR model
LMS = {"A": dict(unit=50, nlayers=2), "B": dict(unit=36, nhid=44, nlayers=3), "C": dict(unit=48, nlayers=1, tie_weights=True)}
DECODES = {"A": [("joint_lm", 4, 0.3, 0.6, -8.0), ("att_lm", 3, 0.0, 0.4, -6.0), ("ctc_lm", 3, 1.0, 0.5, -5.0)],   # name, beam, ctc_weight,
           "B": [("joint_lm", 4, 0.3, 0.6, -8.0)], "C": [("joint_lm", 4, 0.3, 0.6, -8.0)]}                          # lm_weight, maxlenratio

tiny_lm = np.load(os.path.join(HERE, "tiny_lm.npz"))
tmp = tempfile.mkdtemp(prefix="espref_rnnlm_")
asr_yaml = os.path.join(tmp, "asr.yaml")
yaml.safe_dump(refbuild.model_yaml(CFG), open(asr_yaml, "w"))
wave = refbuild.waveform(0, 12000)
V, sos = CFG["vocab"], CFG["vocab"] - 1
g = torch.Generator().manual_seed(5)
prefixes = torch.cat([torch.full((4, 1), sos), torch.randint(2, V - 1, (4, 5), generator=g)], dim=1)   # 4 prefixes of sos + 5 tokens
out = {"cfg": np.array(json.dumps(CFG)), "lms": np.array(json.dumps(LMS)), "wave": wave.numpy(), "prefixes": prefixes.numpy()}
for lm_name, lm_conf in LMS.items():
    lm_yaml = os.path.join(tmp, f"lm_{lm_name}.yaml")
    yaml.safe_dump(dict(token_list=refbuild.token_list(V), lm="seq_rnn", lm_conf=dict(rnn_type="lstm", dropout_rate=0.2, **lm_conf), model_conf={},
                        init=None, use_preprocessor=False), open(lm_yaml, "w"))
    for j, (dn, beam, cw, lw, mlr) in enumerate(DECODES[lm_name]):
        torch.manual_seed(0)
        s2t = Speech2Text(asr_train_config=asr_yaml, asr_model_file=None, lm_train_config=lm_yaml, lm_file=None, device="cpu", dtype="float32",
                          beam_size=beam, ctc_weight=cw, lm_weight=lw, maxlenratio=mlr, nbest=10)
        for k, v in s2t.asr_model.state_dict().items():
            assert np.array_equal(v.numpy(), tiny_lm["w:" + k]), k
        lm = s2t.beam_search.full_scorers["lm"]
        assert type(lm).__name__ == "SequentialRNNLM" and isinstance(lm.rnn, torch.nn.LSTM)
        if j == 0:
            for k, v in lm.state_dict().items():
                out[f"{lm_name}:w:{k}"] = v.numpy()
            with torch.no_grad():
                states, steps = [None] * len(prefixes), []
                for t in range(prefixes.shape[1]):
                    logp, states = lm.batch_score(prefixes[:, :t + 1], states, None)
                    steps.append(logp.numpy())
            out[f"{lm_name}:prefix_logp"] = np.stack(steps)      # [len][n][V]: after feeding prefixes[:, :t+1]
        res = s2t(wave)
        key = f"{lm_name}:{dn}"
        out[f"{key}:params"] = np.array([beam, cw, lw, mlr], dtype=np.float64)
        out[f"{key}:n"] = np.array(len(res))
        for i, (_, _, ids, hyp) in enumerate(res):
            out[f"{key}:{i}:yseq"] = hyp.yseq.numpy()
            out[f"{key}:{i}:score"] = np.array(float(hyp.score))
            out[f"{key}:{i}:scores"] = np.array([float(hyp.scores.get(k, np.nan)) for k in ("decoder", "ctc", "lm")])
        print(key, len(res), res[0][3].yseq.tolist(), float(res[0][3].score))
path = os.path.join(HERE, "rnnlm.npz")
np.savez_compressed(path, **out)
print("wrote", path, os.path.getsize(path) // 1024, "KiB")
