"""Generate tests/golden/streaming_rnnlm.npz from the UNMODIFIED reference Speech2TextStreaming with a SequentialRNNLM (lm: seq_rnn, LSTM)
scorer: the n-best of every push for one joint CTC/attention + LM setting.  Build container only.

    python tests/golden/make_golden_streaming_rnnlm.py

Same streaming model, seed, waveform and pushes as streaming_search.npz, whose weights are not stored again (they are checked to be equal);
the LM has the shape of rnnlm.npz's LM A (unit 50, 2 layers) on this model's vocabulary, its weights stored as they are."""
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
from espnet2.bin.asr_inference_streaming import Speech2TextStreaming  # noqa: E402

base = np.load(os.path.join(HERE, "streaming_search.npz"))
y = json.loads(str(base["yaml"]))
tmp = tempfile.mkdtemp(prefix="espref_stream_rnnlm_")
cfg_path, lm_path = os.path.join(tmp, "config.yaml"), os.path.join(tmp, "lm.yaml")
with open(cfg_path, "w") as f:
    yaml.safe_dump(y, f)
LM = dict(rnn_type="lstm", unit=50, nlayers=2)
with open(lm_path, "w") as f:
    yaml.safe_dump(dict(token_list=y["token_list"], lm="seq_rnn", lm_conf=LM, model_conf={}, init=None, use_preprocessor=False), f)
SETTINGS = {"joint_rnnlm": dict(beam_size=3, ctc_weight=0.3, lm_weight=0.5, nbest=2)}
wave, pushes = torch.from_numpy(base["wave"]), base["pushes"].tolist()
out = {"lm_conf": np.array(json.dumps(LM)), "settings": np.array(json.dumps(SETTINGS))}
for name, kw in SETTINGS.items():
    torch.manual_seed(0)
    s2t = Speech2TextStreaming(asr_train_config=cfg_path, asr_model_file=None, lm_train_config=lm_path, lm_file=None, device="cpu", **kw)
    with torch.no_grad():
        for m in s2t.asr_model.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.running_mean.fill_(0.05)
                m.running_var.fill_(1.2)
    for k, v in s2t.asr_model.state_dict().items():
        assert np.array_equal(v.numpy(), base["w:" + k]), k
    for k, v in s2t.beam_search.full_scorers["lm"].state_dict().items():
        out["lm:" + k] = v.numpy()
    pos = 0
    for i, n in enumerate(pushes):
        res = s2t(wave[pos:pos + n], is_final=(i == len(pushes) - 1))
        pos += n
        out[f"{name}:{i}:n"] = np.array(len(res))
        for j, (_, _, token_int, hyp) in enumerate(res):
            out[f"{name}:{i}:{j}:yseq"] = np.array(hyp.yseq.tolist(), dtype=np.int64)
            out[f"{name}:{i}:{j}:token_int"] = np.array(token_int, dtype=np.int64)
            out[f"{name}:{i}:{j}:score"] = np.array(float(hyp.score), dtype=np.float64)
            for k, v in hyp.scores.items():
                out[f"{name}:{i}:{j}:score:{k}"] = np.array(float(v), dtype=np.float64)
    last = len(pushes) - 1
    print(name, "final:", [out[f"{name}:{last}:{j}:yseq"].tolist() for j in range(int(out[f"{name}:{last}:n"]))])
path = os.path.join(HERE, "streaming_rnnlm.npz")
np.savez_compressed(path, **out)
print("wrote", path, os.path.getsize(path) // 1024, "KiB")
