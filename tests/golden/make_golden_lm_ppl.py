"""Generate tests/golden/lm_ppl.npz from the UNMODIFIED reference: ESPnetLanguageModel.nll / batchify_nll (espnet2/lm/espnet_model.py) and
espnet2/bin/lm_calc_perplexity.calc_perplexity on CPU, for three seeded LMs.  Build container only.

    python tests/golden/make_golden_lm_ppl.py

  tfm64:  TransformerLM, att_unit 64 / 1 head (d_k 64, the fused causal kernel), pos_enc null
  tfm32:  TransformerLM, att_unit 64 / 2 heads (d_k 32, the materialised path), pos_enc sinusoidal
  lstm:   SequentialRNNLM, 2 LSTM layers of 50 (not a multiple of 4: the padded GEMM operands)
One ragged batch of text lengths 1, 63, 64, 65, 130 (sentence 2 holds token id 0 at three places), its nll, and batchify_nll in chunks of
two (the max_length branch).  For calc_perplexity: a char token list, a small text set, and the files the reference writes for it with
batch_size 2, with log_base None and 10.
Every weight is rounded to a value float16 represents before the reference runs, and stored as float16: the fixture holds exactly the
weights the reference computed with, at half the size.
"""
import json
import os
import sys
import tempfile

import numpy as np
import torch
import yaml

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import refshim  # noqa: E402

refshim.install()
from espnet2.bin.lm_calc_perplexity import calc_perplexity  # noqa: E402
from espnet2.lm.espnet_model import ESPnetLanguageModel  # noqa: E402
from espnet2.lm.seq_rnn_lm import SequentialRNNLM  # noqa: E402
from espnet2.lm.transformer_lm import TransformerLM  # noqa: E402

LMS = {
    "tfm64": ("transformer", dict(pos_enc=None, embed_unit=16, att_unit=64, head=1, unit=64, layer=2)),
    "tfm32": ("transformer", dict(pos_enc="sinusoidal", embed_unit=16, att_unit=64, head=2, unit=64, layer=2)),
    "lstm": ("seq_rnn", dict(unit=50, nlayers=2, rnn_type="lstm")),
}
V = 40
LENGTHS = [1, 63, 64, 65, 130]
# char token list of the calc_perplexity set: <blank>=0, <unk>=1, then the characters, <sos/eos> last
CHARS = list("abcdefghijklmnopqrstuvwxyz") + ["<space>", "'"]
TOKEN_LIST = ["<blank>", "<unk>"] + CHARS + [f"x{i}" for i in range(V - 3 - len(CHARS))] + ["<sos/eos>"]
TEXTS = [("utt1", "hello world"), ("utt2", "a"), ("utt3", "it's a small test set"), ("utt4", "zebra?"), ("utt5", "q")]

g = torch.Generator().manual_seed(3)
text = torch.zeros(len(LENGTHS), max(LENGTHS), dtype=torch.long)
for b, n in enumerate(LENGTHS):
    text[b, :n] = torch.randint(1, V - 1, (n,), generator=g)
text[2, [5, 6, 40]] = 0                       # a real token id 0: masked as a key by TransformerLM._target_mask, still scored as a target
lengths = torch.tensor(LENGTHS)

out = {"lms": np.array(json.dumps(LMS)), "V": np.array(V), "text": text.numpy(), "lengths": lengths.numpy(),
       "token_list": np.array(json.dumps(TOKEN_LIST)), "texts": np.array(json.dumps(TEXTS))}
tmp = tempfile.mkdtemp(prefix="espref_lmppl_")
data = os.path.join(tmp, "text")
with open(data, "w", encoding="utf-8") as f:
    for k, t in TEXTS:
        f.write(f"{k} {t}\n")
for seed, (name, (kind, conf)) in enumerate(LMS.items()):
    torch.manual_seed(10 + seed)
    lm = TransformerLM(V, **conf) if kind == "transformer" else SequentialRNNLM(V, **conf)
    model = ESPnetLanguageModel(lm, V).eval()
    with torch.no_grad():
        for p in model.parameters():
            p.copy_(p.half().float())
    for k, v in model.state_dict().items():
        out[f"{name}:w:{k}"] = v.half().numpy()
    with torch.no_grad():
        nll, xl = model.nll(text, lengths)
        out[f"{name}:nll"] = nll.numpy()
        out[f"{name}:x_lengths"] = xl.numpy()
        nll2, _ = model.batchify_nll(text, lengths, batch_size=2)
        out[f"{name}:batchify_nll"] = nll2.numpy()
    cfg = os.path.join(tmp, f"{name}.yaml")
    mdl = os.path.join(tmp, f"{name}.pth")
    yaml.safe_dump(dict(token_list=TOKEN_LIST, token_type="char", bpemodel=None, lm=kind, lm_conf=conf, model_conf=dict(ignore_id=0),
                        use_preprocessor=True, cleaner=None, g2p=None, non_linguistic_symbols=None, init=None), open(cfg, "w"))
    torch.save(model.state_dict(), mdl)
    for tag, base in (("e", None), ("b10", 10.0)):
        od = os.path.join(tmp, f"out_{name}_{tag}")
        calc_perplexity(output_dir=od, batch_size=2, dtype="float32", ngpu=0, seed=0, num_workers=0, log_level="WARNING",
                        data_path_and_name_and_type=[(data, "text", "text")], key_file=None, train_config=cfg, model_file=mdl,
                        log_base=base, allow_variable_data_keys=False)
        for fn in ("utt2ppl", "utt2ntokens", "ppl", "base"):
            out[f"{name}:{tag}:{fn}"] = np.array(open(os.path.join(od, fn), encoding="utf-8").read())
    print(name, float(nll.sum()), open(os.path.join(tmp, f"out_{name}_e", "ppl")).read().strip())
path = os.path.join(HERE, "lm_ppl.npz")
np.savez_compressed(path, **out)
print("wrote", path, os.path.getsize(path) // 1024, "KiB")
