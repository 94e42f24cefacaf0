"""LM perplexity (espnet_b200.ESPnetLanguageModel.nll / batchify_nll, espnet_b200.lm_calc_perplexity) on the host: loading reference
checkpoints, the sos / eos / padding logic of nll and the full-sequence forwards with the C-ABI entry points emulated (tests/emu_lm_ppl.py),
the files calc_perplexity writes, and the refusals.  Against tests/golden/lm_ppl.npz (make_golden_lm_ppl.py, the UNMODIFIED reference)."""
import ctypes
import json
import math
import os

import numpy as np
import pytest
import torch
import yaml

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LMS = ("tfm64", "tfm32", "lstm")


def _z():
    return np.load(os.path.join(GOLDEN, "lm_ppl.npz"))


def _weights(z, name):
    p = f"{name}:w:"
    return {k[len(p):]: torch.from_numpy(z[k]).float() for k in z.files if k.startswith(p)}   # stored as float16, exactly


def write_lm(z, name, root):
    """The LM's config.yaml and checkpoint as the reference's LM training writes them -> (config path, model path)."""
    kind, conf = json.loads(str(z["lms"]))[name]
    cfg, mdl = os.path.join(root, f"{name}.yaml"), os.path.join(root, f"{name}.pth")
    yaml.safe_dump(dict(token_list=json.loads(str(z["token_list"])), token_type="char", bpemodel=None, lm=kind, lm_conf=conf,
                        model_conf=dict(ignore_id=0), use_preprocessor=True, cleaner=None, g2p=None, non_linguistic_symbols=None, init=None),
                   open(cfg, "w"))
    torch.save(_weights(z, name), mdl)
    return cfg, mdl


def write_text(z, root):
    path = os.path.join(root, "text")
    with open(path, "w", encoding="utf-8") as f:
        for k, t in json.loads(str(z["texts"])):
            f.write(f"{k} {t}\n")
    return path


def check_ppl_files(z, name, tag, out_dir):
    """utt2ntokens and base as the reference wrote them, utt2ppl and ppl within rtol 1e-4, the same keys in the same order."""
    rd = lambda fn: open(os.path.join(out_dir, fn), encoding="utf-8").read()  # noqa: E731
    assert rd("utt2ntokens") == str(z[f"{name}:{tag}:utt2ntokens"])
    assert rd("base") == str(z[f"{name}:{tag}:base"])
    got = [ln.split() for ln in rd("utt2ppl").splitlines()]
    want = [ln.split() for ln in str(z[f"{name}:{tag}:utt2ppl"]).splitlines()]
    assert [g[0] for g in got] == [w[0] for w in want]
    np.testing.assert_allclose([float(g[1]) for g in got], [float(w[1]) for w in want], rtol=1e-4)
    np.testing.assert_allclose(float(rd("ppl")), float(str(z[f"{name}:{tag}:ppl"])), rtol=1e-4)


@pytest.mark.parametrize("name", LMS)
def test_reference_checkpoint_loads_strictly(name, tmp_path):
    import espnet_b200

    z = _z()
    cfg, mdl = write_lm(z, name, str(tmp_path))
    model, args = espnet_b200.build_espnet_lm_from_file(cfg, mdl, device="cpu")
    assert isinstance(model, espnet_b200.ESPnetLanguageModel)
    assert sorted(model.state_dict()) == sorted(_weights(z, name))
    model.load_state_dict(_weights(z, name), strict=True)
    assert model.sos == model.eos == int(z["V"]) - 1 and model.ignore_id == 0


@pytest.mark.parametrize("name", LMS)
def test_nll_host_logic_emulated(name, monkeypatch, tmp_path):
    """nll (sos / eos, padding, positions past text_lengths + 1 zeroed, a real token 0 masked as a key and scored as a target) and
    batchify_nll's max_length branch through the emulated kernels, against the reference's own values."""
    import emu_lm_ppl

    import espnet_b200

    emu_lm_ppl.install(monkeypatch)
    z = _z()
    model, _ = espnet_b200.build_espnet_lm_from_file(*write_lm(z, name, str(tmp_path)), device="cpu")
    text, lengths = torch.from_numpy(z["text"]), torch.from_numpy(z["lengths"])
    nll, xl = model.nll(text, lengths)
    assert nll.shape == z[f"{name}:nll"].shape and torch.equal(xl, torch.from_numpy(z[f"{name}:x_lengths"]))
    np.testing.assert_allclose(nll.numpy(), z[f"{name}:nll"], atol=1e-4, rtol=0)
    nll2, xl2 = model.batchify_nll(text, lengths, batch_size=2)
    np.testing.assert_allclose(nll2.numpy(), z[f"{name}:batchify_nll"], atol=1e-4, rtol=0)
    assert torch.equal(xl2, xl)
    logits, hidden = model.lm(text[:2, :8], None)
    assert hidden is None and logits.shape == (2, 8, int(z["V"]))


@pytest.mark.parametrize("log_base", [None, 10.0])
def test_calc_perplexity_files_emulated(log_base, monkeypatch, tmp_path):
    """The files and their format (utt2ppl, utt2ntokens, ppl, base) as the reference writes them, with log_base e and 10."""
    import emu_lm_ppl

    import espnet_b200.lm_calc_perplexity as lcp

    emu_lm_ppl.install(monkeypatch)
    build = lcp.build_espnet_lm_from_file
    monkeypatch.setattr(lcp, "build_espnet_lm_from_file", lambda c, m, device: build(c, m, device="cpu"))
    z = _z()
    cfg, mdl = write_lm(z, "lstm", str(tmp_path))
    out = str(tmp_path / "out")
    lcp.calc_perplexity(output_dir=out, batch_size=2, dtype="float32", ngpu=1, seed=0, num_workers=1, log_level="WARNING",
                        data_path_and_name_and_type=[(write_text(z, str(tmp_path)), "text", "text")], key_file=None, train_config=cfg,
                        model_file=mdl, log_base=log_base, allow_variable_data_keys=False)
    check_ppl_files(z, "lstm", "e" if log_base is None else "b10", out)


def test_refusals(tmp_path):
    import espnet_b200.lm_calc_perplexity as lcp
    from espnet_b200.bin_lm_calc_perplexity import get_parser

    z = _z()
    cfg, mdl = write_lm(z, "lstm", str(tmp_path))
    kw = dict(output_dir=str(tmp_path / "o"), batch_size=1, ngpu=1, seed=0, num_workers=1, log_level="WARNING",
              data_path_and_name_and_type=[(write_text(z, str(tmp_path)), "text", "text")], key_file=None, train_config=cfg, model_file=mdl,
              log_base=None, allow_variable_data_keys=False)
    for dtype in ("float16", "float64"):
        with pytest.raises(NotImplementedError):
            lcp.calc_perplexity(dtype=dtype, **kw)
    with pytest.raises(SystemExit):
        get_parser().parse_args(["--output_dir", "o", "--data_path_and_name_and_type", "t,text,text", "--dtype", "float16"])
    for token_type in ("phn", "hugging_face"):
        args = yaml.safe_load(open(cfg))
        with pytest.raises(NotImplementedError):
            lcp.text_to_ids(type("A", (), dict(args, token_type=token_type))())
    with pytest.raises(NotImplementedError):
        lcp.text_to_ids(type("A", (), dict(yaml.safe_load(open(cfg)), non_linguistic_symbols="nlsyms.txt"))())
    (tmp_path / "bad").write_text("utt1 hello\nutt2\n")
    with pytest.raises(RuntimeError):
        list(lcp.read_text(str(tmp_path / "bad")))
    a = get_parser().parse_args(["--output_dir", "o", "--data_path_and_name_and_type", "t,text,text", "--log_base", "none"])
    assert a.log_base is None and a.data_path_and_name_and_type == [("t", "text", "text")] and a.batch_size == 1


def test_tokenizers_text2tokens():
    from espnet_b200.text import build_tokenizer

    assert build_tokenizer("char").text2tokens("it's a") == ["i", "t", "'", "s", "<space>", "a"]
    assert build_tokenizer("word").text2tokens("hello  world") == ["hello", "world"]


def test_capi_entry_points_bound():
    from espnet_b200 import lib

    for name, n in (("espb_causal_flash_attn_f32", 21), ("espb_causal_softmax_f32", 11), ("espb_nll_rows_f32", 7)):
        assert len(lib._SIGS[name]) == n and name in lib.EXPORTED_SYMBOLS
    if os.path.exists(lib.LIB_PATH):
        handle = ctypes.CDLL(lib.LIB_PATH)
        for name in ("espb_causal_flash_attn_f32", "espb_causal_softmax_f32", "espb_nll_rows_f32"):
            assert hasattr(handle, name)


# ------------------------------------------------------------------------------------------------ float64 references of the kernels
# The values the kernels read in, the result and a per-element bound of the kernel's fp32 arithmetic out (u = 2^-24; expf within 2 ulp
# <= 4u, logf 1 ulp; a value stored split as hi + lo is within 16u).  tests/test_gpu_lm_ppl.py asserts err <= bound;
# test_tolerances_catch_plausible_bugs below shows each bound is tight enough to see the bugs named there.  Peaked scores give key weights
# below fp32's smallest normal 2^-126 (__expf flushes them to 0): the bounds add 2^-126 absolute per weight.
U32 = 2.0 ** -24
TINY = 2.0 ** -126


def _over(diff, tol):
    return (diff / tol.clamp_min(1e-300)).max().item()


def _valid_keys(tok, n, T, diag=0, mask_tok=True, device=None):
    i, j = torch.arange(T, device=device).view(T, 1), torch.arange(T, device=device).view(1, T)
    ok = (j <= i + diag) & (j < n)
    return ok & (tok != 0).view(1, T) if mask_tok else ok


def causal_attn_ref(q, k, v, tok, lens, scale=0.125, diag=0, mask_tok=True):
    """Causal token-masked attention (espb_causal_flash_attn_f32) of q / k / v [B][H][T][64] float64, tok [B][T], lens -> (o, tol), rows
    without a valid key 0.  diag / mask_tok / scale restate bugs: keys up to i + diag admitted, token-0 keys not masked, another scale.
    The bound is the one derived for the fused kernel in tests/test_gpu_attention.py (3xTF32 scores within 67u sum_c |q_c k_c|, a key
    weight off relatively by rho = e_s scale + 4u (m - s scale) + (4 nkt + 20) u, P V in 3xTF32, the row sum and 1 / l) with the counts of
    the causal kernel: a row i of the 128-row block starting at I0 runs nkt = ceil(min(len, I0 + 128) / 64) key tiles, and each thread sums
    a quarter of those keys."""
    B, H, T, _ = q.shape
    o, tol = torch.zeros_like(q), torch.zeros_like(q)
    i0 = torch.arange(T, device=q.device) // 128 * 128
    for b, n in enumerate(lens):
        n = min(int(n), T)
        if n <= 0:
            continue
        ok = _valid_keys(tok[b].to(q.device), n, T, diag, mask_tok, q.device)
        nk = (i0 + 128).clamp(max=n).double().view(T, 1)
        nkt = torch.ceil(nk / 64)
        s = q[b] @ k[b].transpose(-1, -2)
        es = 67 * U32 * (q[b].abs() @ k[b].abs().transpose(-1, -2))
        z = torch.where(ok, s * scale, torch.full((), -math.inf, dtype=q.dtype, device=q.device))
        m = z.max(-1, keepdim=True).values
        has = torch.isfinite(m)
        p = torch.where(ok, torch.exp(z - torch.where(has, m, torch.zeros_like(m))), torch.zeros((), dtype=q.dtype, device=q.device))
        p = p / p.sum(-1, keepdim=True).clamp_min(1e-300)
        ob = p @ v[b]
        rho = torch.where(ok, es * scale + 4 * U32 * (torch.where(has, m, torch.zeros_like(m)) - z).abs(), torch.zeros_like(z)) \
            + (4 * nkt + 20) * U32
        pr = p * rho
        va = v[b].abs()
        tol[b] = pr @ va + pr.sum(-1, keepdim=True) * ob.abs() + (66 + nkt) * U32 * (p @ va) + (nk / 4 + nkt + 20) * U32 * ob.abs() \
            + TINY * (1 + va.sum(-2, keepdim=True))
        o[b] = ob
    return o, tol


def causal_softmax_ref(sc, tok, lens, sqrt_dk, Tp):
    """espb_causal_softmax_f32 of scores sc [B][H][T][Tp] float64 -> (probs, tol) [B][H][T][Tp], pitch columns and rows without a valid key 0.
    Per key: a = s / sqrt_dk and x = a - max round once each (u |a|, u |x|), expf 4u; each lane sums ceil(nk / 32) terms, 5 shuffle adds;
    the divide u; the split store 16u.  rho_j = u (|a_j| + |x_j| + 4) + sum_k p_k u (|a_k| + |x_k| + 4) + (ceil(nk / 32) + 22) u."""
    B, H, T, _ = sc.shape
    pr, tol = torch.zeros_like(sc), torch.zeros_like(sc)
    for b, n in enumerate(lens):
        ok = torch.zeros(T, Tp, dtype=torch.bool, device=sc.device)
        ok[:, :T] = _valid_keys(tok[b].to(sc.device), min(int(n), T), T, device=sc.device)
        a = sc[b] / sqrt_dk
        z = torch.where(ok, a, torch.full((), -math.inf, dtype=sc.dtype, device=sc.device))
        m = z.max(-1, keepdim=True).values
        m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
        p = torch.where(ok, torch.exp(z - m), torch.zeros((), dtype=sc.dtype, device=sc.device))
        p = p / p.sum(-1, keepdim=True).clamp_min(1e-300)
        e = torch.where(ok, U32 * (a.abs() + (a - m).abs() + 4), torch.zeros_like(a))
        nk = torch.arange(T, device=sc.device).clamp(max=int(n) - 1).double().view(T, 1) + 1
        rho = e + (p * e).sum(-1, keepdim=True) + (torch.ceil(nk / 32) + 22) * U32
        pr[b], tol[b] = p, torch.where(ok, p * rho + TINY, torch.zeros_like(p))
    return pr, tol


def nll_ref(x, tgt, ncols=None):
    """espb_nll_rows_f32 of logits x [R][V] float64 (the first ncols columns only: a bug) -> (out, tol); 0 where tgt < 0, NaN where
    tgt >= V.  With m the row max and p_j the softmax: each thread's running logsumexp takes its terms with expf (4u) of an argument
    rounded by u |x_j - m| and adds them in sequence (n = ceil(V / 256) + 3 terms per thread at most, float4 or scalar loads), rescaling
    its sum at most n times by expf of a rounded difference whose magnitudes add up to at most the row's spread r = m - min x (and so do
    those of the 12 merges across lanes and warps, each two expf and two roundings); then logf (2u |log s|), x_t - m (u) and the final
    subtraction (u):  tol = u (sum_j p_j (4 + |x_j - m|) + 6 n + 72 + 2 r + 2 |log s| + |x_t - m| + |out|)."""
    R, V = x.shape
    xs = x if ncols is None else x[:, :ncols]
    t = tgt.long()
    lse = torch.logsumexp(xs, -1)
    xt = x.gather(1, t.clamp(0, V - 1).view(R, 1)).view(R)
    out = lse - xt
    m = x.max(-1).values
    p = torch.softmax(x, -1)
    n = -(-V // 256) + 3
    ls = (lse - m).abs()
    tol = U32 * ((p * (4 + (x - m.view(R, 1)).abs())).sum(-1) + 6 * n + 72 + 2 * (m - x.min(-1).values) + 2 * ls + (xt - m).abs()
                 + out.abs())
    out = torch.where(t < 0, torch.zeros_like(out), torch.where(t >= V, torch.full_like(out, math.nan), out))
    return out, tol


def _attn_case(B, H, T, lens, seed, qscale=1.0, device="cpu"):
    """Seeded q / k / v [B][H][T][64] and token ids: token 0 at every 7th key from 3, at keys 64 and 128, and in the last sentence at every
    key before min(T - 1, 97) when B > 1 (the rows before have no valid key, row 97's only valid key is its own)."""
    g = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(B, H, T, 64, generator=g, dtype=torch.float64) * 0.5 for _ in range(3))
    q = q * qscale
    tok = torch.randint(1, 9, (B, T), generator=g, dtype=torch.int32)
    tok[:, 3::7] = 0
    tok[:, 64:65] = 0
    tok[:, 128:129] = 0
    if B > 1 and T > 1:
        tok[-1, :min(T - 1, 97)] = 0
    return q.to(device), k.to(device), v.to(device), tok


def test_tolerances_catch_plausible_bugs():
    """On the CPU, from the float64 references above: each plausible bug moves the reference by more than 10x the tolerance the GPU tests
    of tests/test_gpu_lm_ppl.py use, at a shape they run: in the causal attention (B 2, T 193) one key past the diagonal admitted, the
    token-0 mask ignored and 1 / d_k in place of 1 / sqrt(d_k); in the NLL (V 257, the row maximum in the last column) a logsumexp over
    V - 1 columns."""
    B, H, T, lens = 2, 1, 193, [193, 193]
    q, k, v, tok = _attn_case(B, H, T, lens, seed=T)
    ref, tol = causal_attn_ref(q, k, v, tok, lens)
    assert float(tol.max()) < 1e-4
    for bug in (dict(diag=1), dict(mask_tok=False), dict(scale=1.0 / 64)):
        o, _ = causal_attn_ref(q, k, v, tok, lens, **bug)
        assert _over((o - ref).abs(), tol) > 10, bug
    g = torch.Generator().manual_seed(257)
    x = (torch.rand(6, 257, generator=g, dtype=torch.float64) * 2 - 1) * 80
    x[0, -1] = 80
    tgt = torch.tensor([256, 3, 7, 100, 0, 200], dtype=torch.int32)
    out, tl = nll_ref(x, tgt)
    out2, _ = nll_ref(x, tgt, ncols=256)
    assert float(tl.max()) < 1e-4 and _over((out2 - out).abs(), tl) > 10
