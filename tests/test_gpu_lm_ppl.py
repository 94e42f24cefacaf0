"""-m gpu: LM perplexity on the CUDA path.

* espb_causal_flash_attn_f32 (d_k = 64, csrc/attention.cu) and espb_causal_softmax_f32 (the materialised path for other d_k,
  csrc/lm_ops.cu) against a float64 restatement of TransformerLM._target_mask through MultiHeadedAttention (key j valid for query i iff
  j <= i, j < len and its token id is not 0; a row without a valid key is 0), at T = 1, T not a multiple of 64 or 128, ragged batches and
  keys holding token 0 (including a run of them at the start of a row, so that whole key tiles are masked);
* espb_nll_rows_f32 against a float64 logsumexp, with rows whose target is negative (written 0), V = 5000 (float4 loads) and V = 37;
* ESPnetLanguageModel.nll / batchify_nll end to end against the reference's values (tests/golden/lm_ppl.npz), atol 1e-4 on the
  log-probabilities, and the calc_perplexity files against the reference's.

The inputs are given to the references as the values the kernels read (hi + lo of the split planes), so the tf32 split of the inputs is not
an error here.  Attention tolerance: 3xTF32 products and the online softmax stay within ~3e-5 of |v| at these randn sizes (the bound
derived in test_gpu_attention.py); 2e-4 absolute plus 1e-4 relative leaves margin while a dropped or extra key moves rows by more.
"""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_lm_ppl_host as host  # noqa: E402

gpu = pytest.mark.gpu

CASES = [(1, 2, 1, [1]), (2, 2, 100, [100, 37]), (3, 2, 200, [200, 129, 1]), (2, 3, 257, [257, 190])]


def _ops():
    from espnet_b200 import ops

    return ops


def _split(x):
    return _ops().split_from(x.float().cuda().contiguous())


def _inputs(B, H, T, dk, lens, seed):
    g = torch.Generator().manual_seed(seed)
    D, M = H * dk, B * T
    qkv = torch.randn(M, 3 * D, generator=g) * 0.5
    tok = torch.randint(1, 9, (B, T), generator=g, dtype=torch.int32)
    tok[:, 3::7] = 0                                    # scattered token-0 keys
    if T > 70:
        tok[-1, 1:70] = 0                               # rows 1..69 of the last sentence see key 0 only: a whole key tile masked
    return qkv, tok, torch.tensor(lens, dtype=torch.int32)


def _reference(qkv_split, tok, lens, B, H, T, dk):
    """float64 causal token-masked attention of the values the kernel reads -> [B*T][D]."""
    q = (qkv_split[0] + qkv_split[1]).double().cpu()
    D = H * dk
    out = torch.zeros(B * T, D, dtype=torch.float64)
    i, j = torch.arange(T).view(T, 1), torch.arange(T).view(1, T)
    for b in range(B):
        ok = (j <= i) & (j < int(lens[b])) & (tok[b] != 0).view(1, T)
        for h in range(H):
            Q = q[b * T:(b + 1) * T, h * dk:(h + 1) * dk]
            K = q[b * T:(b + 1) * T, D + h * dk:D + (h + 1) * dk]
            V = q[b * T:(b + 1) * T, 2 * D + h * dk:2 * D + (h + 1) * dk]
            S = torch.where(ok, Q @ K.t() / math.sqrt(dk), torch.full((), -math.inf, dtype=torch.float64))
            P = torch.where(ok, torch.softmax(S, -1), torch.zeros((), dtype=torch.float64))
            out[b * T:(b + 1) * T, h * dk:(h + 1) * dk] = P @ V
    return out


def _attend(qkv_split, tok_d, lens_d, B, H, T, dk, fused):
    ops, D, M = _ops(), H * dk, B * T
    Tp = (T + 31) // 32 * 32
    vt = torch.empty(2, B, H, dk, Tp, device="cuda")
    ctx = torch.full((2, M, D), float("nan"), device="cuda")
    ops.call("espb_v_transpose_f32", ops.ptr(qkv_split), M * 3 * D, B, T, D, H, ops.ptr(lens_d), ops.ptr(vt), B * H * dk * Tp, Tp)
    if fused:
        ops.call("espb_causal_flash_attn_f32", ops.ptr(qkv_split), 0, M * 3 * D, 3 * D, ops.ptr(qkv_split), D, M * 3 * D, 3 * D, ops.ptr(vt),
                 B * H * dk * Tp, Tp, ops.ptr(tok_d), ops.ptr(lens_d), B, H, T, dk, ops.ptr(ctx), M * D, D)
    else:
        sc, probs = torch.empty(B, H, T, Tp, device="cuda"), torch.empty(2, B, H, T, Tp, device="cuda")
        ops.gemm(T, T, dk, qkv_split, M * 3 * D, 3 * D, qkv_split, M * 3 * D, 3 * D, sc, Tp, nbx=H, nby=B, sa=(dk, T * 3 * D),
                 sb=(dk, T * 3 * D), sc=(T * Tp, H * T * Tp), b_off=D)
        ops.call("espb_causal_softmax_f32", ops.ptr(sc), B, H, T, Tp, ops.ptr(lens_d), ops.ptr(tok_d), math.sqrt(dk), ops.ptr(probs),
                 B * H * T * Tp)
        ops.gemm(T, dk, T, probs, B * H * T * Tp, Tp, vt, B * H * dk * Tp, Tp, ctx, D, c_plane=M * D, split_out=True, nbx=H, nby=B,
                 sa=(T * Tp, H * T * Tp), sb=(dk * Tp, H * dk * Tp), sc=(dk, T * D))
    torch.cuda.synchronize()
    return (ctx[0] + ctx[1]).double().cpu()


def _check_rows(got, ref, lens, T):
    for b, n in enumerate(lens):
        np.testing.assert_allclose(got[b * T:b * T + n].numpy(), ref[b * T:b * T + n].numpy(), atol=2e-4, rtol=1e-4)


@gpu
@pytest.mark.parametrize("B,H,T,lens", CASES)
def test_causal_flash_attn_vs_float64(B, H, T, lens):
    qkv, tok, l32 = _inputs(B, H, T, 64, lens, seed=T)
    qs = _split(qkv)
    got = _attend(qs, tok.cuda(), l32.cuda(), B, H, T, 64, fused=True)
    ref = _reference(qs, tok, l32, B, H, T, 64)
    _check_rows(got, ref, lens, T)


@gpu
def test_causal_flash_attn_row_without_valid_key_is_zero():
    """A sentence whose first token is 0: query 0 has no valid key (the reference's masked_fill(mask, 0.0) gives 0), later rows attend the
    later keys only."""
    B, H, T = 1, 2, 70
    qkv, tok, l32 = _inputs(B, H, T, 64, [T], seed=1)
    tok[0, :5] = 0
    qs = _split(qkv)
    got = _attend(qs, tok.cuda(), l32.cuda(), B, H, T, 64, fused=True)
    assert torch.equal(got[:5], torch.zeros(5, H * 64, dtype=torch.float64))
    _check_rows(got, _reference(qs, tok, l32, B, H, T, 64), [T], T)


@gpu
@pytest.mark.parametrize("dk", [32, 128])
@pytest.mark.parametrize("B,H,T,lens", CASES[:3])
def test_causal_softmax_path_vs_float64(dk, B, H, T, lens):
    qkv, tok, l32 = _inputs(B, H, T, dk, lens, seed=T + dk)
    qs = _split(qkv)
    got = _attend(qs, tok.cuda(), l32.cuda(), B, H, T, dk, fused=False)
    _check_rows(got, _reference(qs, tok, l32, B, H, T, dk), lens, T)


@gpu
def test_causal_softmax_kernel_probabilities():
    """The probabilities themselves: zeros at j > i, at token-0 keys, at j >= len and in the pitch columns; rows sum to 1."""
    ops = _ops()
    B, H, T, Tp = 2, 1, 45, 64
    g = torch.Generator().manual_seed(7)
    sc = torch.randn(B, H, T, Tp, generator=g) * 3
    tok = torch.randint(0, 4, (B, T), generator=g, dtype=torch.int32)
    tok[:, 0] = 5
    lens = torch.tensor([45, 30], dtype=torch.int32)
    probs = torch.full((2, B, H, T, Tp), float("nan"), device="cuda")
    # device copies bound to names: a temporary passed as ops.ptr(t.cuda()) is freed before the launch, and the next copy may reuse it
    sc_d, lens_d, tok_d = sc.cuda(), lens.cuda(), tok.cuda()
    ops.call("espb_causal_softmax_f32", ops.ptr(sc_d), B, H, T, Tp, ops.ptr(lens_d), ops.ptr(tok_d), 8.0, ops.ptr(probs), B * H * T * Tp)
    got = (probs[0] + probs[1]).double().cpu()
    i, j = torch.arange(T).view(T, 1), torch.arange(Tp).view(1, Tp)
    for b in range(B):
        ok = (j <= i) & (j < int(lens[b])) & torch.cat([tok[b] != 0, torch.zeros(Tp - T, dtype=torch.bool)]).view(1, Tp)
        s = torch.where(ok, sc[b, 0].double() / 8, torch.full((), -math.inf, dtype=torch.float64))
        ref = torch.where(ok, torch.softmax(s, -1), torch.zeros((), dtype=torch.float64))
        np.testing.assert_allclose(got[b, 0].numpy(), ref.numpy(), atol=1e-6, rtol=1e-5)


@gpu
@pytest.mark.parametrize("rows,V,ld", [(300, 5000, 5000), (64, 37, 37), (17, 37, 40)])
def test_nll_rows_vs_float64(rows, V, ld):
    ops = _ops()
    g = torch.Generator().manual_seed(V)
    x = torch.randn(rows, ld, generator=g) * 4
    x[1, :V] += 30                                      # large logits: the running max must rescale
    tgt = torch.randint(0, V, (rows,), generator=g, dtype=torch.int32)
    tgt[::5] = -1                                       # ignored positions
    out = torch.full((rows,), float("nan"), device="cuda")
    x_d, tgt_d = x.cuda(), tgt.cuda()
    ops.call("espb_nll_rows_f32", ops.ptr(x_d), rows, ld, V, ops.ptr(tgt_d), ops.ptr(out))
    xd = x[:, :V].double()
    ref = torch.logsumexp(xd, -1) - xd.gather(1, tgt.clamp(min=0).long().view(-1, 1)).view(-1)
    ref = torch.where(tgt < 0, torch.zeros((), dtype=torch.float64), ref)
    got = out.double().cpu()
    assert torch.all(got[tgt < 0] == 0)
    np.testing.assert_allclose(got.numpy(), ref.numpy(), atol=2e-5, rtol=2e-6)


@gpu
def test_nll_rows_all_ignored():
    ops = _ops()
    x = torch.randn(8, 64, device="cuda")
    tgt = torch.full((8,), -1, dtype=torch.int32, device="cuda")
    out = torch.full((8,), float("nan"), device="cuda")
    ops.call("espb_nll_rows_f32", ops.ptr(x), 8, 64, 64, ops.ptr(tgt), ops.ptr(out))
    assert torch.equal(out.cpu(), torch.zeros(8))


@gpu
@pytest.mark.parametrize("name", host.LMS)
def test_nll_end_to_end_vs_reference(name, tmp_path):
    import espnet_b200

    z = host._z()
    model, _ = espnet_b200.build_espnet_lm_from_file(*host.write_lm(z, name, str(tmp_path)), device="cuda")
    text, lengths = torch.from_numpy(z["text"]), torch.from_numpy(z["lengths"])
    nll, xl = model.nll(text, lengths)
    assert torch.equal(xl, torch.from_numpy(z[f"{name}:x_lengths"]))
    np.testing.assert_allclose(nll.cpu().numpy(), z[f"{name}:nll"], atol=1e-4, rtol=0)
    nll2, _ = model.batchify_nll(text, lengths, batch_size=2)
    np.testing.assert_allclose(nll2.cpu().numpy(), z[f"{name}:batchify_nll"], atol=1e-4, rtol=0)
    logits, _ = model.lm(text[:2, :10].cuda(), None)
    assert logits.shape == (2, 10, int(z["V"])) and torch.isfinite(logits).all()


@gpu
@pytest.mark.parametrize("name", host.LMS)
@pytest.mark.parametrize("tag,log_base", [("e", None), ("b10", 10.0)])
def test_calc_perplexity_cli_vs_reference(name, tag, log_base, tmp_path):
    from espnet_b200.bin_lm_calc_perplexity import main

    z = host._z()
    cfg, mdl = host.write_lm(z, name, str(tmp_path))
    out = str(tmp_path / "out")
    cmd = ["--output_dir", out, "--batch_size", "2", "--data_path_and_name_and_type", f"{host.write_text(z, str(tmp_path))},text,text",
           "--train_config", cfg, "--model_file", mdl]
    main(cmd + ([] if log_base is None else ["--log_base", str(log_base)]))
    host.check_ppl_files(z, name, tag, out)
