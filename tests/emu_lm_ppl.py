"""TEST INFRASTRUCTURE: the torch-CPU emulation (tests/emu_backend.py, tests/emu_rnn.py) extended with the entry points of the LMs'
full-sequence forward and their nll (espnet_b200/lm.py): espb_causal_flash_attn_f32, espb_causal_softmax_f32 and espb_nll_rows_f32.  Each
function restates the contract in include/espnet_b200.h.
"""
import math

import torch

import emu_backend as emu
import emu_rnn


def _key_mask(tok, lens, b, T):
    """[T][T] valid (query i, key j): j <= i, j < lens[b], tok[b][j] != 0."""
    i, j = torch.arange(T).view(T, 1), torch.arange(T).view(1, T)
    return (j <= i) & (j < int(lens[b])) & (emu._flat(tok)[b * T:(b + 1) * T] != 0).view(1, T)


def _masked_probs(S, ok):
    p = torch.softmax(torch.where(ok, S, torch.full((), float("-inf"))), dim=-1)
    return torch.where(ok, p, torch.zeros(()))       # rows without a valid key: 0 (the NaNs of an all -inf row are dropped)


def _causal_flash(q, q_off, q_plane, ldq, k, k_off, k_plane, ldk, vt, vt_plane, Tp, tok, lens, B, H, T, dk, out, out_plane, ldo):
    qf, kf, vf, of = emu._flat(q), emu._flat(k), emu._flat(vt), emu._flat(out)
    c = torch.arange(dk)
    for b in range(B):
        rows = (b * T + torch.arange(T)).view(T, 1)
        ok = _key_mask(tok, lens, b, T)
        for h in range(H):
            qo = q_off + rows * ldq + h * dk + c
            ko = k_off + rows * ldk + h * dk + c
            vo = ((b * H + h) * dk + c.view(dk, 1)) * Tp + torch.arange(T).view(1, T)
            S = (qf[qo] + qf[qo + q_plane]) @ (kf[ko] + kf[ko + k_plane]).t() / math.sqrt(dk)
            O = _masked_probs(S, ok) @ (vf[vo] + vf[vo + vt_plane]).t()
            emu._store(of, rows * ldo + h * dk + c, O, True, out_plane)


def _causal_softmax(sc, B, H, T, Tp, lens, tok, sqrt_dk, probs, plane):
    s = emu._flat(sc)[: B * H * T * Tp].view(B, H, T, Tp)
    pf = emu._flat(probs)
    for b in range(B):
        ok = torch.zeros(T, Tp, dtype=torch.bool)
        ok[:, :T] = _key_mask(tok, lens, b, T)
        for h in range(H):
            p = _masked_probs(s[b, h] / sqrt_dk, ok)
            emu._store(pf, ((b * H + h) * T + torch.arange(T).view(T, 1)) * Tp + torch.arange(Tp).view(1, Tp), p, True, plane)


def _nll_rows(x, rows, ld, V, tgt, out):
    xv = emu._flat(x)[: rows * ld].view(rows, ld)[:, :V]
    t = emu._flat(tgt)[:rows].long()
    nll = torch.logsumexp(xv, dim=-1) - xv.gather(1, t.clamp(0, V - 1).view(rows, 1)).view(rows)
    emu._flat(out)[:rows] = torch.where(t < 0, torch.zeros(()), nll)


def install(monkeypatch):
    """emu_rnn.install (search, LSTM LM cells, LSTM recurrence) + the perplexity entry points."""
    emu_rnn.install(monkeypatch)
    for name, fn in (("espb_causal_flash_attn_f32", _causal_flash), ("espb_causal_softmax_f32", _causal_softmax),
                     ("espb_nll_rows_f32", _nll_rows)):
        monkeypatch.setitem(emu._TABLE, name, fn)
