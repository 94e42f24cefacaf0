"""TEST INFRASTRUCTURE: the torch-CPU emulation (tests/emu_backend.py) extended with the two entry points of the LSTM LM --
espnet_b200/lm.py's SequentialRNNLM -- espb_rnnlm_gather_f32 and espb_lstm_cell_f32.  Each function restates the contract in
include/espnet_b200.h (state ring h, c [2][L][n][Hp], split operands [2][n][Kp_l] back to back, pad columns untouched).
"""
import torch

import emu_backend as emu


def _parents(anc, anc_ld, pos, n):
    return anc.view(-1)[torch.arange(n) * anc_ld + pos - 1].long() if pos > 0 else None


def _rnnlm_gather(tok, emb, E, Ep, anc, anc_ld, pos, step_ptr, h_ring, L, n, H, Hp, xs):
    pos += emu._step(step_ptr)
    kp0, kp1 = Ep + Hp, 2 * Hp
    f = emu._flat(xs)
    rows = torch.arange(n).view(n, 1)
    emu._store(f, rows * kp0 + torch.arange(E).view(1, E), emb.view(-1, E)[tok.view(-1)[:n].long()], True, n * kp0)
    p = _parents(anc, anc_ld, pos, n)
    hr = h_ring.view(2, L, n, Hp)
    for l in range(L):
        kp, base, col = (kp0, 0, Ep) if l == 0 else (kp1, 2 * n * kp0 + 2 * (l - 1) * n * kp1, Hp)
        v = hr[(pos - 1) & 1, l][p][:, :H] if p is not None else torch.zeros(n, H)
        emu._store(f, base + rows * kp + col + torch.arange(H).view(1, H), v, True, n * kp)


def _lstm_cell(gates, anc, anc_ld, pos, step_ptr, h_ring, c_ring, layer, L, n, H, Hp, out, out_plane, out_ld):
    pos += emu._step(step_ptr)
    g = emu._flat(gates)[: n * 4 * H].view(n, 4, H)
    p = _parents(anc, anc_ld, pos, n)
    hr, cr = h_ring.view(2, L, n, Hp), c_ring.view(2, L, n, Hp)
    cp = cr[(pos - 1) & 1, layer][p][:, :H] if p is not None else torch.zeros(n, H)
    c = torch.sigmoid(g[:, 1]) * cp + torch.sigmoid(g[:, 0]) * torch.tanh(g[:, 2])
    h = torch.sigmoid(g[:, 3]) * torch.tanh(c)
    hr[pos & 1, layer, :, :H] = h
    cr[pos & 1, layer, :, :H] = c
    emu._store(emu._flat(out), torch.arange(n).view(n, 1) * out_ld + torch.arange(H).view(1, H), h, True, out_plane)


def install(monkeypatch):
    """emu_backend.install_search + the LSTM LM entry points."""
    emu.install_search(monkeypatch)
    for name, fn in (("espb_rnnlm_gather_f32", _rnnlm_gather), ("espb_lstm_cell_f32", _lstm_cell)):
        monkeypatch.setitem(emu._TABLE, name, fn)
