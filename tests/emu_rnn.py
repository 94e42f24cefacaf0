"""TEST INFRASTRUCTURE: the torch-CPU emulation (tests/emu_backend.py) extended with the entry points of the RNN model family --
espnet_b200/rnn_encoder.py and rnn_decoder.py: espb_vgg_conv1_relu_f32, espb_vgg_pool_f32, espb_lstm_rec_step_f32, espb_rnn_proj_post_f32,
espb_att_loc_step_f32 and espb_drop_cand_i32.  Each function restates the contract in include/espnet_b200.h; the implicit-GEMM convs
(a_mode 2) go through emu_subsampling's dense gather, the decoder's gather and cell kernels through emu_rnnlm.
"""
import torch
import torch.nn.functional as F

import emu_backend as emu
import emu_rnnlm
import emu_subsampling


def _span(t, n):
    """A flat view of n elements of t's storage starting at t's first element (entry points receive interior pointers)."""
    return torch.empty(0, dtype=t.dtype).set_(t.untyped_storage(), t.storage_offset(), (n,), (1,))


def _store_split(t, idx, v, plane):
    emu._store(_span(t, int(idx.max()) + 1 + plane), idx, v, True, plane)


def _vgg_conv1(feats, B, Tf, Fr, lens, w, bias, C, out, T):
    Fp, Tp = Fr + 2, T + 2
    o = out.view(B, 2, Fp, Tp, C)
    for b in range(B):
        L = int(lens[b])
        x = torch.zeros(1, 1, T, Fr)
        x[0, 0, :L] = feats.view(B, Tf, Fr)[b, :L]
        y = torch.relu(F.conv2d(x, w.view(C, 1, 3, 3), bias, padding=1))[0]   # [C][T][F]
        y[:, L:] = 0
        v = torch.zeros(Fp, Tp, C)
        v[1:-1, 1:-1] = y.permute(2, 1, 0)
        hi = emu.tf32_hi(v)
        o[b, 0], o[b, 1] = hi, emu.tf32_lo(v, hi)


def _vgg_pool(x, B, Fr, T, C, lens, pool, flat, out, out_plane):
    Fo, To = ((Fr + 1) // 2, (T + 1) // 2) if pool else (Fr, T)
    xs = x.view(B, Fr, T, C)
    f = emu._flat(out)
    for b in range(B):
        L = int(lens[b])
        OL = (L + 1) // 2 if pool else L
        xi = xs[b].permute(2, 1, 0)[None, :, :L]   # [1][C][L][F]
        r = F.max_pool2d(xi, 2, stride=2, ceil_mode=True)[0] if pool else xi[0]
        full = torch.zeros(C, To, Fo)
        full[:, :OL] = r
        if flat:
            idx = b * To * C * Fo + torch.arange(To * C * Fo)
            emu._store(f, idx, full.transpose(0, 1).reshape(-1), True, out_plane)
        else:
            v = torch.zeros(Fo + 2, To + 2, C)
            v[1:-1, 1:-1] = full.permute(2, 1, 0)
            emu._store(f, b * 2 * out_plane + torch.arange(v.numel()), v.reshape(-1), True, out_plane)


def _lstm_rec(xg, hg, lens, s, B, T, H, Hp, ndir, h, h_plane, c, y, y_plane, ldy):
    xgv = emu._flat(xg).view(B, T, ndir, 4, H)
    hgv = emu._flat(hg)[: ndir * B * 4 * H].view(ndir, B, 4, H)
    hf, cf, yf = emu._flat(h), emu._flat(c).view(ndir, B, H), emu._flat(y)
    j = torch.arange(H)
    for d in range(ndir):
        for b in range(B):
            L = int(lens[b])
            if s >= L:
                if s < T:
                    emu._store(yf, (b * T + s) * ldy + d * H + j, torch.zeros(H), True, y_plane)
                continue
            t = L - 1 - s if d else s
            g = xgv[b, t, d].clone()
            cp = torch.zeros(H)
            if s > 0:
                g = g + hgv[d, b]
                cp = cf[d, b]
            cn = torch.sigmoid(g[1]) * cp + torch.sigmoid(g[0]) * torch.tanh(g[2])
            hn = torch.sigmoid(g[3]) * torch.tanh(cn)
            cf[d, b] = cn
            emu._store(hf, (d * B + b) * Hp + j, hn, True, h_plane)
            emu._store(yf, (b * T + t) * ldy + d * H + j, hn, True, y_plane)


def _proj_post(x, B, T, D, lens, act, write_plain, out, out_plane, ldo):
    xv = emu._flat(x)[: B * T * D].view(B, T, D)
    v = torch.tanh(xv) if act else xv.clone()
    for b in range(B):
        v[b, int(lens[b]):] = 0
    if write_plain:
        xv.copy_(v)
    if out is not None:
        rows = torch.arange(B * T).view(-1, 1)
        emu._store(emu._flat(out), rows * ldo + torch.arange(D).view(1, D), v.view(B * T, D), True, out_plane)


def _att_loc(enc_h, enc, enc_plane, lens, W, Tmax, A, E, dec_z, conv_w, chans, filts, att_wt, gvec, gvec_b, anc, anc_ld, pos, step_ptr,
             ring, n, out, out_plane, out_ld, out2, out2_plane, out2_ld):
    pos += emu._step(step_ptr)
    U = n // W
    eh = emu._flat(enc_h)[: U * Tmax * A].view(U, Tmax, A)
    ef = emu._flat(enc)
    ev = (ef[: U * Tmax * E] + ef[enc_plane: enc_plane + U * Tmax * E]).view(U, Tmax, E)
    rv = ring.view(2, n, Tmax)
    prev_ring = rv[(pos - 1) & 1].clone()
    cw = conv_w.view(chans, 1, 1, 2 * filts + 1)
    for s in range(n):
        u, L = s // W, int(lens[s // W])
        if pos == 0:
            prev = torch.full((L,), 1.0 / L)
        else:
            prev = prev_ring[int(anc.view(-1)[s * anc_ld + pos - 1]), :L]
        conv = F.conv2d(prev.view(1, 1, 1, L), cw, padding=(0, filts))[0, :, 0].t()   # (L, chans)
        e = torch.tanh(conv @ att_wt.view(chans, A) + eh[u, :L] + dec_z.view(n, A)[s]) @ gvec + gvec_b[0]
        w = torch.softmax(2.0 * e, dim=0)
        rv[pos & 1, s] = 0
        rv[pos & 1, s, :L] = w
        ctx = w @ ev[u, :L]
        for o, plane, ld in ((out, out_plane, out_ld), (out2, out2_plane, out2_ld)):
            if o is not None:
                _store_split(o, s * ld + torch.arange(E), ctx, plane)


def _drop_cand(valid, n, PC, j):
    emu._flat(valid)[torch.arange(n) * PC + j] = 0


def install(monkeypatch):
    """emu_rnnlm.install (search + LSTM cells) + the subsampling GEMM routing (a_mode 2) + the RNN family's entry points."""
    import espnet_b200.rnn_decoder as rdec

    emu_rnnlm.install(monkeypatch)
    emu_subsampling.install(monkeypatch)
    monkeypatch.setattr(rdec, "call", emu.call, raising=True)
    monkeypatch.setattr(rdec, "ptr", emu.ptr, raising=True)
    for name, fn in (("espb_vgg_conv1_relu_f32", _vgg_conv1), ("espb_vgg_pool_f32", _vgg_pool), ("espb_lstm_rec_step_f32", _lstm_rec),
                     ("espb_rnn_proj_post_f32", _proj_post), ("espb_att_loc_step_f32", _att_loc), ("espb_drop_cand_i32", _drop_cand),
                     ("espb_rnnlm_gather_f32", emu_rnnlm._rnnlm_gather), ("espb_lstm_cell_f32", emu_rnnlm._lstm_cell)):
        monkeypatch.setitem(emu._TABLE, name, fn)
