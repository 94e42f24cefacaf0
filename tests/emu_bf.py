"""TEST INFRASTRUCTURE: the torch-CPU emulation of tests/emu_ebf.py extended with the two entry points of the Branchformer merge --
espb_branch_pool_f32 and espb_branch_merge_f32 -- so that the host logic of espnet_b200/branchformer_encoder.py runs on a box without a GPU.
Each function restates the contract in include/espnet_b200.h."""
import math

import torch

import emu_backend as emu
import emu_ebf


def _rows(x, M, D, ldx):
    """M rows of D floats at row stride ldx, starting where the (possibly column-offset) view x starts."""
    return torch.as_strided(x, (M, D), (ldx, 1))


def _branch_pool(x1, x2, ldx, B, Tmax, D, lens, pool_w, pool_b, weight_w, weight_b, part, merge_w):
    assert part.numel() >= B * 2 * ((Tmax + 31) // 32) * (D + 2), "branch_pool: workspace too small"
    pool_w, weight_w = emu._flat(pool_w).view(2, D), emu._flat(weight_w).view(2, D)
    mw = emu._flat(merge_w)
    for b in range(B):
        n = int(lens[b])
        wk = []
        for k, x in enumerate((x1, x2)):
            xb = _rows(x, B * Tmax, D, ldx)[b * Tmax: b * Tmax + n]
            s = (xb @ pool_w[k] + pool_b[k]) / math.sqrt(D)
            pooled = torch.softmax(s, 0) @ xb
            wk.append(pooled @ weight_w[k] + weight_b[k])
        mw[2 * b: 2 * b + 2] = torch.softmax(torch.stack(wk), 0)


def _branch_merge(x1, x2, ldx, M, D, Tmax, merge_w, w1, w2, out, out_plane):
    a, e = _rows(x1, M, D, ldx), _rows(x2, M, D, ldx)
    if merge_w is None:
        c1, c2 = torch.tensor(w1, dtype=torch.float32), torch.tensor(w2, dtype=torch.float32)
    else:
        w = emu._flat(merge_w).view(-1, 2).repeat_interleave(Tmax, 0)[:M]
        c1, c2 = w[:, :1], w[:, 1:]
    y = c1 * a + c2 * e
    emu._store(emu._flat(out), torch.arange(M * D).view(M, D), y, True, out_plane)


def install(monkeypatch):
    """emu_ebf.install + the Branchformer merge entry points (the Branchformer module launches through ops.*)."""
    emu_ebf.install(monkeypatch)
    for name, fn in (("espb_branch_pool_f32", _branch_pool), ("espb_branch_merge_f32", _branch_merge)):
        monkeypatch.setitem(emu._TABLE, name, fn)
