"""TEST INFRASTRUCTURE: the torch-CPU emulation (tests/emu_backend.py) extended with the entry points of the E-Branchformer encoder --
GELU in the GEMM epilogue, espb_csgu_f32, espb_merge_dwconv_f32, espb_zero_pad_rows_f32 -- so that the host logic of
espnet_b200/e_branchformer_encoder.py runs on a box without a GPU.  Each function restates the contract in include/espnet_b200.h.
"""
import torch

import emu_backend as emu


def gemm(*args, act=0, **kw):
    """emu_backend.gemm plus act 3 (exact GELU).  The encoder uses GELU only as channel_proj1's plain [M, N] output with bias."""
    if act != 3:
        return emu.gemm(*args, act=act, **kw)
    C = args[9]
    assert kw.get("R") is None and kw.get("alpha", 1.0) == 1.0 and not kw.get("split_out") and kw.get("c_off", 0) == 0
    assert C.dim() == 2 and args[10] == C.shape[1] and args[0] == C.shape[0] and args[1] == C.shape[1]
    emu.gemm(*args, act=0, **kw)
    C.copy_(torch.nn.functional.gelu(C))
    return True


def _masked(x, lens, Tmax):
    t = torch.arange(Tmax).view(1, Tmax, 1)
    return torch.where(t < lens.view(-1, 1, 1).long(), x, torch.zeros(()))


def _dwconv(x, w, b):
    C, K = w.shape[0], w.numel() // w.shape[0]
    return torch.nn.functional.conv1d(x.transpose(1, 2), w.reshape(C, 1, K), b, padding=(K - 1) // 2, groups=C).transpose(1, 2)


def _csgu(h, B, Tmax, U, lens, ln_g, ln_b, eps, w, b, K, stats, out, out_plane):
    Uh = U // 2
    hv = emu._flat(h)[: B * Tmax * U].view(B, Tmax, U)
    x_r, x_g = hv[..., :Uh], hv[..., Uh:]
    mean = x_g.sum(-1, keepdim=True) / Uh
    var = ((x_g - mean) ** 2).sum(-1, keepdim=True) / Uh
    g = _masked((x_g - mean) * (1.0 / torch.sqrt(var + eps)) * ln_g + ln_b, lens, Tmax)
    z = _masked(x_r * _dwconv(g, w, b), lens, Tmax)
    emu._store(emu._flat(out), torch.arange(B * Tmax * Uh).view(B, Tmax, Uh), z, True, out_plane)


def _merge_dwconv(cat, B, Tmax, C2, lens, w, b, K, out, out_plane):
    x = _masked(emu._flat(cat)[: B * Tmax * C2].view(B, Tmax, C2), lens, Tmax)
    z = _masked(x + _dwconv(x, w, b), lens, Tmax)
    emu._store(emu._flat(out), torch.arange(B * Tmax * C2).view(B, Tmax, C2), z, True, out_plane)


def _zero_pad_rows(x, B, Tmax, D, lens, plane, nplanes):
    f = emu._flat(x)
    for q in range(nplanes):
        v = f[q * plane: q * plane + B * Tmax * D].view(B, Tmax, D)
        v.copy_(_masked(v, lens, Tmax))


def install(monkeypatch):
    """emu_backend.install + the E-Branchformer module and entry points."""
    import espnet_b200.e_branchformer_encoder as ebf
    import espnet_b200.ops as ops

    emu.install(monkeypatch)
    for name, fn in (("espb_csgu_f32", _csgu), ("espb_merge_dwconv_f32", _merge_dwconv), ("espb_zero_pad_rows_f32", _zero_pad_rows)):
        monkeypatch.setitem(emu._TABLE, name, fn)
    monkeypatch.setattr(ebf, "call", emu.call, raising=True)
    monkeypatch.setattr(ebf, "ptr", emu.ptr, raising=True)
    monkeypatch.setattr(ebf, "gemm", gemm, raising=True)
    monkeypatch.setattr(ebf, "new_split", ops.new_split, raising=True)
    # linear() runs through ops.gemm, which emu.install routed to the emulation without GELU
    monkeypatch.setattr(ops, "gemm", gemm, raising=True)
