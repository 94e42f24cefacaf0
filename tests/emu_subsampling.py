"""TEST INFRASTRUCTURE: the torch-CPU emulation of tests/emu_ebf.py extended with the entry points of the conv2d2 / conv2d6 / conv2d8 input
layers -- espb_conv1_relu_phase_f32, espb_phase_split_f32 and the implicit-GEMM convolutions of EspbGemmDesc.a_mode 1..3 -- so that the
subsampling host logic of espnet_b200/layers.py runs on a box without a GPU.  Each function restates the contract in include/espnet_b200.h."""
import torch

import emu_backend as emu
import emu_ebf

CONV_GEOM = {1: (3, 2), 2: (3, 1), 3: (5, 3)}   # a_mode -> (kernel, stride) (gemm.h: conv_geom)


def _phase_store(out, y, B, s, Th, Fh):
    """y [B][C][T][F] -> out [B][plane*s*s + (t%s)*s + (f%s)][Fh][Th][C], tf32 hi / lo planes."""
    _, C, T, F = y.shape
    sub = Fh * Th * C
    b, c, t, f = torch.meshgrid(torch.arange(B), torch.arange(C), torch.arange(T), torch.arange(F), indexing="ij")
    off = b * 2 * s * s * sub + ((t % s) * s + f % s) * sub + ((f // s) * Th + t // s) * C + c
    emu._store(emu._flat(out), off, y, True, s * s * sub)


def _conv1_relu_phase(feats, B, Tf, F, w, bias, C, out, T1, F1, s, T1h, F1h):
    assert 1 <= s <= 3 and T1h * s >= T1 and F1h * s >= F1
    y = torch.relu(torch.nn.functional.conv2d(feats.view(B, 1, Tf, F), w.view(C, 1, 3, 3), bias, stride=2))   # [B][C][T1][F1]
    assert y.shape[2:] == (T1, F1)
    _phase_store(out, y, B, s, T1h, F1h)


def _phase_split(x, x_plane, B, F, T, C, s, Th, Fh, out):
    xf = emu._flat(x)
    v = (xf[: B * F * T * C] + xf[x_plane: x_plane + B * F * T * C]).view(B, F, T, C).permute(0, 3, 2, 1)   # hi + lo: exact
    _phase_store(out, v, B, s, Th, Fh)


def _conv_operand(A, K, M, nbx, nby, a_mode, conv, a_off):
    """The implicit-GEMM operand of a_mode 1..3 gathered into a dense split [2][nby][nbx][M][K] (lo plane zero: hi + lo is exact)."""
    k, s = CONV_GEOM[a_mode]
    th, fh, cin = conv
    assert K == k * k * cin
    nph = s * s
    Af = emu._flat(A)
    m, kk = torch.arange(M).view(M, 1), torch.arange(K).view(1, K)
    tap, c = kk // cin, kk % cin
    kt, kf = tap // k, tap % k
    par = (kt % s) * s + kf % s
    sub = fh * th * cin
    dense = torch.zeros(2, nby, nbx, M, K)
    for by in range(nby):
        for bx in range(nbx):
            tt, ff = m + kt // s, bx + kf // s
            ok = (tt < th) & (ff < fh)
            off = a_off + by * 2 * nph * sub + (torch.clamp(ff, max=fh - 1) * th + torch.clamp(tt, max=th - 1)) * cin + c
            dense[0, by, bx] = torch.where(ok, Af[off + par * sub] + Af[off + (nph + par) * sub], torch.zeros(()))
    return dense


def install(monkeypatch):
    """emu_ebf.install + the input-layer entry points; the GEMM routes a_mode 1..3 through a dense gather and the installed emulation."""
    import espnet_b200.ops as ops

    emu_ebf.install(monkeypatch)
    for name, fn in (("espb_conv1_relu_phase_f32", _conv1_relu_phase), ("espb_phase_split_f32", _phase_split)):
        monkeypatch.setitem(emu._TABLE, name, fn)
    base = ops.gemm

    def gemm(M, N, K, A, a_plane, lda, *args, a_mode=0, conv=(0, 0, 0), a_off=0, nbx=1, nby=1, **kw):
        if a_mode == 0:
            return base(M, N, K, A, a_plane, lda, *args, nbx=nbx, nby=nby, a_off=a_off, **kw)
        dense = _conv_operand(A, K, M, nbx, nby, a_mode, conv, a_off)
        return base(M, N, K, dense, dense[0].numel(), K, *args, nbx=nbx, nby=nby, sa=(M * K, nbx * M * K), **kw)

    monkeypatch.setattr(ops, "gemm", gemm, raising=True)
