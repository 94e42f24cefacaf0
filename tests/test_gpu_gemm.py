"""wgmma 3xTF32 GEMM and SIMT GEMM vs a float64 reference of the same op (through the C-ABI)."""
import pytest
import torch

import os

pytestmark = pytest.mark.gpu
MODES = [m for m in os.environ.get("ESPB_TEST_GEMM_MODES", "simt,tc,tc2").split(",") if m]


def _split(x):
    from espnet_b200 import ops

    return ops.split_from(x)


def _ref(a, b, bias=None, act=0, res=None, alpha=1.0):
    v = a.double() @ b.double().t()
    if bias is not None:
        v = v + bias.double()
    if act == 1:
        v = torch.relu(v)
    elif act == 2:
        v = v * torch.sigmoid(v)
    v = alpha * v
    if res is not None:
        v = v + res.double()
    return v


def _tol(mode, K, scale=1.0, M=None):
    """SIMT: fp32 FFMA.  tc: all of K accumulates inside the tensor core, so the error of an O(1) output may grow with the number of
    accumulation steps (3*K/8).  tc2 promotes every chunk of 4 k-blocks into fp32 registers, at every M."""
    if mode == "tc":
        return scale * (2e-5 + 1.0e-7 * K)
    return scale * 2e-5   # simt (FFMA) and tc2 (chunked promotion: long accumulation chain in fp32 registers)


SHAPES = [(2000, 512, 2048), (1500, 1536, 512), (128, 64, 32), (128, 256, 64), (200, 130, 96), (640, 512, 512), (937, 512, 2048), (22, 50, 64), (300, 5000, 64),
          (1000, 1536, 512), (129, 65, 33 * 4),
          # decode-step shapes: fewer 128-column tiles than SMs -> 64-column tiles (ragged K, N overhang)
          (640, 512, 2048), (640, 1536, 512), (100, 200, 300), (50, 129, 9 * 32), (640, 2048, 512), (320, 5000, 512),
          # 64-column tiles (N <= d_k = 64): column overhang and a K tail (K must stay a multiple of 4: TMA strides)
          (1500, 48, 520)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_linear_plain(mode, M, N, K):
    from espnet_b200 import ops

    torch.manual_seed(M * 7 + N * 3 + K)
    a, b = torch.randn(M, K, device="cuda"), torch.randn(N, K, device="cuda") / K ** 0.5
    bias = torch.randn(N, device="cuda")
    out = torch.full((M, N), float("nan"), device="cuda")
    used_tc = ops.linear(_split(a), _split(b), out, bias=bias, force=mode)
    assert used_tc == (mode != "simt")
    torch.cuda.synchronize()
    ref = _ref(a, b, bias)
    err = (out.double() - ref).abs().max().item()
    print(f"[{mode}] M{M} N{N} K{K} max abs err {err:.3e}")
    assert err < _tol(mode, K, M=M), f"{mode} M{M} N{N} K{K} max abs err {err}"


@pytest.mark.parametrize("mode", MODES)
def test_linear_epilogues(mode):
    from espnet_b200 import ops

    torch.manual_seed(1)
    M, N, K = 333, 192, 128
    a, b = torch.randn(M, K, device="cuda"), torch.randn(N, K, device="cuda") / K ** 0.5
    bias, res = torch.randn(N, device="cuda"), torch.randn(M, N, device="cuda")
    # swish + split output
    outs = torch.zeros(2, M, N, device="cuda")
    ops.linear(_split(a), _split(b), outs, bias=bias, act=ops.ACT_SWISH, split_out=True, force=mode)
    ref = _ref(a, b, bias, act=2)
    assert ((outs[0].double() + outs[1].double()) - ref).abs().max().item() < _tol(mode, K, M=M)
    assert (outs[0].view(torch.int32) & 0x1FFF).abs().max().item() == 0  # hi plane is exactly tf32
    # relu
    out = torch.zeros(M, N, device="cuda")
    ops.linear(_split(a), _split(b), out, bias=bias, act=ops.ACT_RELU, force=mode)
    assert (out.double() - _ref(a, b, bias, act=1)).abs().max().item() < _tol(mode, K, M=M)
    # in-place residual with alpha
    x = res.clone()
    ops.linear(_split(a), _split(b), x, bias=bias, residual=x, alpha=0.5, force=mode)
    assert (x.double() - _ref(a, b, bias, res=res, alpha=0.5)).abs().max().item() < _tol(mode, K, M=M)


@pytest.mark.parametrize("mode", MODES)
def test_batched_strided_attention_shapes(mode):
    """The three attention GEMMs' addressing: heads as batch-x, utterances as batch-y, shared B operand, K tail."""
    from espnet_b200 import ops

    torch.manual_seed(2)
    Bn, H, T, dk = 3, 4, 77, 16
    D, Tp = H * dk, 80
    M = Bn * T
    q = torch.randn(M, D, device="cuda")
    qkv = torch.randn(M, 3 * D, device="cuda")
    qs, qkvs = _split(q), _split(qkv)
    ac = torch.zeros(Bn, H, T, Tp, device="cuda")
    ops.gemm(T, T, dk, qs, M * D, D, qkvs, M * 3 * D, 3 * D, ac, Tp, nbx=H, nby=Bn, sa=(dk, T * D), sb=(dk, T * 3 * D),
             sc=(T * Tp, H * T * Tp), b_off=D, force=mode)
    qh = q.view(Bn, T, H, dk).permute(0, 2, 1, 3).double()
    kh = qkv[:, D:2 * D].reshape(Bn, T, H, dk).permute(0, 2, 1, 3).double()
    ref = qh @ kh.transpose(-1, -2)
    assert (ac[..., :T].double() - ref).abs().max().item() < _tol(mode, dk, 4, M=T * H * Bn)
    # shared B across batch-y (positional matrix), output pitch Rp
    R, L, Rp = 2 * T - 1, 2, 156
    p_all = torch.randn(R, L * D, device="cuda")
    bd = torch.zeros(Bn, H, T, Rp, device="cuda")
    ops.gemm(T, R, dk, qs, M * D, D, _split(p_all), R * L * D, L * D, bd, Rp, nbx=H, nby=Bn, sa=(dk, T * D), sb=(dk, 0),
             sc=(T * Rp, H * T * Rp), b_off=1 * D, force=mode)
    ph = p_all[:, D:2 * D].reshape(R, H, dk).permute(1, 0, 2).double()
    ref = qh @ ph.transpose(-1, -2).unsqueeze(0)
    assert (bd[..., :R].double() - ref).abs().max().item() < _tol(mode, dk, 4, M=T * H * Bn)
    # P @ V with K = T (not a multiple of 32) and transposed V, output scattered back to [M][D] (split)
    probs = torch.rand(Bn, H, T, Tp, device="cuda")
    probs[..., T:] = 0
    vt = torch.randn(Bn, H, dk, Tp, device="cuda")
    ctx = torch.zeros(2, M, D, device="cuda")
    ops.gemm(T, dk, T, _split(probs), Bn * H * T * Tp, Tp, _split(vt), Bn * H * dk * Tp, Tp, ctx, D, c_plane=M * D, split_out=True,
             nbx=H, nby=Bn, sa=(T * Tp, H * T * Tp), sb=(dk * Tp, H * dk * Tp), sc=(dk, T * D), force=mode)
    ref = (probs[..., :T].double() @ vt[..., :T].double().transpose(-1, -2)).permute(0, 2, 1, 3).reshape(M, D)
    assert ((ctx[0].double() + ctx[1].double()) - ref).abs().max().item() < _tol(mode, T, 4, M=T * H * Bn)


@pytest.mark.parametrize("mode", MODES)
def test_conv2_implicit_gemm_and_outer_k(mode):
    """conv1 kernel -> conv2 as implicit GEMM over the parity-split layout -> embed.out with the K axis split over f."""
    import math

    from espnet_b200 import ops
    from espnet_b200.lib import call, ptr

    torch.manual_seed(3)
    Bn, Tf, F, C, D = 2, 61, 80, 64, 64
    feats = torch.randn(Bn, Tf, F, device="cuda")
    w1, b1 = torch.randn(C, 1, 3, 3, device="cuda") * 0.3, torch.randn(C, device="cuda") * 0.1
    w2, b2 = torch.randn(C, C, 3, 3, device="cuda") * 0.05, torch.randn(C, device="cuda") * 0.1
    T1, F1 = (Tf - 3) // 2 + 1, (F - 3) // 2 + 1
    T2, F2 = (T1 - 3) // 2 + 1, (F1 - 3) // 2 + 1
    T1h, F1h = (T1 + 1) // 2, (F1 + 1) // 2
    wo, bo = torch.randn(D, C * F2, device="cuda") / (C * F2) ** 0.5, torch.randn(D, device="cuda")
    c1 = torch.zeros(Bn, 8, F1h, T1h, C, device="cuda")
    call("espb_conv1_relu_f32", ptr(feats), Bn, Tf, F, ptr(w1.view(C, 9).contiguous()), ptr(b1), C, ptr(c1), T1, F1, T1h, F1h)
    x1 = torch.relu(torch.nn.functional.conv2d(feats.unsqueeze(1).double(), w1.double(), b1.double(), stride=2))  # (B,C,T1,F1)
    # check conv1 through the parity layout
    got = torch.zeros(Bn, C, T1, F1, device="cuda", dtype=torch.float64)
    full = c1[:, :4].double() + c1[:, 4:].double()
    for pt in range(2):
        for pf in range(2):
            sub = full[:, pt * 2 + pf]  # (B, F1h, T1h, C)
            nt, nf = (T1 - pt + 1) // 2, (F1 - pf + 1) // 2
            got[:, :, pt::2, pf::2] = sub[:, :nf, :nt].permute(0, 3, 2, 1)
    assert (got - x1).abs().max().item() < 1e-5
    c2 = torch.zeros(2, Bn, F2, T2, C, device="cuda")
    w2p = ops.split_from(w2.permute(0, 2, 3, 1).reshape(C, 9 * C).contiguous())
    ops.gemm(T2, C, 9 * C, c1, 0, 0, w2p, C * 9 * C, 9 * C, c2, C, c_plane=Bn * F2 * T2 * C, split_out=True, bias=b2, act=ops.ACT_RELU,
             nbx=F2, nby=Bn, sc=(T2 * C, F2 * T2 * C), a_mode=1, conv=(T1h, F1h, C), force=mode)
    x2 = torch.relu(torch.nn.functional.conv2d(x1, w2.double(), b2.double(), stride=2))  # (B,C,T2,F2)
    got2 = (c2[0].double() + c2[1].double()).permute(0, 3, 2, 1)  # (B,F2,T2,C) -> (B,C,T2,F2)
    assert (got2 - x2).abs().max().item() < 5e-5
    x = torch.zeros(Bn * T2, D, device="cuda")
    wop = ops.split_from(wo.view(D, C, F2).permute(0, 2, 1).reshape(D, F2 * C).contiguous())
    ops.gemm(T2, D, F2 * C, c2, Bn * F2 * T2 * C, C, wop, D * F2 * C, F2 * C, x, D, bias=bo, alpha=math.sqrt(D), nbx=1, nby=Bn,
             sa=(T2 * C, F2 * T2 * C), sc=(0, T2 * D), kob=C // 32, force=mode)
    ref = (x2.transpose(1, 2).reshape(Bn, T2, C * F2) @ wo.double().t() + bo.double()) * math.sqrt(D)
    assert (x.view(Bn, T2, D).double() - ref).abs().max().item() < _tol(mode, F2 * C, 10, M=T2 * Bn)
