"""The persistent tensor-core GEMM's tile schedule: tile counts around the SM count, batch slices, windows inside larger outputs, conv2 and
kob addressing, bitwise invariance of a tile's result under the schedule, and the residual aliasing contract (gemm.h)."""
import pytest
import torch

pytestmark = pytest.mark.gpu
VERSIONS = ["tc", "tc2"]


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _split(x):
    from espnet_b200 import ops

    return ops.split_from(x)


def _tol(mode, K, scale=1.0):
    return scale * (2e-5 + 1.0e-7 * K) if mode == "tc" else scale * 2e-5


def _counts():
    s = _sms()
    return {"1": 1, "sms-1": s - 1, "sms": s, "sms+1": s + 1, "3sms+5": 3 * s + 5}


# (tile count, width): 64-column tiles are reachable at every count through N <= 64; 128-column tiles only where the problem has at
# least as many 128-column tiles as SMs
CASES = [(c, 64) for c in ("1", "sms-1", "sms", "sms+1", "3sms+5")] + [(c, 128) for c in ("sms", "sms+1", "3sms+5")]


@pytest.mark.parametrize("mode", VERSIONS)
@pytest.mark.parametrize("count,width", CASES)
@pytest.mark.parametrize("layout", ["rows", "batched"])
def test_tile_counts(mode, count, width, layout):
    """tiles = count: `rows` as 128-row blocks of one slice (ragged last block), `batched` as count slices of one tile each, with per-slice
    A / B / bias, and C written as the right half of a [.., 2N] row (column offset, ldc = 2N) with 128 padding rows after each slice's M
    rows.  Everything outside each slice's [M, N] window stays NaN."""
    from espnet_b200 import ops

    c = _counts()[count]
    N = 48 if width == 64 else 100   # one column tile either way; N > 64 keeps 128-column tiles when there are >= SMs of them
    K = 96
    torch.manual_seed(c * 3 + width)
    if layout == "rows":
        nb, M = 1, 128 * (c - 1) + 37
    else:
        nb, M = c, 90
    nby = 2 if nb % 2 == 0 else 1
    nbx = nb // nby
    a = torch.randn(nb, M, K, device="cuda")
    b = torch.randn(nb, N, K, device="cuda") / K ** 0.5
    bias = torch.randn(nb, N, device="cuda")
    Mp = M + 128   # rows M..M+127 of each slice: what a ragged last row block would write past the window
    out = torch.full((nb, Mp, 2 * N), float("nan"), device="cuda")
    ops.gemm(M, N, K, _split(a), nb * M * K, K, _split(b), nb * N * K, K, out, 2 * N, bias=bias, sbias_x=N, nbx=nbx, nby=nby,
             sa=(M * K, nbx * M * K), sb=(N * K, nbx * N * K), sc=(Mp * 2 * N, nbx * Mp * 2 * N), c_off=N, force=mode)
    torch.cuda.synchronize()
    ref = a.double() @ b.double().transpose(1, 2) + bias.double()[torch.arange(nb) % nbx, None, :]   # bias follows batch-x only
    assert torch.isnan(out[:, :M, :N]).all()
    assert torch.isnan(out[:, M:]).all()
    err = (out[:, :M, N:].double() - ref).abs().max().item()
    assert err < _tol(mode, K), f"{mode} tiles {c} width {width} {layout}: max abs err {err}"


def _sub_gemm(mode, a, b, bias, out, r0, r1, c0, c1):
    from espnet_b200 import ops

    M, K = a.shape[1], a.shape[2]
    N = b.shape[1]
    ops.gemm(r1 - r0, c1 - c0, K, a, M * K, K, b, N * K, K, out, N, c_plane=M * N, split_out=True, bias=bias, act=ops.ACT_SWISH,
             a_off=r0 * K, b_off=c0 * K, c_off=r0 * N + c0, bias_off=c0, force=mode)


@pytest.mark.parametrize("mode", VERSIONS)
def test_schedule_invariance_bitwise(mode):
    """A GEMM with several column bands (B larger than one band) equals, bit for bit, its four 128-row / 128-column aligned quarters
    computed as separate GEMMs: each quarter keeps 128-column tiles but runs its tiles on other CTAs, in another order."""
    M, N, K = 16000, 3584, 1024   # 125 x 28 tiles: B (28 MiB) is walked in bands of 8 column tiles (8 MiB), the quarters (14 MiB) are not
    r_split, c_split = 64 * 128, 14 * 128
    assert min(r_split // 128, (M - r_split + 127) // 128) * ((min(c_split, N - c_split) + 127) // 128) >= _sms()
    torch.manual_seed(11)
    a, b = _split(torch.randn(M, K, device="cuda")), _split(torch.randn(N, K, device="cuda") / K ** 0.5)
    bias = torch.randn(N, device="cuda")
    whole = torch.full((2, M, N), float("nan"), device="cuda")
    parts = torch.full((2, M, N), float("nan"), device="cuda")
    _sub_gemm(mode, a, b, bias, whole, 0, M, 0, N)
    for r0, r1 in ((0, r_split), (r_split, M)):
        for c0, c1 in ((0, c_split), (c_split, N)):
            _sub_gemm(mode, a, b, bias, parts, r0, r1, c0, c1)
    torch.cuda.synchronize()
    assert not torch.isnan(whole).any()
    assert torch.equal(whole.view(torch.int32), parts.view(torch.int32))


@pytest.mark.parametrize("mode", VERSIONS)
def test_inplace_residual_bitwise(mode):
    """x += 0.5 * (a b^T + bias) in place equals the same GEMM reading a separate copy of x, on more tiles than SMs."""
    from espnet_b200 import ops

    M, N, K = 8000, 512, 512
    assert ((M + 127) // 128) * (N // 128) > _sms()
    torch.manual_seed(12)
    a, b = _split(torch.randn(M, K, device="cuda")), _split(torch.randn(N, K, device="cuda") / K ** 0.5)
    bias, x0 = torch.randn(N, device="cuda"), torch.randn(M, N, device="cuda")
    x = x0.clone()
    ops.linear(a, b, x, bias=bias, residual=x, alpha=0.5, force=mode)
    y = torch.full((M, N), float("nan"), device="cuda")
    ops.linear(a, b, y, bias=bias, residual=x0.clone(), alpha=0.5, force=mode)
    torch.cuda.synchronize()
    assert torch.equal(x.view(torch.int32), y.view(torch.int32))


@pytest.mark.parametrize("mode", VERSIONS + ["simt"])
def test_partial_residual_overlap_refused(mode):
    from espnet_b200 import ops

    M, N, K = 256, 128, 64
    a, b = _split(torch.randn(M, K, device="cuda")), _split(torch.randn(N, K, device="cuda"))
    buf = torch.zeros(M + 1, N, device="cuda")
    with pytest.raises(RuntimeError, match="overlaps"):   # R one row below C: the rows of C are residual rows of other threads
        ops.gemm(M, N, K, a, M * K, K, b, N * K, K, buf, N, R=buf, ldr=N, r_off=N, force=mode)


@pytest.mark.parametrize("mode", VERSIONS)
def test_conv2_and_kob_many_tiles(mode):
    """Implicit-GEMM conv2 (a_mode 1) over more tiles than SMs and the kob-split embed.out behind it, against float64 references."""
    import math

    from espnet_b200 import ops

    torch.manual_seed(13)
    Bn, T2, F2, C, D = 8, 300, 9, 64, 128
    T1h, F1h = T2 + 1, F2 + 1
    assert ((T2 + 127) // 128) * F2 * Bn > _sms()
    s1 = _split(torch.randn(Bn, 4, F1h, T1h, C, device="cuda"))
    c1 = torch.cat([s1[0], s1[1]], dim=1)   # parity planes: hi in 0-3, lo in 4-7
    w2 = torch.randn(C, 9 * C, device="cuda") / (9 * C) ** 0.5
    b2 = torch.randn(C, device="cuda")
    c2 = torch.full((2, Bn, F2, T2, C), float("nan"), device="cuda")
    ops.gemm(T2, C, 9 * C, c1, 0, 0, _split(w2), C * 9 * C, 9 * C, c2, C, c_plane=Bn * F2 * T2 * C, split_out=True, bias=b2, act=ops.ACT_RELU,
             nbx=F2, nby=Bn, sc=(T2 * C, F2 * T2 * C), a_mode=1, conv=(T1h, F1h, C), force=mode)
    full = c1[:, :4].double() + c1[:, 4:].double()   # (B, parity, F1h, T1h, C)
    taps = []
    for kt in range(3):
        for kf in range(3):
            par = (kt & 1) * 2 + (kf & 1)
            taps.append(full[:, par, kf >> 1:(kf >> 1) + F2, kt >> 1:(kt >> 1) + T2, :])
    ref2 = torch.relu(torch.cat(taps, dim=-1) @ w2.double().t() + b2.double())   # (B, F2, T2, C)
    got2 = c2[0].double() + c2[1].double()
    assert (got2 - ref2).abs().max().item() < _tol(mode, 9 * C, 4)
    wo, bo = torch.randn(D, F2 * C, device="cuda") / (F2 * C) ** 0.5, torch.randn(D, device="cuda")
    x = torch.full((Bn * T2, D), float("nan"), device="cuda")
    ops.gemm(T2, D, F2 * C, c2, Bn * F2 * T2 * C, C, _split(wo), D * F2 * C, F2 * C, x, D, bias=bo, alpha=math.sqrt(D), nbx=1, nby=Bn,
             sa=(T2 * C, F2 * T2 * C), sc=(0, T2 * D), kob=C // 32, force=mode)
    a_ref = got2.permute(0, 2, 1, 3).reshape(Bn, T2, F2 * C)
    ref = (a_ref @ wo.double().t() + bo.double()) * math.sqrt(D)
    assert (x.view(Bn, T2, D).double() - ref).abs().max().item() < _tol(mode, F2 * C, 10 * math.sqrt(D))
