"""The tensor-core GEMM's epilogue, which runs on its own warps from a shared-memory staging buffer while the consumer warpgroups start the
next tile: every epilogue option at shapes with at least 3 tiles per CTA, for 128- and 64-column tiles.  Each whole GEMM is compared bit
for bit with aligned sub-GEMMs launched separately (other CTAs, other tile order, other staging-buffer turns), and against a float64
reference, so a race on the staging buffer, a tile stored at another tile's position or a scrambled staging layout all fail."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
VERSIONS = ["tc", "tc2"]
K = 256   # 8 k-blocks: two promotion chunks in tc2


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _split(x):
    from espnet_b200 import ops

    return ops.split_from(x)


# width -> (M, N, row split, column split or None).  128: N > 64 and every quarter keeps at least SM-count 128-column tiles; 64: N <= 64.
SHAPES = {128: (16000, 1024, 64 * 128, 512), 64: (60000, 64, 235 * 128, None)}

CASES = {
    "bias": dict(act="none"),
    "bias_relu": dict(act="relu"),
    "bias_swish": dict(act="swish"),
    "bias_gelu": dict(act="gelu"),
    "alpha": dict(act="none", alpha=0.37),
    "residual_inplace": dict(act="none", alpha=0.5, residual="inplace"),
    "residual_disjoint": dict(act="swish", alpha=1.5, residual="disjoint"),
    "split_out": dict(act="swish", split=True),
    "odd_ldc": dict(act="relu", ldc_pad=1, residual="disjoint", split=True),
    "ragged": dict(act="gelu", ragged=True, residual="inplace", alpha=0.25),
}


def _act(name):
    from espnet_b200 import ops

    return {"none": ops.ACT_NONE, "relu": ops.ACT_RELU, "swish": ops.ACT_SWISH, "gelu": ops.ACT_GELU}[name]


def _ref_act(x, name):
    if name == "relu":
        return torch.relu(x)
    if name == "swish":
        return x * torch.sigmoid(x)
    if name == "gelu":
        return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))
    return x


def _check_tiles(M, N, width):
    tiles = ((M + 127) // 128) * ((N + width - 1) // width)
    assert tiles >= 3 * _sms(), (M, N, width, tiles)


@pytest.mark.parametrize("mode", VERSIONS)
@pytest.mark.parametrize("width", [128, 64])
@pytest.mark.parametrize("case", sorted(CASES))
def test_epilogue_bitwise(mode, width, case):
    from espnet_b200 import ops

    opt = CASES[case]
    M, N, r_split, c_split = SHAPES[width]
    if opt.get("ragged"):
        M, N = M - 37, N - 3   # ragged last row block; N not a multiple of 8 (nor of 4)
    _check_tiles(M, N, width)
    ldc = (SHAPES[width][1] if opt.get("ragged") else N) + opt.get("ldc_pad", 0)
    split, alpha, act, res = opt.get("split", False), opt.get("alpha", 1.0), opt["act"], opt.get("residual")
    torch.manual_seed(width + sorted(CASES).index(case))
    a32, b32 = torch.randn(M, K, device="cuda"), torch.randn(N, K, device="cuda") / K ** 0.5
    a, b = _split(a32), _split(b32)
    bias = torch.randn(N, device="cuda")
    planes = 2 if split else 1
    x0 = torch.randn(planes, M, ldc, device="cuda")
    r_dis = torch.randn(M, N, device="cuda") if res == "disjoint" else None

    def run(out, r0, r1, c0, c1):
        R, ldr, r_off = None, 0, 0
        if res == "inplace":
            R, ldr, r_off = out, ldc, r0 * ldc + c0
        elif res == "disjoint":
            R, ldr, r_off = r_dis, N, r0 * N + c0
        ops.gemm(r1 - r0, c1 - c0, K, a, M * K, K, b, N * K, K, out, ldc, c_plane=M * ldc if split else 0, split_out=split, bias=bias,
                 R=R, ldr=ldr, alpha=alpha, act=_act(act), a_off=r0 * K, b_off=c0 * K, c_off=r0 * ldc + c0, r_off=r_off, bias_off=c0,
                 force=mode)

    def fresh():
        out = torch.full((planes, M, ldc), float("nan"), device="cuda")
        if res == "inplace":   # the residual is the output window itself (plane 0: split output is not combined with in-place R)
            out[0, :, :N] = x0[0, :, :N]
        return out

    if res == "inplace":
        assert not split
    whole, parts = fresh(), fresh()
    run(whole, 0, M, 0, N)
    col_splits = ((0, N),) if c_split is None else ((0, c_split), (c_split, N))
    for r0, r1 in ((0, r_split), (r_split, M)):
        for c0, c1 in col_splits:
            run(parts, r0, r1, c0, c1)
    torch.cuda.synchronize()
    assert not torch.isnan(whole[:, :, :N]).any()
    assert torch.isnan(whole[:, :, N:]).all()   # the padding columns of ldc are never written
    assert torch.equal(whole.view(torch.int32), parts.view(torch.int32)), f"{mode} width {width} {case}: whole != aligned parts"

    ref = (a[0].double() + a[1].double()) @ (b[0].double() + b[1].double()).t() + bias.double()
    ref = _ref_act(ref, act) * alpha
    if res == "inplace":
        ref = ref + x0[0, :, :N].double()
    elif res == "disjoint":
        ref = ref + r_dis.double()
    got = whole[:, :, :N].double().sum(dim=0)
    err = (got - ref).abs().max().item()
    assert err < 1e-4 * max(1.0, alpha) * 4, f"{mode} width {width} {case}: max abs err {err}"
    if split:   # hi plane is tf32-rounded: its low 13 mantissa bits are 0
        assert ((whole[0, :, :N].view(torch.int32) & 0x1FFF) == 0).all()


@pytest.mark.parametrize("mode", VERSIONS)
@pytest.mark.parametrize("width", [128, 64])
def test_epilogue_batch_slices_bitwise(mode, width):
    """nbx x nby batch slices with per-slice A, B, bias (batch-x only), disjoint residual and output windows inside padded slices equal,
    bit for bit, the same slices computed one GEMM each."""
    from espnet_b200 import ops

    nbx, nby = 2, 2
    nb = nbx * nby
    M, N = (4224, 512) if width == 128 else (15000, 60)   # 128: 33 x 4 = 132 tiles per slice, so a lone slice keeps 128-column tiles
    assert ((M + 127) // 128) * ((N + width - 1) // width) * nb >= 3 * _sms()
    if width == 128:
        assert ((M + 127) // 128) * ((N + 127) // 128) >= _sms()
    Mp, ldc = M + 64, N + 4
    torch.manual_seed(width)
    a, b = _split(torch.randn(nb, M, K, device="cuda")), _split(torch.randn(nb, N, K, device="cuda") / K ** 0.5)
    bias, R = torch.randn(nbx, N, device="cuda"), torch.randn(nb, M, N, device="cuda")
    whole = torch.full((nb, Mp, ldc), float("nan"), device="cuda")
    parts = torch.full((nb, Mp, ldc), float("nan"), device="cuda")
    ops.gemm(M, N, K, a, nb * M * K, K, b, nb * N * K, K, whole, ldc, bias=bias, sbias_x=N, R=R, ldr=N, alpha=0.75, act=ops.ACT_SWISH,
             nbx=nbx, nby=nby, sa=(M * K, nbx * M * K), sb=(N * K, nbx * N * K), sc=(Mp * ldc, nbx * Mp * ldc), sr=(M * N, nbx * M * N),
             force=mode)
    for z in range(nb):
        ops.gemm(M, N, K, a, nb * M * K, K, b, nb * N * K, K, parts, ldc, bias=bias, bias_off=(z % nbx) * N, R=R, ldr=N, alpha=0.75,
                 act=ops.ACT_SWISH, a_off=z * M * K, b_off=z * N * K, c_off=z * Mp * ldc, r_off=z * M * N, force=mode)
    torch.cuda.synchronize()
    assert not torch.isnan(whole[:, :M, :N]).any()
    assert torch.isnan(whole[:, M:]).all() and torch.isnan(whole[:, :, N:]).all()
    assert torch.equal(whole.view(torch.int32), parts.view(torch.int32))
