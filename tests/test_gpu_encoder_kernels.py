"""-m gpu: the encoder glue kernels (csrc/encoder_ops.cu) one by one, each called through the C ABI on seeded inputs and compared with a
restatement of the same operation written here: float64 for LayerNorm, the softmaxes, the convolution module and the block framing of the
streaming encoder, bit-exact float32 (numpy) for the copies, the tf32 split and q + pos_bias.

Every element a kernel must not read is NaN (frames at or beyond an utterance's length, bd outside the rel-pos band, pe rows nobody asks
for, context rows of other layers) and every output starts as NaN, so a stray read or a missing write fails.  Split outputs (hi plane a
tf32 value, lo plane the remainder) are checked for a hi plane with its 13 low mantissa bits zero, and hi + lo is what is compared.  hi + lo
differs from the fp32 value it splits by less than 2^-20 |y| = 16u |y| (lo keeps 11 of the remainder's up to 14 significant bits), which
every tolerance of a split output includes.  u = 2^-24 throughout.

Tolerances (per element, from the kernel's arithmetic).  test_tolerances_catch_plausible_bugs checks on the CPU that each plausible
LayerNorm, softmax and convolution bug named below moves the float64 reference by more than 10x the tolerance at a tested shape:
* LayerNorm.  Each lane sums ceil(D/32) <= 64 values in sequence, then 5 butterfly levels: the mean is off by <= (D/32 + 5) u mean|x|,
  the variance relatively by about as much, rstd by half that plus 2 ulp; y = (x - mean) rstd g + b adds 3 roundings.
  tol = (D/32 + 8) 4u (|z g| + |g| + |b|) + 16u |y|  with z the float64 standardised value (<= 1.5e-4 at D = 2048, x ~ 2 randn + 0.5).
  Bugs at D = 2048: the last column left out of the statistics moves y by up to 7e-3 (67x the tolerance); the unbiased (D - 1) variance
  by up to 1.5e-3 (11x).
* relpos / masked softmax.  s = (ac + bd) / sqrt(d_k) carries 2u |s|, s - max adds u |s - m|, expf 2 ulp; the row sum adds
  (len/32 + 5) u in sequence and tree; p = e / sum one more rounding.
  tol = p u (8 (max|s| + |m|) + len/32 + 30)  (relative 1.2e-5 at len 2812).
  Bugs at T = 2812: bd read one column off the band, or 1/d_k in place of 1/sqrt(d_k), move p by O(p) (> 1e6x the tolerance); the last
  key dropped moves p by 1/len = 3.6e-4 relatively (900x).
* GLU -> depthwise conv -> BatchNorm -> Swish.  The GLU input is within 4u of its value, the fmaf chain over K taps adds K u sum|w v|,
  the bias and the folded BatchNorm 3 more roundings, swish' <= 1.1 and swish itself 4u.
  tol = 1.1 (|bn_a| ((K + 5) u S + u |acc|) + 2u (|acc bn_a| + |bn_b|)) + 20u |out|,  S = sum_k |w_k v_{t+k}|.
  Bugs at K = 127: a dropped tap moves outputs by up to 0.35 (1e4x the tolerance, which stays below 7e-5); the window one frame late by
  O(1).
* cbe_build_chunks.  Frame rows x scale + pe: at most 2 roundings, tol = 2u (|x| scale + |pe|).  The context vector sums <= block frames in
  sequence: tol = (len + 4) u scale mean|x| + 2u (|pe| + |ref|).  A frame or pe row off by one moves a row by O(1) (randn inputs), and
  the previous block's context vector must match, bit for bit, the one that block wrote.
The copies, q + pos_bias_u / v and the tf32 split are compared bit for bit.
"""
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu

U32 = 2.0 ** -24          # fp32 unit roundoff
NAN = float("nan")
NAN_BITS = np.float32(NAN).view(np.int32)


_KEEP = []    # device copies made inline in a call's argument list: only a raw pointer reaches the library, so keep the tensors alive


@pytest.fixture(autouse=True)
def _release_inputs():
    yield
    if _KEEP:
        torch.cuda.synchronize()
    _KEEP.clear()


def _call(name, *args):
    from espnet_b200.lib import call

    call(name, *args)


def _ptr(t):
    from espnet_b200.lib import ptr

    return ptr(t)


def _dev(a):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    _KEEP.append(t)
    return t


def _i32(a):
    return _dev(np.asarray(a, dtype=np.int32))


def _np(t):
    return t.detach().cpu().numpy()


def _split_np(x):
    """tf32_hi / tf32_lo of common.cuh in numpy float32: hi = x with its 13 low bits cleared, lo = (x - hi) with its 13 low bits cleared."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    hi = (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
    lo = ((x - hi).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
    return hi, lo


def _joined(hi, lo):
    """hi + lo (float64) of a split output, after checking that hi is a tf32 value."""
    assert int((hi.view(torch.int32) & 0x1FFF).abs().max()) == 0, "hi plane has low mantissa bits set"
    return hi.double() + lo.double()


def _same_bits(a, b):
    a = _np(a) if isinstance(a, torch.Tensor) else np.asarray(a)
    b = _np(b) if isinstance(b, torch.Tensor) else np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def _all_nan_bits(t):
    return bool((t.view(torch.int32) == int(NAN_BITS)).all())


def _key_mask(lens, n, device="cuda"):
    """[B][n] bool: column j < lens[b]."""
    return torch.arange(n, device=device).view(1, -1) < torch.as_tensor(lens, device=device).view(-1, 1)


# ============================================================================================================== LayerNorm
LN_D = [64, 144, 255, 256, 257, 512, 1000, 1024, 1025, 1536, 2048]
LN_ROWS = [1, 7, 4096, 4097, 20000]


def _ln_ref(x, g, b, eps=1e-12):
    """float64 LayerNorm (layer_norm.py:12-42): returns y and the standardised z."""
    xd = x.double()
    mu = xd.mean(-1, keepdim=True)
    var = ((xd - mu) ** 2).mean(-1, keepdim=True)
    z = (xd - mu) / torch.sqrt(var + eps)
    return z * g.double() + b.double(), z


def _ln_tol(D, z, g, b, y, split):
    t = (math.ceil(D / 32) + 8) * 4 * U32 * ((z * g.double()).abs() + g.double().abs() + b.double().abs())
    return t + (16 * U32 * y.abs() if split else 0)


def _ln_inputs(rows, D, seed, device="cuda"):
    g = torch.Generator(device=device).manual_seed(seed)
    x = 2 * torch.randn(rows, D, generator=g, device=device) + 0.5
    gamma = 1 + 0.3 * torch.randn(D, generator=g, device=device)
    beta = 0.3 * torch.randn(D, generator=g, device=device)
    return x, gamma, beta


def _ln_run(x, gamma, beta, rows, D, off, plain, split):
    """One call; `off` shifts x and both outputs by one float (4-byte, not 16-byte aligned).  Returns (plain, split) views or None."""
    n = rows * D
    xb = torch.full((n + off,), NAN, device="cuda")
    xb[off:] = x.reshape(-1)
    op = torch.full((n + off + 3,), NAN, device="cuda") if plain else None
    plane = n + 4 + off                      # a multiple of 4 when off == 0: the vector kernel's condition
    os_ = torch.full((off + 2 * plane,), NAN, device="cuda") if split else None
    _call("espb_layernorm_f32", _ptr(xb[off:]), rows, D, _ptr(gamma), _ptr(beta), 1e-12, _ptr(op[off:]) if plain else None,
          _ptr(os_[off:]) if split else None, plane)
    torch.cuda.synchronize()
    res_p = res_s = None
    if plain:
        assert _all_nan_bits(op[:off]) and _all_nan_bits(op[off + n:]), "layernorm wrote outside its plain output"
        res_p = op[off:off + n].view(rows, D)
    if split:
        assert _all_nan_bits(os_[off + n:off + plane]) and _all_nan_bits(os_[off + plane + n:]), "layernorm wrote outside its split planes"
        res_s = (os_[off:off + n].view(rows, D), os_[off + plane:off + plane + n].view(rows, D))
    return res_p, res_s


def _check_layernorm(rows, D, off, seed):
    x, gamma, beta = _ln_inputs(rows, D, seed)
    p_only, _ = _ln_run(x, gamma, beta, rows, D, off, True, False)
    _, s_only = _ln_run(x, gamma, beta, rows, D, off, False, True)
    p_both, s_both = _ln_run(x, gamma, beta, rows, D, off, True, True)
    ref, z = _ln_ref(x, gamma, beta)
    err = (p_only.double() - ref).abs()
    tol = _ln_tol(D, z, gamma, beta, ref, split=False)
    assert bool((err <= tol).all()), f"plain: max err {err.max().item():.3e}, worst err/tol {(err / tol).max().item():.2f}"
    err = (_joined(*s_only) - ref).abs()
    tol = _ln_tol(D, z, gamma, beta, ref, split=True)
    assert bool((err <= tol).all()), f"split: max err {err.max().item():.3e}, worst err/tol {(err / tol).max().item():.2f}"
    # writing one output or both computes the same values, and the split is exactly the split of the plain value
    # (fp32(hi + lo) itself can drop the 2 lowest bits of y: lo is truncated to tf32)
    assert _same_bits(p_only, p_both) and _same_bits(s_only[0], s_both[0]) and _same_bits(s_only[1], s_both[1])
    hi, lo = _split_np(_np(p_both))
    assert _same_bits(s_both[0], hi) and _same_bits(s_both[1], lo)


@gpu
@pytest.mark.parametrize("rows", LN_ROWS)
@pytest.mark.parametrize("D", LN_D)
def test_layernorm_vs_fp64(D, rows):
    """Default dispatch: vec<2/4/8> for D % 4 == 0, D <= 1024 (2 rows per block up to 4096 rows, 8 beyond); scalar<8/16/32/64> otherwise."""
    _check_layernorm(rows, D, 0, seed=D * 7 + rows)


@gpu
@pytest.mark.parametrize("rows", [7, 4097])
@pytest.mark.parametrize("D", LN_D)
def test_layernorm_unaligned_pointers(D, rows):
    """x and the outputs one float past a 16-byte boundary: the scalar kernels for every D."""
    _check_layernorm(rows, D, 1, seed=D * 11 + rows)


@gpu
@pytest.mark.parametrize("D", [0, 2049])
def test_layernorm_refuses_D(D):
    x = torch.zeros(4 * 2100, device="cuda")
    g, b = torch.ones(2100, device="cuda"), torch.zeros(2100, device="cuda")
    out = torch.full((4 * 2100,), NAN, device="cuda")
    with pytest.raises(RuntimeError, match="layernorm: D must be"):
        _call("espb_layernorm_f32", _ptr(x), 4, D, _ptr(g), _ptr(b), 1e-12, _ptr(out), None, 0)
    torch.cuda.synchronize()
    assert _all_nan_bits(out)


# ============================================================================================================== tf32 split
@gpu
@pytest.mark.parametrize("n", [1, 255, 256, 257, 1000, 65537])
def test_split_tf32_bit_exact(n):
    rng = np.random.default_rng(n)
    x = (rng.standard_normal(n) * np.exp(rng.uniform(-30, 30, n))).astype(np.float32)
    special = np.array([0.0, -0.0, 1e-45, -1e-45, 1.17e-38, -2.3e-39, 5.9e-39, 3.4028235e38, -3.4028235e38, 1.0, -1.0 - 2 ** -23,
                        1 + 2 ** -11, 1 + 2 ** -12 + 2 ** -20], dtype=np.float32)   # signed zeros, subnormals, the largest values
    m = min(n, len(special))
    x[:m] = special[:m]
    assert np.isfinite(x).all()
    plane = n + 3
    out = torch.full((2 * plane + 5,), NAN, device="cuda")
    _call("espb_split_tf32_f32", _ptr(_dev(x)), n, _ptr(out), plane)
    torch.cuda.synchronize()
    hi, lo = _split_np(x)
    assert _same_bits(out[:n], hi) and _same_bits(out[plane:plane + n], lo)
    assert _all_nan_bits(out[n:plane]) and _all_nan_bits(out[plane + n:])


# ============================================================================================================== attention glue
def _split_dev(x, gap=0):
    """Split planes of float32 numpy x as one device buffer [2][x.size + gap] and its plane stride."""
    hi, lo = _split_np(x)
    plane = x.size + gap
    buf = np.full(2 * plane, np.nan, dtype=np.float32)
    buf[:x.size], buf[plane:plane + x.size] = hi.ravel(), lo.ravel()
    return _dev(buf), plane


@gpu
@pytest.mark.parametrize("M,D", [(1, 64), (37, 144), (300, 256), (1000, 512)])
def test_qu_qv_bit_exact(M, D):
    rng = np.random.default_rng(M + D)
    q = rng.standard_normal((M, D), dtype=np.float32)
    qkv = np.full((M, 3 * D), np.nan, dtype=np.float32)     # k and v columns must not be read
    qkv[:, :D] = q
    qkv_d, qkv_plane = _split_dev(qkv, gap=7)
    hi, lo = _split_np(qkv)
    pu, pv = rng.standard_normal(D, dtype=np.float32), rng.standard_normal(D, dtype=np.float32)
    out_plane = M * D + 5
    qu = torch.full((2 * out_plane,), NAN, device="cuda")
    qv = torch.full((2 * out_plane,), NAN, device="cuda")
    _call("espb_qu_qv_f32", _ptr(qkv_d), qkv_plane, M, D, _ptr(_dev(pu)), _ptr(_dev(pv)), _ptr(qu), _ptr(qv),
          out_plane)
    torch.cuda.synchronize()
    qj = hi[:, :D] + lo[:, :D]
    for out, p in ((qu, pu), (qv, pv)):
        h, l = _split_np(qj + p)
        assert _same_bits(out[:M * D].view(M, D), h) and _same_bits(out[out_plane:out_plane + M * D].view(M, D), l)
        assert _all_nan_bits(out[M * D:out_plane]) and _all_nan_bits(out[out_plane + M * D:])


@gpu
@pytest.mark.parametrize("D,H,Tp", [(256, 4, 132), (144, 3, 80), (64, 4, 68), (512, 8, 940)])
def test_v_transpose_bit_exact(D, H, Tp):
    """V^T [b][h][dk][Tp] of the split qkv buffer; keys t >= len (also t >= Tmax up to Tp) are 0; d_k = 16, 48, 64."""
    rng = np.random.default_rng(D + Tp)
    lens = [Tp - 5, 1, (Tp * 2) // 3]
    B, Tmax, dk = len(lens), Tp - 3, D // H
    lens[0] = Tmax
    qkv = np.full((B, Tmax, 3 * D), np.nan, dtype=np.float32)   # q and k columns, and v rows t >= len, must not be read
    for b, n in enumerate(lens):
        qkv[b, :n, 2 * D:] = rng.standard_normal((n, D), dtype=np.float32)
    qkv_d, qkv_plane = _split_dev(qkv, gap=4)
    hi, lo = _split_np(qkv)
    vt_plane = B * H * dk * Tp + 9
    vt = torch.full((2 * vt_plane,), NAN, device="cuda")
    _call("espb_v_transpose_f32", _ptr(qkv_d), qkv_plane, B, Tmax, D, H, _ptr(_i32(lens)), _ptr(vt), vt_plane, Tp)
    torch.cuda.synchronize()
    v = np.zeros((B, Tp, D), dtype=np.float32)
    for b, n in enumerate(lens):
        v[b, :n] = hi[b, :n, 2 * D:] + lo[b, :n, 2 * D:]
    ref = v.reshape(B, Tp, H, dk).transpose(0, 2, 3, 1)
    h, l = _split_np(ref)
    n = B * H * dk * Tp
    assert _same_bits(vt[:n].view(B, H, dk, Tp), h) and _same_bits(vt[vt_plane:vt_plane + n].view(B, H, dk, Tp), l)
    assert _all_nan_bits(vt[n:vt_plane]) and _all_nan_bits(vt[vt_plane + n:])


def _softmax_ref(s, lens):
    """float64 masked softmax over the last axis (attention.py:121-151) of s [B][H][T][T'] with keys j >= lens[b] masked; p, max."""
    B, _, _, Tk = s.shape
    km = _key_mask(lens, Tk, s.device).view(B, 1, 1, Tk)
    s = torch.where(km, s, torch.tensor(-math.inf, dtype=s.dtype, device=s.device))
    m = s.max(-1, keepdim=True).values
    e = torch.exp(s - m)
    return e / e.sum(-1, keepdim=True), torch.where(km, s, torch.zeros((), dtype=s.dtype, device=s.device)), m


def _softmax_tol(p, s, m, lens):
    B = p.shape[0]
    ln = torch.as_tensor(lens, device=p.device, dtype=torch.float64).view(B, 1, 1, 1)
    smax = s.abs().max(-1, keepdim=True).values
    return p * U32 * (8 * (smax + m.abs()) + ln / 32 + 30)


def _check_probs(probs, plane, B, H, T, Tp, lens, ref, s, m, what):
    n = B * H * T * Tp
    assert _all_nan_bits(probs[n:plane]) and _all_nan_bits(probs[plane + n:]), f"{what}: wrote outside its output"
    hi, lo = probs[:n].view(B, H, T, Tp), probs[plane:plane + n].view(B, H, T, Tp)
    km = _key_mask(lens, Tp).view(B, 1, 1, Tp).expand(B, H, T, Tp)
    assert bool((hi[~km] == 0).all()) and bool((lo[~km] == 0).all()), f"{what}: columns >= len not exactly 0"
    assert not bool(hi.view(torch.int32)[~km].ne(0).any()), f"{what}: -0 in a masked column"
    got = _joined(hi, lo)[..., :T]
    err = (got - ref).abs()
    tol = _softmax_tol(ref, s, m, lens)
    assert bool((err <= tol).all()), f"{what}: max err {err.max().item():.3e}, worst err/tol {(err / tol).nan_to_num(1e9).max().item():.2f}"


def _relpos_inputs(T, Tp, Rp, lens, H, seed):
    """ac [B][H][T][Tp] NaN at keys >= len; bd [B][H][T][Rp] NaN everywhere but the band columns T-1-i+j, j < len, of row i."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    B = len(lens)
    ac = 6 * torch.randn(B, H, T, Tp, generator=g, device="cuda")
    ac.masked_fill_(~_key_mask(lens, Tp).view(B, 1, 1, Tp), NAN)
    bd = 6 * torch.randn(B, H, T, Rp, generator=g, device="cuda")
    j = torch.arange(Rp, device="cuda").view(1, Rp) - (T - 1 - torch.arange(T, device="cuda").view(T, 1))   # key of column c in row i
    ln = torch.as_tensor(lens, device="cuda").view(B, 1, 1, 1)
    bd.masked_fill_(~((j >= 0).view(1, 1, T, Rp) & (j.view(1, 1, T, Rp) < ln)), NAN)
    return ac, bd


def _relpos_ref(ac, bd, T, lens, sqrt_dk, shift=0):
    """rel_shift (attention.py:391-414: key j of query i reads bd column T-1-i+j), / sqrt(d_k), masked softmax -- float64."""
    B, H, _, _ = ac.shape
    idx = (T - 1 - torch.arange(T, device=ac.device).view(T, 1) + torch.arange(T, device=ac.device).view(1, T) + shift).clamp(0, bd.shape[-1] - 1)
    bds = bd.double().gather(-1, idx.view(1, 1, T, T).expand(B, H, T, T))
    return _softmax_ref((ac[..., :T].double() + bds) / sqrt_dk, lens)


def _ragged(T):
    """Key lengths of a ragged batch: the whole T, two thirds of it, and a single key."""
    return [T, max(1, (2 * T) // 3), 1] if T > 1 else [1]


def _check_relpos(T, Tp, lens, H, seed, dk=64):
    B, Rp = len(lens), 2 * T - 1 + 3
    ac, bd = _relpos_inputs(T, Tp, Rp, lens, H, seed)
    plane = B * H * T * Tp + 12
    probs = torch.full((2 * plane,), NAN, device="cuda")
    _call("espb_relpos_softmax_f32", _ptr(ac), _ptr(bd), B, H, T, Tp, Rp, _ptr(_i32(lens)), math.sqrt(dk), _ptr(probs), plane)
    torch.cuda.synchronize()
    ref, s, m = _relpos_ref(ac, bd, T, lens, math.sqrt(dk))
    _check_probs(probs, plane, B, H, T, Tp, lens, ref, s, m, f"relpos T {T} Tp {Tp}")


# T <= 128: register kernel <4>; 128 < T, Tp <= 1536 (Tp % 4 == 0, aligned): shared-memory kernel; Tp > 1536: three-pass kernel.
@gpu
@pytest.mark.parametrize("T", [1, 37, 128, 129, 300, 937, 1536, 1537, 2812])
def test_relpos_softmax_vs_fp64(T):
    Tp = (T + 3) // 4 * 4
    _check_relpos(T, Tp, _ragged(T), H=2, seed=T)


@gpu
@pytest.mark.parametrize("T", [129, 300, 937])
def test_relpos_softmax_three_pass(T):
    """The three-pass kernel at lengths the shared-memory kernel would take, through a Tp that is not a multiple of 4."""
    _check_relpos(T, T + 1, _ragged(T), H=2, seed=T + 1)


def _check_masked(T, Tp, lens, H, seed, dk=64):
    B = len(lens)
    g = torch.Generator(device="cuda").manual_seed(seed)
    sc = 8 * torch.randn(B, H, T, Tp, generator=g, device="cuda")
    sc.masked_fill_(~_key_mask(lens, Tp).view(B, 1, 1, Tp), NAN)
    plane = B * H * T * Tp + 12
    probs = torch.full((2 * plane,), NAN, device="cuda")
    _call("espb_masked_softmax_f32", _ptr(sc), B, H, T, Tp, _ptr(_i32(lens)), math.sqrt(dk), _ptr(probs), plane)
    torch.cuda.synchronize()
    ref, s, m = _softmax_ref(sc[..., :T].double() / math.sqrt(dk), lens)
    _check_probs(probs, plane, B, H, T, Tp, lens, ref, s, m, f"masked T {T} Tp {Tp}")


@gpu
@pytest.mark.parametrize("T,Tp", [(1, 4), (37, 40), (42, 42), (42, 44), (128, 128), (129, 131), (937, 940), (2812, 2812)])
def test_masked_softmax_vs_fp64(T, Tp):
    """42 = block + 2: the streaming encoder's chunk (block 40 framed by two context tokens)."""
    _check_masked(T, Tp, _ragged(T), H=3, seed=T + Tp)


# ============================================================================================================== row helpers
@gpu
@pytest.mark.parametrize("nplanes", [1, 2])
@pytest.mark.parametrize("lens", [[50, 50], [1, 50, 17], [50]])
def test_zero_pad_rows_bit_exact(lens, nplanes):
    rng = np.random.default_rng(len(lens) * 10 + nplanes)
    B, Tmax, D = len(lens), 50, 144
    plane = B * Tmax * D + 6
    x = rng.standard_normal(nplanes * plane + 3).astype(np.float32)
    for q in range(nplanes):
        for b, n in enumerate(lens):
            x[q * plane + (b * Tmax + n) * D:q * plane + (b + 1) * Tmax * D] = np.nan   # pad rows: must become 0, never be read
    xd = _dev(x)
    _call("espb_zero_pad_rows_f32", _ptr(xd), B, Tmax, D, _ptr(_i32(lens)), plane, nplanes)
    torch.cuda.synchronize()
    ref = x.copy()
    for q in range(nplanes):
        for b, n in enumerate(lens):
            ref[q * plane + (b * Tmax + n) * D:q * plane + (b + 1) * Tmax * D] = 0.0
    assert _same_bits(xd, ref)


@gpu
@pytest.mark.parametrize("row0,every,count,nplanes", [(0, 42, 5, 1), (41, 42, 5, 2), (3, 1, 7, 2), (0, 42, 0, 1)])
def test_zero_rows_bit_exact(row0, every, count, nplanes):
    rng = np.random.default_rng(row0 + every + count)
    rows, D = 220, 256
    plane = rows * D + 4
    x = rng.standard_normal(nplanes * plane + 2).astype(np.float32)
    xd = _dev(x)
    _call("espb_zero_rows_f32", _ptr(xd), row0, every, count, D, plane, nplanes)
    torch.cuda.synchronize()
    ref = x.copy()
    for q in range(nplanes):
        for k in range(count):
            r = row0 + k * every
            ref[q * plane + r * D:q * plane + (r + 1) * D] = 0.0
    assert _same_bits(xd, ref)


@gpu
@pytest.mark.parametrize("N,D", [(1, 64), (3, 256), (2, 520)])
def test_gather_rows_bit_exact(N, D):
    rng = np.random.default_rng(N * D)
    src_rows, idx = 30, np.array([0, 29, 5, 5, 17, 1, 28], dtype=np.int32)
    src = np.full((N, src_rows, D), np.nan, dtype=np.float32)
    for r in set(idx.tolist()):
        src[:, r] = rng.standard_normal((N, D), dtype=np.float32)    # rows nobody gathers stay NaN
    nout = len(idx)
    out = torch.full((N * nout * D + 5,), NAN, device="cuda")
    _call("espb_gather_rows_f32", _ptr(_dev(src)), N, src_rows, _ptr(_i32(idx)), nout, D, _ptr(out))
    torch.cuda.synchronize()
    assert _same_bits(out[:N * nout * D].view(N, nout, D), src[:, idx])
    assert _all_nan_bits(out[N * nout * D:])


# ============================================================================================================== contextual block processing
@gpu
@pytest.mark.parametrize("N,nb,layer,L,past", [(1, 1, 0, 1, False), (2, 4, 2, 3, True), (3, 5, 0, 2, False), (2, 1, 1, 2, True)])
def test_cbe_ctx_propagate_bit_exact(N, nb, layer, L, past):
    """layer = L - 1 is the last layer; past_ctx rows of other layers are NaN (must not be read), next_ctx rows of other layers kept."""
    rng = np.random.default_rng(N * 100 + nb * 10 + layer)
    S, D = 42, 256
    x = rng.standard_normal((N, nb, S, D), dtype=np.float32)
    x[:, :, 0] = np.nan                    # token 0 is overwritten, never read
    pc = np.full((N, L, D), np.nan, dtype=np.float32)
    pc[:, layer] = rng.standard_normal((N, D), dtype=np.float32)
    nc0 = rng.standard_normal((N, L, D), dtype=np.float32)
    xd, ncd = _dev(x), _dev(nc0)
    _call("espb_cbe_ctx_propagate_f32", _ptr(xd), N, nb, S, D, _ptr(_dev(pc)) if past else None, _ptr(ncd), layer, L)
    torch.cuda.synchronize()
    ref = x.copy()
    ref[:, 1:, 0] = x[:, :-1, S - 1]
    ref[:, 0, 0] = pc[:, layer] if past else x[:, 0, S - 1]
    nref = nc0.copy()
    nref[:, layer] = x[:, nb - 1, S - 1]
    assert _same_bits(xd, ref) and _same_bits(ncd, nref)


def _cbe_ref(xs, nb, block, hop, pe, pos0, ctx0, scale, prev):
    """contextual_block_conformer_encoder.py:506-541 in float64: per block the previous context vector, the positionally encoded frames
    (zero rows past a trailing partial block), and this block's context vector pos_enc(mean of its frames, ctx0 + i)."""
    N, Tt, D = xs.shape
    x, p = xs.astype(np.float64), pe.astype(np.float64)
    S = block + 2
    ch = np.zeros((N, nb, S, D))
    addin = np.zeros((N, nb, D))
    lens = []
    for i in range(nb):
        cur = i * hop
        n = min(block, Tt - cur)
        lens.append(n)
        ch[:, i, 1:1 + n] = x[:, cur:cur + n] * scale + p[pos0 + cur:pos0 + cur + n]
        addin[:, i] = x[:, cur:cur + n].mean(1) * scale + p[ctx0 + i]
        ch[:, i, S - 1] = addin[:, i]
        ch[:, i, 0] = addin[:, i - 1] if i else (prev.astype(np.float64) if prev is not None else addin[:, 0])
    return ch, addin[:, nb - 1], lens


CBE_CASES = [   # N, Tt, D, block, hop, nb, pos0, ctx0, prev_addin
    (1, 40, 64, 40, 16, 1, 0, 0, False),        # one whole block
    (2, 7, 512, 40, 16, 1, 12, 3, True),        # one partial block
    (3, 100, 256, 40, 16, 5, 37, 5, True),      # trailing partial block (36 frames)
    (2, 88, 64, 40, 16, 4, 0, 0, False),        # blocks end exactly at Tt
    (2, 66, 512, 20, 8, 7, 160, 11, False),     # last block of 18 frames
]


@gpu
@pytest.mark.parametrize("N,Tt,D,block,hop,nb,pos0,ctx0,prev", CBE_CASES)
def test_cbe_build_chunks_vs_fp64(N, Tt, D, block, hop, nb, pos0, ctx0, prev):
    rng = np.random.default_rng(Tt * D + nb)
    xs = rng.standard_normal((N, Tt, D), dtype=np.float32)
    P = max(pos0 + Tt, ctx0 + nb) + 10
    pe = np.full((P, D), np.nan, dtype=np.float32)    # pe rows no frame or context vector asks for stay NaN
    pe[pos0:pos0 + Tt] = rng.standard_normal((Tt, D), dtype=np.float32)
    pe[ctx0:ctx0 + nb] = rng.standard_normal((nb, D), dtype=np.float32)
    pa = rng.standard_normal((N, D), dtype=np.float32) if prev else None
    scale = math.sqrt(D)
    S = block + 2
    chunks = torch.full((N * nb * S * D + 7,), NAN, device="cuda")
    addin = torch.full((N * D + 3,), NAN, device="cuda")
    _call("espb_cbe_build_chunks_f32", _ptr(_dev(xs)), N, Tt, D, nb, block, hop, _ptr(_dev(pe)), pos0, ctx0,
          scale, _ptr(_dev(pa)) if prev else None, _ptr(addin), _ptr(chunks))
    torch.cuda.synchronize()
    assert _all_nan_bits(chunks[N * nb * S * D:]) and _all_nan_bits(addin[N * D:])
    got = _np(chunks[:N * nb * S * D]).reshape(N, nb, S, D)
    ref, aref, lens = _cbe_ref(xs, nb, block, hop, pe, pos0, ctx0, scale, pa)
    pe64 = np.abs(pe.astype(np.float64))
    for i, n in enumerate(lens):
        cur = i * hop
        fr = np.abs(got[:, i, 1:1 + n] - ref[:, i, 1:1 + n])
        tol = 2 * U32 * (np.abs(xs[:, cur:cur + n].astype(np.float64)) * scale + pe64[pos0 + cur:pos0 + cur + n])
        assert (fr <= tol).all(), f"block {i}: frame rows max err {fr.max():.3e}"
        assert not got[:, i, 1 + n:S - 1].view(np.int32).any(), f"block {i}: pad rows not exactly 0"
        ctol = (n + 4) * U32 * scale * np.abs(xs[:, cur:cur + n].astype(np.float64)).mean(1) + 2 * U32 * (pe64[ctx0 + i] + np.abs(ref[:, i, S - 1]))
        assert (np.abs(got[:, i, S - 1] - ref[:, i, S - 1]) <= ctol).all(), f"block {i}: context vector"
        if i:   # the previous context vector is recomputed in the same order: bit-identical to what block i - 1 wrote
            assert _same_bits(got[:, i, 0], got[:, i - 1, S - 1])
    assert _same_bits(got[:, 0, 0], pa if prev else got[:, 0, S - 1])
    assert _same_bits(addin[:N * D].view(N, D), got[:, nb - 1, S - 1])
    assert np.abs(_np(addin[:N * D]).reshape(N, D) - aref).max() < 1e-3


@gpu
def test_cbe_build_chunks_refuses_bad_shape():
    xs = torch.zeros(40 * 64, device="cuda")
    chunks = torch.full((2 * 42 * 64,), NAN, device="cuda")
    with pytest.raises(RuntimeError, match="cbe_build_chunks: bad shape"):   # block 2 would start at frame 32 >= Tt = 30
        _call("espb_cbe_build_chunks_f32", _ptr(xs), 1, 30, 64, 3, 40, 16, _ptr(xs), 0, 0, 8.0, None, _ptr(xs), _ptr(chunks))
    torch.cuda.synchronize()
    assert _all_nan_bits(chunks)


# ============================================================================================================== convolution module
DW_LENS = [200, 1, 77]     # Tmax 200 (not a multiple of the 64-frame tile), a 1-frame utterance, a ragged one


def _dw_inputs(B, Tmax, C, K, lens, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    y = torch.randn(B, Tmax, 2 * C, generator=g, device="cuda")
    y.masked_fill_(~_key_mask(lens, Tmax).view(B, Tmax, 1), NAN)     # frames t >= len must not be read
    w = torch.randn(C, K, generator=g, device="cuda") / math.sqrt(K)
    db = 0.3 * torch.randn(C, generator=g, device="cuda")
    ba = 1 + 0.3 * torch.randn(C, generator=g, device="cuda")
    bb = 0.3 * torch.randn(C, generator=g, device="cuda")
    return y, w, db, ba, bb


def _dw_run(y, w, db, ba, bb, lens):
    B, Tmax, C2 = y.shape
    C, K = w.shape
    plane = B * Tmax * C + 8
    out = torch.full((2 * plane,), NAN, device="cuda")
    _call("espb_glu_dwconv_bn_swish_f32", _ptr(y), B, Tmax, C, _ptr(_i32(lens)), _ptr(w), _ptr(db), K, _ptr(ba), _ptr(bb), _ptr(out), plane)
    torch.cuda.synchronize()
    n = B * Tmax * C
    assert _all_nan_bits(out[n:plane]) and _all_nan_bits(out[plane + n:]), "dwconv wrote outside its output"
    return out[:n].view(B, Tmax, C), out[plane:plane + n].view(B, Tmax, C)


def _dw_ref(y, w, db, ba, bb, lens):
    """convolution.py:56-79 in float64: GLU over channels, depthwise conv zero-padded at the utterance's own ends, BatchNorm folded to
    x a + b, Swish; rows t >= len are 0.  Also returns S = sum_k |w_k v_{t+k}| and the conv output for the tolerance."""
    import torch.nn.functional as F

    B, Tmax, C2 = y.shape
    C, K = w.shape
    km = _key_mask(lens, Tmax, y.device).view(B, Tmax, 1)
    yd = torch.where(km, y.double(), torch.zeros((), dtype=torch.float64, device=y.device))
    v = yd[..., :C] * torch.sigmoid(yd[..., C:])
    conv = lambda a, ww: F.conv1d(a.transpose(1, 2), ww.view(C, 1, K), padding=(K - 1) // 2, groups=C).transpose(1, 2)
    acc = conv(v, w.double()) + db.double()
    S = conv(v.abs(), w.double().abs())
    z = acc * ba.double() + bb.double()
    out = torch.where(km, z * torch.sigmoid(z), torch.zeros((), dtype=torch.float64, device=y.device))
    return out, acc, S


def _dw_tol(K, ref, acc, S, ba, bb):
    a, b = ba.double().abs(), bb.double().abs()
    return 1.1 * (a * ((K + 5) * U32 * S + U32 * acc.abs()) + 2 * U32 * (acc.abs() * a + b)) + 20 * U32 * ref.abs()


@gpu
@pytest.mark.parametrize("C", [64, 144, 512])
@pytest.mark.parametrize("K", [1, 3, 7, 15, 31, 33, 63, 65, 127])
def test_glu_dwconv_bn_swish_vs_fp64(K, C):
    """K = 15 / 31: the register-window kernels; every other odd K: the generic tile kernel (K >= 65 needs more than 48 KB of shared memory)."""
    B, Tmax = len(DW_LENS), max(DW_LENS)
    y, w, db, ba, bb = _dw_inputs(B, Tmax, C, K, DW_LENS, seed=K * 1000 + C)
    hi, lo = _dw_run(y, w, db, ba, bb, DW_LENS)
    ref, acc, S = _dw_ref(y, w, db, ba, bb, DW_LENS)
    got = _joined(hi, lo)
    km = _key_mask(DW_LENS, Tmax).view(B, Tmax, 1).expand(B, Tmax, C)
    assert not bool(hi.view(torch.int32)[~km].ne(0).any()) and not bool(lo.view(torch.int32)[~km].ne(0).any()), "rows t >= len not exactly 0"
    err = (got - ref).abs()
    tol = _dw_tol(K, ref, acc, S, ba, bb)
    assert bool((err <= tol).all()), f"max err {err.max().item():.3e}, worst err/tol {(err / tol).max().item():.2f}"


@gpu
@pytest.mark.parametrize("K", [2, 0, 129])
def test_glu_dwconv_refuses_kernel_size(K):
    y = torch.zeros(64 * 128, device="cuda")
    out = torch.full((2 * 64 * 64,), NAN, device="cuda")
    with pytest.raises(RuntimeError, match="odd and <= 127"):
        _call("espb_glu_dwconv_bn_swish_f32", _ptr(y), 1, 64, 64, _ptr(_i32([64])), _ptr(y), _ptr(y), K, _ptr(y), _ptr(y), _ptr(out), 64 * 64)
    torch.cuda.synchronize()
    assert _all_nan_bits(out)


@gpu
@pytest.mark.parametrize("kernel", [7, 65])
def test_conformer_other_kernel_sizes_vs_oracle(kernel):
    """A Conformer whose convolution module has no register-window kernel (7) or needs more than 48 KB of shared memory (65), end to end."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import oracle
    from gpu_util import random_weights, refbuild, speech2text
    from test_gpu_pipeline import _maxerr, enc_tol

    cfg = dict(d_model=64, heads=4, ff=128, enc_layers=2, dec_layers=1, vocab=50, kernel=kernel)
    w = random_weights(cfg, seed=kernel)
    s2t = speech2text(cfg, w, beam_size=2, ctc_weight=0.3)
    o = oracle.OracleSpeech2Text(cfg, w, beam_size=2, ctc_weight=0.3)
    lens = [24000, 9000]
    waves = [refbuild.waveform(70 + i, n) for i, n in enumerate(lens)]
    speech, sl = s2t._to_batch(waves)
    enc, elens = s2t.asr_model.encode(speech, sl)
    for i, wv in enumerate(waves):
        ref = o.encode(wv)
        assert int(elens[i]) == ref.shape[0]
        assert _maxerr(enc[i, :ref.shape[0]], ref) < enc_tol()


def test_conformer_encoders_refuse_unsupported_kernel_sizes():
    import espnet_b200

    for k in (30, 129, 0):
        with pytest.raises(NotImplementedError, match=f"cnn_module_kernel={k}"):
            espnet_b200.ConformerEncoder(80, 64, rel_pos_type="latest", macaron_style=True, cnn_module_kernel=k)
        with pytest.raises(NotImplementedError, match=f"cnn_module_kernel={k}"):
            espnet_b200.ContextualBlockConformerEncoder(80, 64, cnn_module_kernel=k)


# ============================================================================================================== tolerance checks
def _max_over_tol(bugged, ref, tol):
    return ((bugged - ref).abs() / tol).max().item()


def test_tolerances_catch_plausible_bugs():
    """On the CPU, from the float64 references above: each plausible bug named in the module docstring moves the reference by more than
    10x the tolerance the GPU tests use at the tested shapes (so those tests would catch it)."""
    g = torch.Generator().manual_seed(0)
    # LayerNorm, D = 2048: the last column left out of the statistics; the unbiased variance
    D = 2048
    x, gamma, beta = _ln_inputs(64, D, 0, device="cpu")
    ref, z = _ln_ref(x, gamma, beta)
    tol = _ln_tol(D, z, gamma, beta, ref, split=True)
    xd = x.double()
    mu = xd[:, :-1].mean(-1, keepdim=True)
    var = ((xd[:, :-1] - mu) ** 2).mean(-1, keepdim=True)
    assert _max_over_tol((xd - mu) / torch.sqrt(var + 1e-12) * gamma.double() + beta.double(), ref, tol) > 10
    assert _max_over_tol(z * math.sqrt(D / (D - 1)) * gamma.double() + beta.double(), ref, tol) > 10
    # relpos softmax at T = 2812: band off by one column, 1/d_k for 1/sqrt(d_k), last key dropped
    T, dk = 2812, 64
    lens = [T]
    ac = 6 * torch.randn(1, 1, T, T, generator=g, dtype=torch.float64)
    bd = 6 * torch.randn(1, 1, T, 2 * T - 1, generator=g, dtype=torch.float64)
    ref, s, m = _relpos_ref(ac, bd, T, lens, math.sqrt(dk))
    ref, s, m = ref.to("cpu"), s.to("cpu"), m.to("cpu")
    B = 1
    ln = torch.tensor(lens, dtype=torch.float64).view(B, 1, 1, 1)
    tol = ref * U32 * (8 * (s.abs().max(-1, keepdim=True).values + m.abs()) + ln / 32 + 30)
    rows = slice(T // 2, T // 2 + 8)     # the shifted band reads a defined column in the middle rows
    shifted, _, _ = _relpos_ref(ac, bd, T, lens, math.sqrt(dk), shift=1)
    assert _max_over_tol(shifted[..., rows, :], ref[..., rows, :], tol[..., rows, :]) > 10
    assert _max_over_tol(_relpos_ref(ac, bd, T, lens, dk)[0], ref, tol) > 10
    assert _max_over_tol(_relpos_ref(ac, bd, T, [T - 1], math.sqrt(dk))[0][..., :T - 1], ref[..., :T - 1], tol[..., :T - 1]) > 10
    # convolution module, K = 127: the last tap dropped; the window one frame late
    K, C, Tmax = 127, 64, 200
    y = torch.randn(1, Tmax, 2 * C, generator=g)
    w = torch.randn(C, K, generator=g) / math.sqrt(K)
    db, ba, bb = 0.3 * torch.randn(C, generator=g), 1 + 0.3 * torch.randn(C, generator=g), 0.3 * torch.randn(C, generator=g)
    ref, acc, S = _dw_ref(y, w, db, ba, bb, [Tmax])
    tol = _dw_tol(K, ref, acc, S, ba, bb)
    w_drop = w.clone()
    w_drop[:, -1] = 0
    assert _max_over_tol(_dw_ref(y, w_drop, db, ba, bb, [Tmax])[0], ref, tol) > 10
    late = torch.cat([torch.zeros(1, 1, 2 * C), y[:, :-1]], 1)
    assert _max_over_tol(_dw_ref(late, w, db, ba, bb, [Tmax])[0], ref, tol) > 10
