"""-m gpu: the fused wgmma self-attention kernel (csrc/attention.cu, espb_flash_attn_f32) against a float64 restatement of
RelPositionMultiHeadedAttention / MultiHeadedAttention (attention.py:416-459, 391-414, 121-151) on seeded inputs, called through the C ABI
in the two forms the encoders use:
* rel-pos (layers.py: _relpos_attn): q = q + pos_bias_u, its own split [M][D] buffer (ldq = D); k from the fused q|k|v buffer (k_off = D,
  ldk = 3D); bd [B][H][T][Rp], Rp = 2T - 1 rounded up to 32, the unshifted (q + pos_bias_v) p^T;
* plain (layers.py: _attn, the Transformer encoder): q and k both from q|k|v (q_off 0, k_off D, ldq = ldk = 3D) and no bd.
V reaches the kernel as the V^T planes written by espb_v_transpose_f32, which zeroes the keys t >= len: that pair is what the encoders run.

Poisoning.  K and V rows t >= len of q|k|v are NaN, bd is NaN outside each row's band [T-1-i, T-1-i+len-1] (so also at columns >= 2T-1),
and the output is a window (ldo = H*64 + 32, a plane larger than needed) of a buffer that starts NaN: the 32 columns past each row, the
gap after each plane and the tail must still be NaN after the call.  Rows < len are compared with the reference; rows len <= t < T must
be finite; rows of query blocks (128 rows) that start at or beyond len, and every row when len = 0, are exactly +0 in both planes.

The reference takes the split inputs as the values hi + lo the kernel reads, so the tf32 split of the inputs is not an error here.
Tolerance, per output element o[i][c], u = 2^-24 (test_tolerances_catch_plausible_bugs checks on the CPU that each plausible bug named
below moves the reference by more than 10x it):
* Scores.  s = q . k in 3xTF32: the dropped lo*lo term is < 2^-20 |q_c k_c| per product (each lo < 2^-10 of its value); the wgmma
  accumulation is 24 accumulator updates (8 k-steps x 3 products) of at most 2u each plus 2u for the products summed inside one MMA
  -- together < 66u S with S = sum_c |q_c k_c|.  Adding bd rounds once more: e_s = 66u S + u (S + |bd|).
* Softmax weights.  The scale 1/8 is exact.  fmaf(s, 1/8, -m) rounds by u |x| (x = s/8 - m <= 0), the multiply by log2 e inside __expf by
  another u |x| and ex2.approx is within 2 ulp; each rescale exp(m_old - m_new) of a later tile adds the same for its argument, and these
  arguments sum to at most |x|.  A key's weight is therefore off relatively by
  rho = e_s / 8 + 4u (m - s/8) + (4 nkt + 4) u,  nkt = ceil(len / 64) key tiles,
  and the tf32 hi/lo split of P (lo truncated: < 2^-20 relative) by 16u more.  A relative weight error rho_j moves o by at most
  sum_j p_j rho_j (|v_j| + |o|).
* P V.  3xTF32 again (66u sum_j p_j |v_j|) plus one fmaf rounding per key tile into the running accumulator (nkt u sum_j p_j |v_j|).
* Row sum, 1/l and the output split.  Each thread sums len/4 positive terms in sequence, 2 butterfly adds and nkt rescale fmafs:
  (len/4 + nkt + 2) u relative; 1/l and o * (1/l) one rounding each; hi + lo of the stored output is within 16u |o| of the fp32 result.
tol = sum_j p_j (rho_j + 16u) (|v_j| + |o|) + (66 + nkt) u sum_j p_j |v_j| + (len/4 + nkt + 20) u |o|.
The bound is relative to the score magnitudes: at randn inputs it is about 3e-5 relative to |v|, at the peaked rows (scaled logits
+-60, max in the last or the first key tile, so exp(m_old - m_new) underflows to 0) about 3e-4.
Bugs, at T = 129 (rel-pos, randn): bd read one column off (T-i+j), 1/d_k in place of 1/sqrt(d_k), the last key dropped, and the bd row
of query i+1 used for query i each move o by more than 10x the tolerance.
"""
import math

import numpy as np
import pytest
import torch

gpu = pytest.mark.gpu

DK = 64
U32 = 2.0 ** -24
NAN = float("nan")
NAN_BITS = int(np.float32(NAN).view(np.int32))

CASES = [(1, 1, 37, [37]), (2, 2, 100, [100, 64]), (2, 2, 300, [300, 129]), (3, 2, 520, [520, 256, 1]), (1, 8, 937, [937]), (2, 3, 700, [699, 513])]

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


def _split_np(x):
    """tf32_hi / tf32_lo of common.cuh in numpy float32: hi = x with its 13 low bits cleared, lo = (x - hi) with its 13 low bits cleared."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    hi = (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
    lo = ((x - hi).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
    return hi, lo


def _split_dev(x, gap=4):
    """Split planes of float32 numpy x as one device buffer [2][x.size + gap] (gap a multiple of 4: the plane is a TMA stride), its plane
    stride, and the float64 value hi + lo the kernel reads."""
    hi, lo = _split_np(x)
    plane = x.size + gap
    buf = np.full(2 * plane, np.nan, dtype=np.float32)
    buf[:x.size], buf[plane:plane + x.size] = hi.ravel(), lo.ravel()
    return _dev(buf), plane, hi.astype(np.float64) + lo.astype(np.float64)


def _all_nan_bits(t):
    return bool((t.view(torch.int32) == NAN_BITS).all())


def _pitch(n):
    return (n + 31) // 32 * 32


def _band_mask(T, Rp, lens):
    """[B][1][T][Rp] bool: column c of row i is key c - (T-1-i) of that row, inside [0, len)."""
    j = np.arange(Rp)[None, :] - (T - 1 - np.arange(T)[:, None])
    return np.stack([(j >= 0) & (j < n) for n in lens])[:, None]


def _inputs(B, H, T, lens, relpos, regime, seed, poison=True):
    """float32 inputs: qkv [B][T][3D], qu [B][T][D] (rel-pos) and bd [B][H][T][Rp] (rel-pos).  poison: K and V rows t >= len NaN, bd NaN
    outside the band.  regime: "randn"; "zero" (q = 0 and bd = 0: uniform weights); "peaked" (scaled logits +-60: even rows peak at two
    keys of the last key tile, odd rows at keys 0 and 1 of the first)."""
    D = H * DK
    rng = np.random.default_rng(seed)
    qkv = rng.standard_normal((B, T, 3 * D), dtype=np.float32)
    qu = rng.standard_normal((B, T, D), dtype=np.float32) if relpos else None
    Rp = _pitch(2 * T - 1)
    bd = (2 * rng.standard_normal((B, H, T, Rp))).astype(np.float32) if relpos else None
    q = (qu if relpos else qkv[..., :D]).reshape(B, T, H, DK)
    k = qkv[..., D:2 * D].reshape(B, T, H, DK)
    if regime == "zero":
        q[...] = 0
        if relpos:
            bd[...] = 0
    elif regime == "peaked":
        q *= 0.3
        if relpos:
            bd *= 0.25
        for b, n in enumerate(lens):
            if n == 0:
                continue
            last = 64 * ((n - 1) // 64)
            k[b, :, :, 0:2] = -1
            k[b, [n - 1, last], :, 0] = 1          # planted in the last key tile
            k[b, [0, min(1, n - 1)], :, 1] = 1     # planted in the first
        q[:, 0::2, :, 0], q[:, 0::2, :, 1] = 480, 0
        q[:, 1::2, :, 0], q[:, 1::2, :, 1] = 0, 480
    if poison:
        for b, n in enumerate(lens):
            qkv[b, n:, D:] = np.nan
        if relpos:
            bd[~np.broadcast_to(_band_mask(T, Rp, lens), bd.shape)] = np.nan
    return qkv, qu, bd, Rp


def _reference(q, k, v, bd, lens, T, scale=0.125, shift=0, bd_row=0, drop_last=False):
    """float64 attention of q / k / v [B][H][T][64] (rows >= len of k and v are not read) with the rel-pos term bd [B][H][T][Rp] (or None)
    -> (o, tol), both [B][H][T][64], zero for utterances of length 0.  shift / bd_row / scale / drop_last restate plausible bugs: the band
    read shift columns late, row i + bd_row of bd used for query i, another scale, the last key left out."""
    o, tol = torch.zeros_like(q), torch.zeros_like(q)
    ar = torch.arange(T, device=q.device)
    for b, n in enumerate(lens):
        n = min(n, T) - (1 if drop_last and n > 1 else 0)
        if n <= 0:
            continue
        qb, kb, vb = q[b], k[b, :, :n], v[b, :, :n]
        s = qb @ kb.transpose(-1, -2)
        S = qb.abs() @ kb.abs().transpose(-1, -2)
        es = 66 * U32 * S
        if bd is not None:
            rows = (ar + bd_row).clamp(max=T - 1)
            idx = (T - 1 - ar.view(T, 1) + torch.arange(n, device=q.device).view(1, n) + shift).clamp(0, bd.shape[-1] - 1)
            band = bd[b][:, rows].gather(-1, idx.expand(bd.shape[1], T, n))
            s = s + band
            es = es + U32 * (S + band.abs())
        else:
            es = es + U32 * S
        z = s * scale
        m = z.max(-1, keepdim=True).values
        e = torch.exp(z - m)
        p = e / e.sum(-1, keepdim=True)
        ob = p @ vb
        nkt = (n + 63) // 64
        rho = es * scale + 4 * U32 * (m - z) + (4 * nkt + 4 + 16) * U32
        pr = p * rho
        va = vb.abs()
        tol[b] = pr @ va + pr.sum(-1, keepdim=True) * ob.abs() + (66 + nkt) * U32 * (p @ va) + (n / 4 + nkt + 20) * U32 * ob.abs()
        o[b] = ob
    return o, tol


def _heads(x, B, T, H):
    """[B][T][H*64] (numpy or torch, float64) -> torch [B][H][T][64] on the GPU."""
    x = torch.as_tensor(np.ascontiguousarray(x)) if isinstance(x, np.ndarray) else x
    return x.view(B, T, H, DK).permute(0, 2, 1, 3).contiguous().cuda()


def _run(B, H, T, lens, relpos, regime="randn", seed=0):
    """One espb_flash_attn_f32 call in the encoder's form (rel-pos or plain) on poisoned inputs; checks the output window and compares
    rows < len with the float64 reference within the derived tolerance."""
    D, M, Tp = H * DK, B * T, _pitch(T)
    qkv, qu, bd, Rp = _inputs(B, H, T, lens, relpos, regime, seed)
    qkv_d, qkv_plane, qkv_v = _split_dev(qkv)
    lens_d = _dev(np.asarray(lens, dtype=np.int32))
    vt_plane = B * H * DK * Tp + 8
    vt = torch.full((2 * vt_plane,), NAN, device="cuda")
    _call("espb_v_transpose_f32", _ptr(qkv_d), qkv_plane, B, T, D, H, _ptr(lens_d), _ptr(vt), vt_plane, Tp)
    if relpos:
        q_d, q_plane, q_v = _split_dev(qu)
        ldq, bd_d = D, _dev(bd)
    else:
        q_d, q_plane, q_v, ldq, bd_d = qkv_d, qkv_plane, qkv_v[..., :D], 3 * D, None
    ldo = D + 32
    n_out = M * ldo
    out_plane = n_out + 12
    out = torch.full((2 * out_plane + 20,), NAN, device="cuda")
    _call("espb_flash_attn_f32", _ptr(q_d), 0, q_plane, ldq, _ptr(qkv_d), D, qkv_plane, 3 * D, _ptr(vt), vt_plane, Tp, _ptr(bd_d), Rp,
          _ptr(lens_d), B, H, T, DK, _ptr(out), out_plane, ldo)
    torch.cuda.synchronize()
    hi, lo = out[:n_out].view(M, ldo), out[out_plane:out_plane + n_out].view(M, ldo)
    what = f"B{B} H{H} T{T} lens{lens} {'relpos' if relpos else 'plain'} {regime}"
    assert _all_nan_bits(hi[:, D:]) and _all_nan_bits(lo[:, D:]), f"{what}: wrote past a row's H*64 columns"
    assert _all_nan_bits(out[n_out:out_plane]) and _all_nan_bits(out[out_plane + n_out:]), f"{what}: wrote outside its planes"
    hi, lo = hi[:, :D], lo[:, :D]
    assert int((hi.view(torch.int32) & 0x1FFF).abs().max()) == 0, f"{what}: hi plane is not a tf32 value"
    got = (hi.double() + lo.double()).view(B, T, H, DK).permute(0, 2, 1, 3)
    vv = qkv_v[..., 2 * D:].copy()
    kv = qkv_v[..., D:2 * D].copy()
    for b, n in enumerate(lens):       # the reference reads only keys < len; zero the NaN rows so that 0 * NaN never reaches a product
        vv[b, n:], kv[b, n:] = 0, 0
    bd_t = None
    if relpos:
        bd_t = torch.from_numpy(np.nan_to_num(bd.astype(np.float64), nan=0.0)).cuda()
    ref, tol = _reference(_heads(q_v, B, T, H), _heads(kv, B, T, H), _heads(vv, B, T, H), bd_t, lens, T)
    hib, lob = hi.view(B, T, D), lo.view(B, T, D)
    for b, n in enumerate(lens):
        n = min(n, T)
        err = (got[b, :, :n] - ref[b, :, :n]).abs()
        if n:
            worst = (err / tol[b, :, :n]).max().item()
            print(f"{what} b{b}: max abs err {err.max().item():.3e}, worst err/tol {worst:.3f}")
            assert bool((err <= tol[b, :, :n]).all()), f"{what} b{b}: max abs err {err.max().item():.3e}, worst err/tol {worst:.2f}"
        assert bool(torch.isfinite(hib[b, n:]).all()) and bool(torch.isfinite(lob[b, n:]).all()), f"{what} b{b}: padding rows not finite"
        z0 = min(T, (n + 127) // 128 * 128)          # first row of the first query block that is all padding
        assert not bool(hib[b, z0:].view(torch.int32).ne(0).any()), f"{what} b{b}: padding query block not +0 in the hi plane"
        assert not bool(lob[b, z0:].view(torch.int32).ne(0).any()), f"{what} b{b}: padding query block not +0 in the lo plane"


@gpu
@pytest.mark.parametrize("relpos", [True, False])
@pytest.mark.parametrize("B,H,T,lens", CASES)
def test_flash_attention_vs_fp64(B, H, T, lens, relpos):
    """Single and multiple key tiles, ragged batches (masked keys, query blocks that are all padding, a 1-frame utterance), T = 937."""
    _run(B, H, T, lens, relpos, seed=B * 1000 + T)


EDGE_LENS = [1, 2, 63, 64, 65, 127, 128, 129, 192, 193]


@gpu
@pytest.mark.parametrize("relpos", [True, False])
@pytest.mark.parametrize("n", EDGE_LENS)
def test_flash_attention_tile_edges(n, relpos):
    """Lengths at the 64-key tile and 128-query block edges with len = T (T < 64: the Q and K boxes run past T into the TMA zero fill)."""
    _run(1, 1, n, [n], relpos, seed=n)


@gpu
@pytest.mark.parametrize("relpos", [True, False])
def test_flash_attention_edge_lengths_inside_larger_T(relpos):
    """The same lengths as utterances of one batch at T = 450: padding queries, and whole padding query blocks (up to 3 per utterance)."""
    _run(len(EDGE_LENS), 4, 450, EDGE_LENS, relpos, seed=450)


@gpu
@pytest.mark.parametrize("relpos", [True, False])
@pytest.mark.parametrize("B,H,T,lens", [(1, 1, 1, [1]), (2, 4, 17, [17, 9]), (3, 8, 42, [42, 40, 0]), (2, 16, 42, [0, 41]),
                                        (2, 2, 2250, [2250, 1499])])
def test_flash_attention_shapes(B, H, T, lens, relpos):
    """T = 1; 17 and 42 (not multiples of 4; 42 = the streaming encoder's 40-token block + 2); len = 0 (every row +0 in both planes);
    H 1 to 16; T = 2250 (90 s at conv2d)."""
    _run(B, H, T, lens, relpos, seed=T * 10 + H)


@gpu
@pytest.mark.parametrize("relpos", [True, False])
def test_flash_attention_transformer_bench_shape(relpos):
    """H = 16, D = 1024, T = 937: the Transformer encoder's bench shape (plain form), 4 utterances = 512 CTAs, more than 3 waves of 132."""
    _run(4, 16, 937, [937, 900, 513, 128], relpos, seed=937)


@gpu
@pytest.mark.parametrize("regime", ["peaked", "zero"])
@pytest.mark.parametrize("relpos", [True, False])
@pytest.mark.parametrize("B,H,T,lens", [(2, 2, 300, [300, 193]), (1, 4, 64, [64]), (2, 1, 937, [937, 65])])
def test_flash_attention_score_regimes(B, H, T, lens, relpos, regime):
    """peaked: scaled logits +-60 with the row maximum in the last key tile (even rows: exp(m_old - m_new) = exp(-120) underflows to 0) or
    in the first (odd rows: every later key's weight underflows); zero: q = 0 (and bd = 0), uniform weights, o = mean of V over the keys."""
    _run(B, H, T, lens, relpos, regime, seed=T + H)


# ============================================================================================================== refusals
def _refusal_args(**over):
    """A valid plain-form call at B = 1, H = 1, T = 64 (arguments as a dict, `over` replaces some) and its NaN output buffer."""
    T, D = 64, DK
    qkv = _dev(np.random.default_rng(0).standard_normal(2 * (T * 3 * D + 4), dtype=np.float32))
    vt = _dev(np.zeros(2 * (DK * T + 4), dtype=np.float32))
    out = torch.full((2 * (T * D + 4) + 8,), NAN, device="cuda")
    _KEEP.append(out)
    a = dict(q=qkv, q_off=0, q_plane=T * 3 * D + 4, ldq=3 * D, k=qkv, k_off=D, k_plane=T * 3 * D + 4, ldk=3 * D, vt=vt, vt_plane=DK * T + 4,
             Tp=T, bd=None, Rp=0, lens=_dev(np.array([T], dtype=np.int32)), B=1, H=1, T=T, dk=DK, out=out, out_plane=T * D + 4, ldo=D)
    a.update(over)
    return a, out


def _flash(a):
    _call("espb_flash_attn_f32", _ptr(a["q"]), a["q_off"], a["q_plane"], a["ldq"], _ptr(a["k"]), a["k_off"], a["k_plane"], a["ldk"],
          _ptr(a["vt"]), a["vt_plane"], a["Tp"], _ptr(a["bd"]), a["Rp"], _ptr(a["lens"]), a["B"], a["H"], a["T"], a["dk"], _ptr(a["out"]),
          a["out_plane"], a["ldo"])


@gpu
@pytest.mark.parametrize("bad,match", [
    (dict(dk=32), "d_k must be 64"), (dict(B=0), "bad shape"), (dict(H=0), "bad shape"), (dict(T=0), "bad shape"),
    (dict(ldq=3 * DK + 2), "16-byte aligned"), (dict(ldo=DK + 2), "16-byte aligned"), (dict(out_plane=64 * DK + 2), "16-byte aligned"),
    (dict(q_plane=64 * 3 * DK + 2), "16-byte aligned"), (dict(q_off=1), "16-byte aligned"), (dict(out="+1"), "16-byte aligned"),
    (dict(ldk=3 * DK + 2), "TMA stride not a multiple of 16 bytes")])
def test_flash_attn_refusals(bad, match):
    """Each bad argument is refused with a message before any launch, and the output stays untouched; the same call without it runs."""
    if bad.get("out") == "+1":
        a, out = _refusal_args()
        a["out"] = out[1:]                       # 4 bytes past a 16-byte boundary
    else:
        a, out = _refusal_args(**bad)
    with pytest.raises(RuntimeError, match=match):
        _flash(a)
    torch.cuda.synchronize()
    assert _all_nan_bits(out)
    good, out = _refusal_args()
    _flash(good)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(out[:64 * DK]).all())


# ============================================================================================================== tolerance checks
def test_tolerances_catch_plausible_bugs():
    """On the CPU, from the float64 reference above: each plausible bug named in the module docstring moves the output by more than 10x
    the tolerance the GPU tests use, at a tested shape (rel-pos, T = len = 129, randn inputs)."""
    B, H, T, lens = 1, 1, 129, [129]
    qkv, qu, bd, Rp = _inputs(B, H, T, lens, True, "randn", seed=T, poison=False)
    D = H * DK
    f = lambda x: torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64)).view(B, T, H, DK).permute(0, 2, 1, 3)  # noqa: E731
    q, k, v, bdd = f(qu), f(qkv[..., D:2 * D]), f(qkv[..., 2 * D:]), torch.from_numpy(bd.astype(np.float64))
    ref, tol = _reference(q, k, v, bdd, lens, T)
    assert float(tol.max()) < 1e-3

    def over(**bug):
        o, _ = _reference(q, k, v, bdd, lens, T, **bug)
        return ((o - ref).abs() / tol).max().item()

    assert over(shift=1) > 10                   # band one column off: key j of query i reads bd[i][T-i+j]
    assert over(scale=1.0 / DK) > 10            # 1/d_k in place of 1/sqrt(d_k)
    assert over(drop_last=True) > 10            # the last key dropped
    assert over(bd_row=1) > 10                  # the bd row of query i+1 used for query i
