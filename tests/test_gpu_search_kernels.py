"""-m gpu: the beam-search kernels (csrc/search_ops.cu, csrc/ctc_ops.cu) one by one, each called through the C ABI on seeded inputs and
compared with a restatement of the same operation written here: float64 for the attention and CTC prefix-scorer kernels, bit-exact float32
(numpy, which never fuses a multiply into an add) for top-k and beam selection.

Every element a kernel must not read is NaN (frames at or beyond an utterance's length, pad columns beyond V, cache rows off a slot's
ancestor path, scores of inactive slots) and every output starts as NaN, so a stray read or a missing write fails.  Split outputs (hi plane a
tf32 value, lo plane the remainder) are checked for a hi plane with its 13 low mantissa bits zero, and hi + lo is what is compared.

Tolerances:
* attention context: 2e-5 absolute on O(1) outputs (randn q, k, v), as test_gpu_attention.py.  Dropping the last frame of a 937-frame
  utterance moves the context by ~1e-3, a wrong 1/sqrt(d_k) by O(0.1).
* CTC forward variables.  The recursion r_t = logaddexp(r_{t-1}, phi_{t-1}) + x_t has partial derivatives that sum to 1, so an error made at
  one frame is carried forward without growth and errors add up over frames.  Per frame ctc_advance_kernel makes ~1e-6 absolute in its
  __expf / __logf log-add-exp (log of a value in [1, 2], 2^-21.4 absolute, plus the 2-ulp exponential) and two fp32 roundings of the O(|r_t|)
  sum.  So frame t of a state started at frame t0 is allowed  2e-6 (t - t0 + 2) + 4u sum_{t0 <= t' <= t} (|r^n_t'| + |r^b_t'|),  u = 2^-24;
  ctc_init_state's plain blank cumsum gets  1e-6 + 2u sum_{t' <= t} |r^b_t'|.  Values at or below -1e9 are the logzero class (-1e10 plus
  a few log-probabilities, which fp32 cannot resolve) and must simply stay there.
* log_psi (a log-sum-exp over n frames): each term is phi + x rounded once (2u max|term|), the fp32 sum of n exponentials is off by at most
  (n_seq + 8) 4u relatively (n_seq = terms summed by one thread: n/32 per lane in the warp kernels, n in the dense kernel), and the final
  m + log(sum) rounds once: tol = 4u (max|term| + |psi|) + 4u (n_seq + 8) + 1e-6.  part = psi - s_prev adds 2u (|psi| + |s_prev|).
* log-softmax: the row's log-sum-exp is off by (V/256 + 16) 2u (256 threads, V/256 sequential adds each, tree reduction), the subtraction
  rounds once: tol = (V/256 + 16) 2u + 4u |out|.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24          # fp32 unit roundoff
LOGZERO = -1e10           # ctc_prefix_score.py:34
LZ_CLASS = -1e9           # at or below: the logzero class
NAN = float("nan")


def _call(name, *args):
    from espnet_b200.lib import call

    call(name, *args)


def _ptr(t):
    from espnet_b200.lib import ptr

    return ptr(t)


_KEEP = []    # device copies made inline in a call's argument list: only a raw pointer reaches the library, so keep the tensors alive


@pytest.fixture(autouse=True)
def _release_inputs():
    yield
    torch.cuda.synchronize()
    _KEEP.clear()


def _dev(a):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    _KEEP.append(t)
    return t


def _i32(a):
    return _dev(np.asarray(a, dtype=np.int32))


def _bits(a):
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    return a.view(np.int32)


def _joined(split):
    """hi + lo of a split [2][...] output, after checking that hi is a tf32 value."""
    hi, lo = split[0], split[1]
    assert int((hi.view(torch.int32) & 0x1FFF).abs().max()) == 0, "hi plane has low mantissa bits set"
    return hi.double() + lo.double()


# ============================================================================================== decoder cross-attention
SRC_LENS = [1, 7, 63, 64, 65, 937, 2812]
SRC_LENS_SHORT = [1, 7, 63, 64, 65, 937]
W_ALL = [1, 4, 5, 10, 16, 17, 20, 60, 64]


def _ffma_fits(Wg, dk, Tmax):
    """Shared-memory need of the FFMA cross-attention kernel (q, the [W][Tmax] scores, a 128-row K tile) against its 200 KB cap."""
    scs = (Wg * Tmax + 3) // 4 * 4
    return 4 * (Wg * dk + max(scs, 8 * Wg * dk) + 128 * (dk + 4)) <= 200 * 1024


def _src_inputs(dk, H, W, lens, Tmax, seed):
    g = np.random.default_rng(seed)
    U, D = len(lens), H * dk
    q = g.standard_normal((U * W, D), dtype=np.float32)
    k = g.standard_normal((U, H, Tmax, dk), dtype=np.float32)
    v = g.standard_normal((U, H, Tmax, dk), dtype=np.float32)
    for u, T in enumerate(lens):
        k[u, :, T:] = NAN
        v[u, :, T:] = NAN
    return q, k, v


def _src_run(q, k, v, lens, W, H):
    U, _, Tmax, dk = k.shape
    D = H * dk
    ctx = torch.full((2, U * W, D), NAN, device="cuda")
    _call("espb_dec_src_attn_f32", _ptr(_dev(q)), _ptr(_dev(k)), _ptr(_dev(v)), U, Tmax, _ptr(_i32(lens)), W, D, H, _ptr(ctx), U * W * D)
    torch.cuda.synchronize()
    return ctx


def _src_reference(q, k, v, lens, W, H):
    """softmax over t < lens[u] of q . k_t / sqrt(d_k), times v (float64)."""
    U, _, _, dk = k.shape
    out = torch.empty(U * W, H * dk, dtype=torch.float64, device="cuda")
    qd = torch.from_numpy(q).cuda().double().view(U, W, H, dk)
    for u, T in enumerate(lens):
        ku = torch.from_numpy(k[u, :, :T]).cuda().double()
        vu = torch.from_numpy(v[u, :, :T]).cuda().double()
        p = torch.softmax(torch.einsum("whd,htd->wht", qd[u], ku) / math.sqrt(dk), dim=-1)
        out[u * W:(u + 1) * W] = torch.einsum("wht,htd->whd", p, vu).reshape(W, H * dk)
    return out


def _check_src(dk, H, W, lens, Tmax, seed):
    q, k, v = _src_inputs(dk, H, W, lens, Tmax, seed)
    ctx = _src_run(q, k, v, lens, W, H)
    got, ref = _joined(ctx), _src_reference(q, k, v, lens, W, H)
    for u, T in enumerate(lens):
        e = (got[u * W:(u + 1) * W] - ref[u * W:(u + 1) * W]).abs().max().item()
        assert e < 2e-5, f"d_k {dk} W {W} utterance {u} (T {T}): max abs err {e:.3e}"


def _src_lens_for(Wg, dk):
    """The 2812-frame batch unless the FFMA kernel (the path for d_k != 64) cannot hold its [W][Tmax] scores."""
    if dk != 64 and not _ffma_fits(Wg, dk, max(SRC_LENS) + 1):
        return SRC_LENS_SHORT
    return SRC_LENS


@pytest.mark.parametrize("W", W_ALL)
@pytest.mark.parametrize("dk,H", [(16, 3), (32, 3), (48, 2), (64, 2), (128, 2)])
def test_src_attn_default_path_vs_fp64(dk, H, W):
    """Default dispatch: the single-pass mma kernel at d_k = 64, the run-time FFMA kernel otherwise; slot groups of 16 with w0 > 0 and a
    partial last group for W > 16."""
    lens = _src_lens_for(min(W, 16), dk)
    _check_src(dk, H, W, lens, max(lens) + 1, seed=dk * 100 + W)


@pytest.mark.parametrize("dk,H,Tmax", [(32, 2, 3200), (48, 2, 2813), (128, 2, 2813)])
def test_src_attn_refuses_beyond_shared_memory(dk, H, Tmax):
    """Past the FFMA kernel's shared-memory cap the launcher returns an error and launches nothing."""
    W = 16
    assert not _ffma_fits(W, dk, Tmax)
    lens = [Tmax] if Tmax == 3200 else [1, Tmax - 1]
    q, k, v = _src_inputs(dk, H, W, lens, Tmax, seed=1)
    D = H * dk
    ctx = torch.full((2, len(lens) * W, D), NAN, device="cuda")
    with pytest.raises(RuntimeError, match="shared memory"):
        _call("espb_dec_src_attn_f32", _ptr(_dev(q)), _ptr(_dev(k)), _ptr(_dev(v)), len(lens), Tmax, _ptr(_i32(lens)), W, D, H, _ptr(ctx),
              len(lens) * W * D)
    torch.cuda.synchronize()
    assert bool(ctx.isnan().all())


# ============================================================================================== decoder self-attention and the ancestor table
def _ancestors(n, pos, rng, anc_ld, step_form):
    """Ancestor table after `pos` steps of random selections (permutations and repeated parents), built by espb_anc_update_i32, each
    update checked against n_anc[s][:j] = anc[parent[s]][:j], n_anc[s][j] = parent[s], the rest untouched."""
    anc = np.zeros((n, anc_ld), dtype=np.int32)
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    for j in range(pos):
        parent = rng.permutation(n) if j % 2 else rng.integers(0, max(1, n // 2), n)
        parent = parent.astype(np.int32)
        out = torch.full((n, anc_ld), -7, dtype=torch.int32, device="cuda")
        if step_form:
            step.fill_(j // 2)
            _call("espb_anc_update_i32", _ptr(_i32(anc)), _ptr(out), anc_ld, _ptr(_i32(parent)), j - j // 2, _ptr(step), n)
        else:
            _call("espb_anc_update_i32", _ptr(_i32(anc)), _ptr(out), anc_ld, _ptr(_i32(parent)), j, None, n)
        ref = np.full((n, anc_ld), -7, dtype=np.int32)
        ref[:, :j] = anc[parent, :j]
        ref[:, j] = parent
        np.testing.assert_array_equal(out.cpu().numpy(), ref, err_msg=f"anc_update at pos {j}")
        anc = ref
    anc[anc < 0] = 0      # columns >= pos are never read; keep them in range
    return anc


SELF_KERNELS = [(64, 2, "fast"), (64, 2, "misaligned"), (16, 4, ""), (32, 3, ""), (48, 2, ""), (128, 2, "")]


@pytest.mark.parametrize("step_form", [False, True])
@pytest.mark.parametrize("pos", [0, 1, 7, 8, 31, 32, 33, 64, 100])
@pytest.mark.parametrize("dk,H,variant", SELF_KERNELS)
def test_dec_self_attn_vs_fp64(dk, H, variant, pos, step_form):
    """The d_k = 64 kernel, the generic kernel (d_k 16 / 32 / 48 / 128, and d_k = 64 with a ctx pointer off 16-byte alignment) over a cache
    gathered through a random ancestor table; the position as a value or value + *step_ptr."""
    rng = np.random.default_rng(1000 * dk + 10 * pos + step_form)
    n, D = 6, H * dk
    max_pos = pos + 3 if step_form else pos
    Lmax = max_pos + 1
    anc = _ancestors(n, pos, rng, Lmax, step_form)
    kc = np.full((Lmax, n, D), NAN, dtype=np.float32)   # rows off every slot's ancestor path stay NaN
    vc = np.full((Lmax, n, D), NAN, dtype=np.float32)
    for j in range(pos):
        for r in set(anc[:, j].tolist()):
            kc[j, r] = rng.standard_normal(D, dtype=np.float32)
            vc[j, r] = rng.standard_normal(D, dtype=np.float32)
    qkv = rng.standard_normal((n, 3 * D), dtype=np.float32)
    kcd, vcd = _dev(kc), _dev(vc)
    off = 1 if variant == "misaligned" else 0
    buf = torch.full((2 * n * D + 8,), NAN, device="cuda")
    ctx_ptr = _ptr(buf[off:off + 2 * n * D])
    if step_form:
        sp = _i32([pos // 2])
        _call("espb_dec_self_attn_f32", _ptr(_dev(qkv)), _ptr(kcd), _ptr(vcd), _ptr(_i32(anc)), Lmax, n, D, H, pos - pos // 2, _ptr(sp), max_pos,
              ctx_ptr, n * D)
    else:
        _call("espb_dec_self_attn_f32", _ptr(_dev(qkv)), _ptr(kcd), _ptr(vcd), _ptr(_i32(anc)), Lmax, n, D, H, pos, None, max_pos, ctx_ptr, n * D)
    torch.cuda.synchronize()
    # the cache: row pos holds this step's k, v bit for bit, nothing else changed
    kc_ref, vc_ref = kc.copy(), vc.copy()
    kc_ref[pos], vc_ref[pos] = qkv[:, D:2 * D], qkv[:, 2 * D:]
    np.testing.assert_array_equal(_bits(kcd), kc_ref.view(np.int32))
    np.testing.assert_array_equal(_bits(vcd), vc_ref.view(np.int32))
    assert bool(buf[:off].isnan().all()) and bool(buf[off + 2 * n * D:].isnan().all()), "write outside ctx"
    got = _joined(buf[off:off + 2 * n * D].view(2, n, D)).cpu().numpy()
    ref = np.empty((n, D))
    for s in range(n):
        K = np.stack([kc[j, anc[s, j]] for j in range(pos)] + [qkv[s, D:2 * D]]).astype(np.float64)
        Vv = np.stack([vc[j, anc[s, j]] for j in range(pos)] + [qkv[s, 2 * D:]]).astype(np.float64)
        for h in range(H):
            sl = slice(h * dk, (h + 1) * dk)
            sc = K[:, sl] @ qkv[s, sl].astype(np.float64) / math.sqrt(dk)
            p = np.exp(sc - sc.max())
            ref[s, sl] = (p / p.sum()) @ Vv[:, sl]
    e = np.abs(got - ref).max()
    assert e < 2e-5, f"max abs err {e:.3e}"


@pytest.mark.parametrize("D,H", [(512, 2), (100, 3)])
def test_dec_self_attn_refuses_unsupported_heads(D, H):
    """d_k > 128 (lanes hold 4 elements of a head each) and D % H != 0 are refused before any launch."""
    n = 2
    qkv = torch.randn(n, 3 * D, device="cuda")
    kc = torch.full((2, n, D), NAN, device="cuda")
    vc = torch.full((2, n, D), NAN, device="cuda")
    ctx = torch.full((2, n, D), NAN, device="cuda")
    anc = torch.zeros(n, 2, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError, match="d_k"):
        _call("espb_dec_self_attn_f32", _ptr(qkv), _ptr(kc), _ptr(vc), _ptr(anc), 2, n, D, H, 0, None, 0, _ptr(ctx), n * D)
    torch.cuda.synchronize()
    assert bool(ctx.isnan().all()) and bool(kc.isnan().all())


# ============================================================================================== CTC prefix scorer
CTC_LENS = [1, 2, 3, 31, 32, 33, 97, 2812]
CTC_V, BLANK, EOS, CTC_W = 128, 0, 127, 4


def _lae(a, b):
    m = max(a, b)
    return m + math.log1p(math.exp(-abs(a - b)))


def _posteriors(lens, Tmax, V, rng):
    """log_softmax(3 randn) with the blank raised on ~60 % of the frames (peaky, blank-heavy); NaN at frames >= lens[u]."""
    logits = 3.0 * rng.standard_normal((len(lens), Tmax, V))
    logits[..., BLANK] += np.where(rng.random((len(lens), Tmax)) < 0.6, 8.0, 0.0)
    m = logits.max(-1, keepdims=True)
    x = (logits - m - np.log(np.exp(logits - m).sum(-1, keepdims=True))).astype(np.float32)
    for u, T in enumerate(lens):
        x[u, T:] = NAN
    return x


def _close(got, ref, tol, what):
    """Logzero-class references must give logzero-class values; elsewhere |got - ref| <= tol."""
    got, ref, tol = np.asarray(got, np.float64), np.asarray(ref, np.float64), np.broadcast_to(tol, np.shape(ref))
    lz = ref <= LZ_CLASS
    bad_lz = lz & ~(got <= LZ_CLASS)
    assert not bad_lz.any(), f"{what}: expected logzero at {np.argwhere(bad_lz)[:5].tolist()}, got {got[bad_lz][:5]}"
    err = np.where(lz, 0.0, np.abs(got - ref))
    bad = ~(err <= tol)
    assert not bad.any(), (f"{what}: {int(bad.sum())} values off, first at {np.argwhere(bad)[:3].tolist()}: got {got[bad][:3]}, "
                           f"ref {ref[bad][:3]}, tol {tol[bad][:3]}")


def _mag(v):
    v = np.abs(np.asarray(v, np.float64))
    return np.where(v >= -LZ_CLASS, 0.0, v)


def _phi(rp, same):
    """log_phi[t] of a state (ctc_prefix_score.py:135-144): r^b for a repeated label, else logaddexp(r^n, r^b) (float64)."""
    rp = rp.astype(np.float64)
    return rp[:, 1] if same else np.logaddexp(rp[:, 0], rp[:, 1])


def _psi_ref(x, T, rp, cands, last, out_len, n_seq_div):
    """log_psi of every candidate and its tolerance (ctc_prefix_score.py:166-189) from one slot's previous state rp [Tmax][4]."""
    from scipy.special import logsumexp

    psi, tol = np.empty(len(cands)), np.empty(len(cands))
    start = max(out_len, 1)
    for i, c in enumerate(cands):
        if c == EOS:
            psi[i] = np.logaddexp(float(rp[T - 1, 0]), float(rp[T - 1, 1]))
            tol[i] = 4 * U32 * _mag(psi[i]) + 1e-6
            continue
        if c == BLANK:
            psi[i], tol[i] = LOGZERO, 0.0
            continue
        terms = _phi(rp, c == last)[start - 1:T - 1] + x[start:T, c].astype(np.float64)
        terms = np.append(terms, float(x[0, c]) if out_len == 0 else LOGZERO)
        psi[i] = logsumexp(terms)
        tol[i] = 4 * U32 * (_mag(terms).max() + _mag(psi[i])) + 4 * U32 * (len(terms) / n_seq_div + 8) + 1e-6
    return psi, tol


def _advance_ref(x, T, Tmax, rp, c, last, out_len):
    """New forward variables [Tmax][3] (r^n, r^b, r_sum) of the prefix extended by c (ctc_prefix_score.py:128-164) and their tolerance."""
    out = np.full((Tmax, 3), LOGZERO)
    tol = np.zeros(Tmax)
    start = max(out_len, 1)
    if start - 1 >= T:        # prefix longer than the encoder output: all logzero
        return out, tol
    phi = _phi(rp, c == last)
    rn, rb = (float(x[0, c]) if out_len == 0 else LOGZERO), LOGZERO
    out[start - 1] = (rn, rb, _lae(rn, rb))
    mass = 0.0
    for t in range(start, T):
        rn, rb = _lae(rn, phi[t - 1]) + float(x[t, c]), _lae(rn, rb) + float(x[t, BLANK])
        out[t] = (rn, rb, _lae(rn, rb))
        mass += (abs(rn) if rn > LZ_CLASS else 0.0) + (abs(rb) if rb > LZ_CLASS else 0.0)
        tol[t] = 2e-6 * (t - start + 2) + 4 * U32 * mass
    tol[start - 1] = 1e-6
    return out, tol


def _check_state(got, ref, tol, what):
    """got [Tmax][4] kernel state vs ref [Tmax][3]; the fourth float is 0."""
    for k, name in enumerate(("r^n", "r^b", "r_sum")):
        _close(got[:, k], ref[:, k], tol, f"{what} {name}")
    assert not got[:, 3].any(), f"{what}: fourth component not zero"


def _check_init(r, s_prev, x, lens, Tmax, W):
    r = r.cpu().numpy()
    assert not s_prev.cpu().numpy().any()
    for s in range(r.shape[0]):
        T = lens[s // W]
        ref = np.full((Tmax, 3), LOGZERO)
        cs = np.cumsum(x[s // W, :T, BLANK].astype(np.float64))
        ref[:T, 1] = ref[:T, 2] = cs
        tol = 1e-6 + 2 * U32 * np.concatenate([np.cumsum(np.abs(cs)), np.zeros(Tmax - T)])
        _check_state(r[s], ref, tol, f"init slot {s}")
        assert (r[s, :, 0] == np.float32(LOGZERO)).all()


def _candidates(rng, P, last, w):
    """P distinct tokens; per slot position w the list holds blank, eos (its duplicate is flagged invalid) or the slot's last token."""
    c = rng.permutation(CTC_V)[:P]
    want = [BLANK, EOS, last, None][w % 4]
    if want is None:
        c[c == EOS] = 1
    elif want not in c:
        c[rng.integers(P)] = want
    return c.astype(np.int32)


def _ctc_chain(P, token_major, seed, steps=35, dense_at=(0, 1, 2, 33)):
    """init, then `steps` rounds of (score the candidates [and the dense vocabulary] of every slot, advance every slot by a chosen token and
    parent): each kernel's output is compared with the float64 restatement applied to the kernel's own input state."""
    rng = np.random.default_rng(seed)
    lens, Tmax, W = CTC_LENS, max(CTC_LENS) + 1, CTC_W
    U, V = len(lens), CTC_V
    n = U * W
    x = _posteriors(lens, Tmax, V, rng)
    xd, lens32 = _dev(x), _i32(lens)
    if token_major:
        xk = torch.full((U, V, Tmax), NAN, device="cuda")
        _call("espb_transpose_tv_f32", _ptr(xd), U, Tmax, V, _ptr(xk))
        np.testing.assert_array_equal(_bits(xk), np.ascontiguousarray(x.transpose(0, 2, 1)).view(np.int32))
    else:
        xk = xd
    r = torch.full((n, Tmax, 4), NAN, device="cuda")
    s_prev = torch.full((n,), NAN, device="cuda")
    _call("espb_ctc_init_state_f32", _ptr(xd), U, Tmax, V, _ptr(lens32), BLANK, W, _ptr(r), _ptr(s_prev))
    _check_init(r, s_prev, x, lens, Tmax, W)
    last = np.full(n, EOS, dtype=np.int32)           # sos = eos
    live = np.ones(n, dtype=bool)
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    for L in range(steps):
        rh, sp_h = r.cpu().numpy(), s_prev.cpu().numpy()
        if L % 2:                                      # the step_ptr form: out_len = value + *step_ptr
            step.fill_(L // 2)
            arg, sp = L - L // 2, _ptr(step)
        else:
            arg, sp = L, None
        # ---- candidate scoring
        cand = np.stack([_candidates(rng, P, int(last[s]), s) for s in range(n)])
        part = torch.full((n, P + 1), NAN, device="cuda")
        psi = torch.full((n, P + 1), NAN, device="cuda")
        valid = torch.full((n, P + 1), -1, dtype=torch.int32, device="cuda")
        _call("espb_ctc_score_cands_f32", _ptr(xk), U, Tmax, V, _ptr(lens32), BLANK, EOS, W, _ptr(r), _ptr(s_prev), _ptr(_i32(last)), arg, sp,
              _ptr(_i32(cand)), P, _ptr(part), _ptr(psi), _ptr(valid), token_major)
        part_h, psi_h = part.cpu().numpy(), psi.cpu().numpy()
        v_ref = np.ones((n, P + 1), dtype=np.int32)
        v_ref[:, P] = ~(cand == EOS).any(1)
        np.testing.assert_array_equal(valid.cpu().numpy(), v_ref, err_msg=f"valid at out_len {L}")
        for s in range(n):
            T = lens[s // W]
            if L > T + 1:      # the search stops such an utterance (IndexError boundary)
                continue
            ref, tol = _psi_ref(x[s // W], T, rh[s], list(cand[s]) + [EOS], int(last[s]), L, 32)
            _close(psi_h[s], ref, tol, f"psi slot {s} out_len {L} P {P} token_major {token_major}")
            ok = (ref > LZ_CLASS) & (sp_h[s] > LZ_CLASS)
            _close(part_h[s][ok], (ref - float(sp_h[s]))[ok], (tol + 2 * U32 * (_mag(ref) + _mag(sp_h[s])))[ok], f"part slot {s} out_len {L}")
        # ---- dense scoring ([u][t][v] layout only)
        if L in dense_at and not token_major:
            dense = torch.full((n, V), NAN, device="cuda")
            _call("espb_ctc_score_dense_f32", _ptr(xd), U, Tmax, V, _ptr(lens32), BLANK, EOS, W, _ptr(r), _ptr(s_prev), _ptr(_i32(last)), L,
                  _ptr(dense))
            dh = dense.cpu().numpy()
            for s in range(n):
                T = lens[s // W]
                if L > T + 1:
                    continue
                ref, tol = _psi_ref(x[s // W], T, rh[s], list(range(V)), int(last[s]), L, 1)
                ok = (ref > LZ_CLASS) & (sp_h[s] > LZ_CLASS)
                _close(dh[s][ok], (ref - float(sp_h[s]))[ok], (tol + 2 * U32 * (_mag(ref) + _mag(sp_h[s])))[ok], f"dense slot {s} out_len {L}")
        # ---- advance: parents among the live slots of the utterance; slot 0 extends by a regular token, slot 1 repeats the parent's last
        # token (the r^b branch), slot 2 takes blank / eos / a regular token, slot 3 is inactive every other step
        parent = np.empty(n, dtype=np.int32)
        tok = np.empty(n, dtype=np.int32)
        act = np.ones(n, dtype=np.int32)
        for s in range(n):
            u, w = divmod(s, W)
            alive = [u * W + i for i in range(W) if live[u * W + i]] or [u * W]
            parent[s] = alive[0] if w == 0 else rng.choice(alive)
            regular = int(rng.integers(1, EOS))
            pl = int(last[parent[s]])
            tok[s] = [regular, pl if 0 < pl < EOS else regular, [BLANK, EOS, regular][L % 3], regular][w]
            act[s] = 0 if (w == 3 and L % 2) else 1
        r_new = torch.full((n, Tmax, 4), NAN, device="cuda")
        s_new = torch.full((n,), NAN, device="cuda")
        _call("espb_ctc_advance_f32", _ptr(xk), U, Tmax, V, _ptr(lens32), BLANK, EOS, W, _ptr(r), _ptr(_i32(parent)), _ptr(_i32(last)),
              _ptr(_i32(tok)), _ptr(_i32(act)), arg, sp, _ptr(r_new), _ptr(s_new), token_major)
        rn_h, sn_h = r_new.cpu().numpy(), s_new.cpu().numpy()
        z4 = np.array([LOGZERO, LOGZERO, LOGZERO, 0.0], dtype=np.float32)
        for s in range(n):
            u, T, c, p = s // W, lens[s // W], int(tok[s]), int(parent[s])
            if not act[s] or c in (EOS, BLANK):
                np.testing.assert_array_equal(rn_h[s].view(np.int32), np.broadcast_to(z4, rn_h[s].shape).view(np.int32),
                                              err_msg=f"zeroed state slot {s}")
                assert sn_h[s] == np.float32(LOGZERO if (act[s] and c == BLANK) else 0.0), f"s_new slot {s}"
                continue
            if L > T + 1:
                continue
            ref, tol = _advance_ref(x[u], T, Tmax, rh[p], c, int(last[p]), L)
            _check_state(rn_h[s], ref, tol, f"advance slot {s} out_len {L} T {T}")
            pr, pt = _psi_ref(x[u], T, rh[p], [c], int(last[p]), L, 32)
            _close(sn_h[s:s + 1], pr, pt, f"s_new slot {s} out_len {L}")
        r, s_prev, last = r_new, s_new, tok
        live = (act == 1) & (tok != EOS) & (tok != BLANK)
    return x, r


@pytest.mark.parametrize("token_major", [0, 1])
@pytest.mark.parametrize("P", [1, 15, 96])
def test_ctc_prefix_scorer_chain_vs_fp64(P, token_major):
    """lens 1, 2, 3, 31, 32, 33, 97, 2812 in one batch; out_len 0 .. 34, i.e. T - 2 .. T + 1 for the short utterances (all-logzero state
    once start - 1 >= T); candidates equal to blank, eos (duplicated: valid = 0) and the slot's last token; inactive slots and new tokens
    blank / eos (zeroed state, s_new 0 / logzero); every other step through step_ptr."""
    _ctc_chain(P, token_major, seed=P * 10 + token_major)


@pytest.mark.parametrize("T_new", [57, 40])
def test_ctc_extend_state_vs_fp64(T_new):
    """Streaming extension of kernel-made states from T_old = 40 frames: frames < T_old copied bit for bit, later frames blank-only."""
    rng = np.random.default_rng(T_new)
    T_old, W, V = 40, 4, CTC_V
    x = _posteriors([T_new], T_new, V, rng)[0]
    xo = _dev(np.ascontiguousarray(x[None, :T_old]))
    lens32 = _i32([T_old])
    r = torch.full((W, T_old, 4), NAN, device="cuda")
    s_prev = torch.full((W,), NAN, device="cuda")
    _call("espb_ctc_init_state_f32", _ptr(xo), 1, T_old, V, _ptr(lens32), BLANK, W, _ptr(r), _ptr(s_prev))
    last = np.full(W, EOS, dtype=np.int32)
    for L in range(3):
        tok = rng.integers(1, EOS, W).astype(np.int32)
        r_new = torch.full((W, T_old, 4), NAN, device="cuda")
        s_new = torch.full((W,), NAN, device="cuda")
        _call("espb_ctc_advance_f32", _ptr(xo), 1, T_old, V, _ptr(lens32), BLANK, EOS, W, _ptr(r), _ptr(_i32(np.arange(W))), _ptr(_i32(last)),
              _ptr(_i32(tok)), _ptr(_i32(np.ones(W))), L, None, _ptr(r_new), _ptr(s_new), 0)
        r, last = r_new, tok
    xn = x.copy()
    xn[:T_old] = NAN          # frames the extension must not read
    out = torch.full((W, T_new, 4), NAN, device="cuda")
    _call("espb_ctc_extend_state_f32", _ptr(_dev(xn)), T_new, V, BLANK, W, _ptr(r), T_old, _ptr(out))
    old, got = r.cpu().numpy(), out.cpu().numpy()
    np.testing.assert_array_equal(got[:, :T_old].view(np.int32), old.view(np.int32))
    for s in range(W):
        rb = np.float64(old[s, T_old - 1, 1]) + np.cumsum(x[T_old:, BLANK].astype(np.float64))
        ref = np.stack([np.full(T_new - T_old, LOGZERO), rb, rb], 1)
        _check_state(got[s, T_old:], ref, 1e-6 + 2 * U32 * np.cumsum(np.abs(rb)), f"extend slot {s}")


# ============================================================================================== top-k, log-softmax, argmax, greedy collapse
def _topk_rows(V, scale, rng):
    """Rows: randn; small integers (exact ties); mostly -inf (fewer finite entries than k); all -inf; constant."""
    rows = [rng.standard_normal(V), rng.integers(-3, 3, V).astype(np.float64)]
    if scale != 0:            # -inf * 0 is NaN
        r = np.full(V, -np.inf)
        idx = rng.permutation(V)[:max(1, V // 10)]
        r[idx] = rng.integers(-2, 2, len(idx))
        rows += [r, np.full(V, -np.inf)]
    rows.append(np.full(V, 1.5))
    return np.stack(rows).astype(np.float32)


@pytest.mark.parametrize("scale", [1.0, 0.7, 0.0])
@pytest.mark.parametrize("V", [1, 7, 1024, 1025, 5120, 5121, 10240, 10241, 32768])
def test_rows_topk_bit_exact(V, scale):
    """ids and vals of every k equal a stable sort of float32(x) * float32(scale) by (-value, index), -inf entries included."""
    rng = np.random.default_rng(V + int(10 * scale))
    x = _topk_rows(V, scale, rng)
    rows, ld = x.shape[0], V + 3
    xp = np.full((rows, ld), NAN, dtype=np.float32)
    xp[:, :V] = x
    xd = _dev(xp)
    prod = x * np.float32(scale)
    order = np.argsort(-prod, axis=1, kind="stable")
    for k in [kk for kk in (1, 15, 90, 128) if kk <= V]:
        ids = torch.full((rows, k), -1, dtype=torch.int32, device="cuda")
        vals = torch.full((rows, k), NAN, device="cuda")
        _call("espb_rows_topk_f32", _ptr(xd), rows, ld, V, scale, k, _ptr(ids), _ptr(vals))
        ref_ids = order[:, :k].astype(np.int32)
        np.testing.assert_array_equal(ids.cpu().numpy(), ref_ids, err_msg=f"ids k={k}")
        np.testing.assert_array_equal(_bits(vals), np.take_along_axis(prod, ref_ids, 1).view(np.int32), err_msg=f"vals k={k}")


@pytest.mark.parametrize("V,k", [(32769, 1), (1000, 129), (10, 11)])
def test_rows_topk_refuses(V, k):
    x = torch.zeros(1, V, device="cuda")
    ids = torch.full((1, k), -1, dtype=torch.int32, device="cuda")
    vals = torch.full((1, k), NAN, device="cuda")
    with pytest.raises(RuntimeError, match="rows_topk"):
        _call("espb_rows_topk_f32", _ptr(x), 1, V, V, 1.0, k, _ptr(ids), _ptr(vals))
    assert bool((ids == -1).all())


@pytest.mark.parametrize("V", [1, 2, 2048, 2049, 5120, 5121, 8192, 8193, 32000])
def test_log_softmax_rows_vs_fp64(V):
    """Register kernels (V <= 2048 / 5120 / 8192) and the three-pass kernel; pad columns untouched."""
    rng = np.random.default_rng(V)
    rows, ld = 5, V + 5
    x = np.stack([3 * rng.standard_normal(V), rng.standard_normal(V), np.full(V, 2.5), 10 * rng.standard_normal(V),
                  rng.standard_normal(V)]).astype(np.float32)
    x[4, V // 2] = x[4].max() + 80.0      # one logit 80 above the rest
    xp = np.full((rows, ld), 12345.0, dtype=np.float32)
    xp[:, :V] = x
    xd = _dev(xp)
    _call("espb_log_softmax_rows_f32", _ptr(xd), rows, ld, V)
    got = xd.cpu().numpy()
    np.testing.assert_array_equal(got[:, V:], xp[:, V:])
    xx = x.astype(np.float64)
    m = xx.max(1, keepdims=True)
    lse = m + np.log(np.exp(xx - m).sum(1, keepdims=True))
    ref = xx - lse
    tol = (V / 256 + 16) * 2 * U32 + 4 * U32 * (np.abs(ref) + np.abs(lse))
    err = np.abs(got[:, :V] - ref)
    assert (err <= tol).all(), f"max err {err.max():.3e}, at {np.unravel_index(np.argmax(err - tol), err.shape)}"


@pytest.mark.parametrize("rows", [1, 7, 9, 13])
@pytest.mark.parametrize("V", [1, 31, 32, 33, 5000])
def test_argmax_rows_first_index_on_ties(rows, V):
    rng = np.random.default_rng(rows * 100 + V)
    ld = V + 2
    x = np.full((rows, ld), np.inf, dtype=np.float32)       # pad columns: larger than anything
    x[:, :V] = rng.integers(-3, 3, (rows, V))
    out = torch.full((rows + 3,), -1, dtype=torch.int32, device="cuda")
    _call("espb_argmax_rows_f32", _ptr(_dev(x)), rows, ld, V, _ptr(out))
    ref = np.concatenate([np.argmax(x[:, :V], 1), [-1, -1, -1]]).astype(np.int32)
    np.testing.assert_array_equal(out.cpu().numpy(), ref)


def test_ctc_collapse():
    """Lengths 0, 1, 31, 32, 33, 97; a run of one token across the 32-frame boundary; frames past the length must be ignored."""
    rng = np.random.default_rng(0)
    lens, Tmax, blank = [0, 1, 31, 32, 33, 97, 97], 100, 0
    a = rng.integers(0, 4, (len(lens), Tmax)).astype(np.int32)
    a[5, 30:34] = 3
    a[6, 31] = a[6, 32] = 2
    for b, n in enumerate(lens):
        a[b, n:] = 5
    ids = torch.full((len(lens), Tmax), -1, dtype=torch.int32, device="cuda")
    out_len = torch.full((len(lens),), -1, dtype=torch.int32, device="cuda")
    _call("espb_ctc_collapse_i32", _ptr(_dev(a)), len(lens), Tmax, _ptr(_i32(lens)), blank, _ptr(ids), _ptr(out_len))
    got, gl = ids.cpu().numpy(), out_len.cpu().numpy()
    for b, n in enumerate(lens):
        ref = [int(v) for t, v in enumerate(a[b, :n]) if v != blank and (t == 0 or a[b, t - 1] != v)]
        assert gl[b] == len(ref)
        assert got[b, :len(ref)].tolist() == ref
        assert (got[b, len(ref):] == -1).all()


# ============================================================================================== beam selection
def _beam_ref(inp, U, W, P, V, step, mode, eos, w_dec, w_ctc, pen, maxlen, minlen, ended_cap, maxlen_cap, out):
    """float32 restatement of beam_select_kernel with the reference's arithmetic: each product rounded, then the adds in the order of
    batch_beam_search.py:293-309; W rounds of arg-max (ties -> lower flat index)."""
    f = np.float32
    PC = P + 1 if mode == 1 else P
    o = {k: v.copy() for k, v in out.items()}
    for u in range(U):
        done = inp["utt_done"][u] != 0
        tot = np.full(W * PC, -np.inf, dtype=f)
        if not done:
            for w in range(W):
                s = u * W + w
                if not inp["active"][s]:
                    continue
                with np.errstate(invalid="ignore"):
                    if mode == 1:
                        dec = np.append(inp["cand_val"][s], f(w_dec) * inp["logp"][s, eos])
                        t = ((dec + f(pen)) + f(w_ctc) * inp["part"][s]) + inp["score"][s]
                        t = np.where(inp["valid"][s] != 0, t, f(-np.inf))
                    else:
                        t = (inp["cand_val"][s] + f(pen)) + inp["score"][s]
                tot[w * PC:(w + 1) * PC] = t
        last_step = step == maxlen[u] - 1
        for k in range(W):
            ns, bp = u * W + k, step * U * W + u * W + k
            bidx = int(np.argmax(tot))
            best = tot[bidx]
            if best == -np.inf:
                o["n_active"][ns], o["n_score"][ns], o["n_sc_dec"][ns], o["n_sc_ctc"][ns], o["n_last_tok"][ns] = 0, 0, 0, 0, eos
                o["n_parent"][ns], o["bp_parent"].flat[bp], o["bp_token"].flat[bp] = ns, -1, eos
                continue
            tot[bidx] = -np.inf
            w, j = divmod(bidx, PC)
            s = u * W + w
            tk = eos if (mode == 1 and j == P) else int(inp["cand_ids"][s, j])
            dl = inp["logp"][s, tk] if mode != 2 else f(0)
            cp = inp["part"][s, j] if mode == 1 else (inp["part"][s, tk] if mode == 2 else f(0))
            ndec, nctc = inp["sc_dec"][s] + dl, inp["sc_ctc"][s] + cp
            o["bp_parent"].flat[bp], o["bp_token"].flat[bp], o["n_parent"][ns] = s, tk, s
            o["n_score"][ns], o["n_sc_dec"][ns], o["n_sc_ctc"][ns], o["n_last_tok"][ns] = best, ndec, nctc, tk
            ended = last_step or tk == eos
            o["n_active"][ns] = 0 if ended else 1
            if ended and step >= minlen[u]:
                e = o["ended_count"][u]
                if e < ended_cap:
                    i = u * ended_cap + e
                    o["ended_step"][i], o["ended_slot"][i], o["ended_score"][i], o["ended_dec"][i], o["ended_ctc"][i] = step, ns, best, ndec, nctc
                    o["ended_count"][u] = e + 1
        if not done and last_step:
            o["utt_done"][u] = 1
    return o


# (W, candidates per slot): W * PC on both sides of each kernel instance's capacity (32 x 6, 32 x 12, 32 x 24, 32 x 52 for W <= 32,
# 256 x 14, 256 x 28), and the wide beam W = 64 with P = 96.
BEAM_SHAPES = [(4, 48), (1, 193), (8, 48), (5, 77), (16, 48), (1, 769), (32, 52), (32, 53), (33, 50), (33, 51), (64, 56), (15, 239), (64, 97)]


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("W,PC", BEAM_SHAPES)
def test_beam_select_bit_exact(W, PC, mode):
    """Utterance 0: quantised values (exact ties), one inactive slot, invalid entries, eos winners appended (minlen 0); 1: finished;
    2: one live slot with few valid candidates (fewer than W), eos ended under minlen (not appended); 3: the last step (everything ends)."""
    rng = np.random.default_rng(W * 1000 + PC * 3 + mode)
    f = np.float32
    U, V, eos, step, ended_cap, maxlen_cap = 4, 1000, 999, 5, 4 * 64 + 8, 16
    P = PC - 1 if mode == 1 else PC
    n = U * W
    w_dec, w_ctc, pen = 0.7, 0.3, 0.25
    q = lambda a: np.round(a * 4) / 4                                   # noqa: E731
    score = (-5 * rng.random(n)).astype(f)
    sc_dec, sc_ctc = rng.standard_normal(n).astype(f), rng.standard_normal(n).astype(f)
    active = np.ones(n, dtype=np.int32)
    if W > 1:
        active[1] = 0
    active[2 * W + 1:3 * W] = 0
    cand_ids = np.stack([rng.permutation(V - 1)[:P] for _ in range(n)]).astype(np.int32)
    logp = np.log(rng.dirichlet(np.ones(V), n)).astype(f)
    part_c = (-np.abs(2 * rng.standard_normal((n, PC))) - 0.5).astype(f)
    part_d = (-np.abs(2 * rng.standard_normal((n, V))) - 0.5).astype(f)
    logp[::2, eos] = -0.05                                               # eos is a strong candidate on every other slot ...
    if mode != 1:
        cand_ids[::3, 0] = eos
    score[0], part_c[0, PC - 1], part_d[0, eos] = 0.0, 0.0, 0.0         # ... and wins outright on slot 0
    cand_val = np.take_along_axis(part_d, cand_ids, 1) * f(w_ctc) if mode == 2 else np.take_along_axis(logp, cand_ids, 1) * f(w_dec)
    valid = (rng.random((n, PC)) < 0.9).astype(np.int32)
    valid[0, PC - 1] = 1
    k2 = W // 2                                                          # utterance 2: fewer live candidates than W
    valid[2 * W, :] = 0
    valid[2 * W, :k2] = 1
    if mode != 1:
        cand_val[2 * W, k2:] = -np.inf
    # utterance 0 on a grid of quarters: many exact ties
    for a in (score, sc_dec, sc_ctc):
        a[:W] = q(a[:W])
    cand_val[:W] = q(cand_val[:W])
    part_c[:W] = q(part_c[:W])
    # poison what must not be read: inactive slots, the finished utterance, invalid entries
    dead = active == 0
    dead[W:2 * W] = True
    for a in (score, sc_dec, sc_ctc):
        a[dead] = NAN
    cand_val[dead], logp[dead], part_c[dead], part_d[dead] = NAN, NAN, NAN, NAN
    if mode == 1:
        cand_val[valid[:, :P] == 0] = NAN
        part_c[valid == 0] = NAN
    part = part_c if mode == 1 else part_d
    maxlen = np.array([100, 100, 100, step + 1], dtype=np.int32)
    minlen = np.array([0, 0, step + 1, 0], dtype=np.int32)
    utt_done = np.array([0, 1, 0, 0], dtype=np.int32)
    inp = dict(score=score, sc_dec=sc_dec, sc_ctc=sc_ctc, active=active, cand_ids=cand_ids, cand_val=cand_val, logp=logp, part=part,
               valid=valid, utt_done=utt_done)
    out = dict(n_score=np.full(n, NAN, f), n_sc_dec=np.full(n, NAN, f), n_sc_ctc=np.full(n, NAN, f), n_active=np.full(n, -9, np.int32),
               n_last_tok=np.full(n, -9, np.int32), n_parent=np.full(n, -9, np.int32), bp_parent=np.full((maxlen_cap, n), -9, np.int32),
               bp_token=np.full((maxlen_cap, n), -9, np.int32), ended_count=np.array([2, 0, 0, 1], np.int32),
               ended_step=np.full(U * ended_cap, -9, np.int32), ended_slot=np.full(U * ended_cap, -9, np.int32),
               ended_score=np.full(U * ended_cap, NAN, f), ended_dec=np.full(U * ended_cap, NAN, f), ended_ctc=np.full(U * ended_cap, NAN, f),
               utt_done=utt_done.copy())
    ref = _beam_ref(inp, U, W, P, V, step, mode, eos, w_dec, w_ctc, pen, maxlen, minlen, ended_cap, maxlen_cap, out)
    d = {k: _dev(v) for k, v in out.items()}
    best_at = torch.full((U, maxlen_cap), -np.inf, device="cuda")
    best_all = torch.full((U,), -np.inf, device="cuda")
    step_ptr = _i32([2]) if (W + PC) % 2 else None
    _call("espb_beam_select", _ptr(_dev(score)), _ptr(_dev(sc_dec)), _ptr(_dev(sc_ctc)), _ptr(_dev(active)), _ptr(d["n_score"]),
          _ptr(d["n_sc_dec"]), _ptr(d["n_sc_ctc"]), _ptr(d["n_active"]), _ptr(d["n_last_tok"]), _ptr(d["n_parent"]), _ptr(d["bp_parent"]),
          _ptr(d["bp_token"]), _ptr(d["ended_count"]), _ptr(d["ended_step"]), _ptr(d["ended_slot"]), _ptr(d["ended_score"]),
          _ptr(d["ended_dec"]), _ptr(d["ended_ctc"]), ended_cap, _ptr(best_at), _ptr(best_all), _ptr(d["utt_done"]), U, W, P, V,
          step - 2 if step_ptr is not None else step, _ptr(step_ptr), _ptr(_i32(maxlen)), _ptr(_i32(minlen)), eos, w_dec, w_ctc, pen, mode,
          _ptr(_dev(cand_ids)), _ptr(_dev(cand_val)), None if mode == 2 else _ptr(_dev(logp)), _ptr(_dev(part)), _ptr(_dev(valid)), 0,
          maxlen_cap)
    for k, v in ref.items():
        np.testing.assert_array_equal(_bits(d[k]), v.view(np.int32), err_msg=k)
    assert ref["ended_count"][0] > 2 and ref["ended_count"][3] == 1 + W, "the case must append eos winners and every last-step winner"
    assert (ref["n_active"][2 * W:3 * W] == 0).any(), "utterance 2 must have fewer live candidates than beam slots"
