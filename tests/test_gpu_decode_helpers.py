"""-m gpu: the small decode-step helpers of csrc/search_ops.cu (decoder / LM input rows, the LSTM LM's operand gather, per-scorer score
tracking, the weighted score sum, the device step counter and the active-slot count), each called through the C ABI on seeded inputs.

They are copies and one- or two-operation float32 arithmetic, so every comparison is bit for bit against numpy float32, which rounds every
operation and never fuses a multiply into an add:
* axpby: (wa * a) + (wb * b) with both products rounded, as the kernel writes it (__fmul_rn / __fadd_rn).
* e * scale + p (dec_embed, relu_posenc): the compiler may contract it into one FMA, so each element must equal exactly the unfused
  float32 result or the fused one.  The fused one is float32(float64(e) * scale + p): the float64 product is exact (24 + 24 bits), so
  only the final rounding differs from a true FMA, and only when the float64 sum lands exactly on a float32 rounding midpoint.
* Split outputs are compared plane by plane with numpy's tf32_hi / tf32_lo.

Every element a kernel must not read is NaN (embedding rows of other tokens, pe rows of other positions, the ring half and the slots a step
does not use, scores of other hypotheses) and every output starts as a NaN sentinel, so a stray read or a missing write fails, and
elements a kernel must leave alone (pad columns, other steps' history rows) keep their sentinel bit for bit.  Each kernel that takes a
step as `value + *step_ptr` runs with step_ptr NULL and with a device step, so a wrong offset fails.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

NAN = float("nan")


_KEEP = []    # device copies made inline in a call's argument list: only a raw pointer reaches the library, so keep the tensors alive


@pytest.fixture(autouse=True)
def _release_inputs():
    yield
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
    x = np.ascontiguousarray(x, dtype=np.float32)
    hi = (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
    lo = ((x - hi).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
    return hi, lo


def _bits(a):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.ascontiguousarray(a)
    return a.view(np.int32)


def _same_bits(a, b):
    a, b = _bits(a), _bits(b)
    return a.shape == b.shape and np.array_equal(a, b)


def _fma_or_not(got, e, scale, p):
    """Every element of got equals (e * scale) + p rounded twice, or rounded once (FMA)."""
    unf = (e * np.float32(scale)) + p
    fused = (e.astype(np.float64) * np.float64(np.float32(scale)) + p.astype(np.float64)).astype(np.float32)
    g = _bits(got)
    return bool(((g == unf.view(np.int32)) | (g == fused.view(np.int32))).all())


def _step(use_ptr, value, offset):
    """(value passed, step_ptr) for a kernel that must see value + offset."""
    if not use_ptr:
        return value + offset, None
    return value, torch.tensor([offset], dtype=torch.int32, device="cuda")


# ====================================================================================================== decoder / LM input rows
@pytest.mark.parametrize("step_ptr", [False, True])
@pytest.mark.parametrize("n,D", [(1, 64), (20, 256), (64, 520)])
def test_dec_embed_bit_exact(n, D, step_ptr):
    rng = np.random.default_rng(n * D)
    V, P, pos = 50, 40, 17
    tok = rng.integers(0, V, n).astype(np.int32)
    emb = np.full((V, D), np.nan, dtype=np.float32)
    emb[tok] = rng.standard_normal((len(tok), D), dtype=np.float32)          # rows of tokens nobody asks for stay NaN
    pe = np.full((P, D), np.nan, dtype=np.float32)
    pe[pos] = rng.standard_normal(D, dtype=np.float32)
    scale = float(np.sqrt(D))
    val, sp = _step(step_ptr, 5, pos - 5)
    x = torch.full((n * D + 3,), NAN, device="cuda")
    _call("espb_dec_embed_f32", _ptr(_dev(tok)), _ptr(_dev(emb)), _ptr(_dev(pe)), val, _ptr(sp), n, D, scale, _ptr(x))
    torch.cuda.synchronize()
    assert _fma_or_not(x[:n * D].view(n, D), emb[tok], scale, np.broadcast_to(pe[pos], (n, D)))
    assert bool(x[n * D:].isnan().all())


@pytest.mark.parametrize("n,E", [(1, 30), (12, 256), (64, 650)])
def test_gather_rows_split_bit_exact(n, E):
    rng = np.random.default_rng(n + E)
    V = 70
    tok = rng.integers(0, V, n).astype(np.int32)
    tok[0] = V - 1
    emb = np.full((V, E), np.nan, dtype=np.float32)
    emb[tok] = rng.standard_normal((len(tok), E), dtype=np.float32)
    plane = n * E + 5
    out = torch.full((2 * plane,), NAN, device="cuda")
    _call("espb_gather_rows_split_f32", _ptr(_dev(tok)), _ptr(_dev(emb)), n, E, _ptr(out), plane)
    torch.cuda.synchronize()
    hi, lo = _split_np(emb[tok])
    assert _same_bits(out[:n * E].view(n, E), hi) and _same_bits(out[plane:plane + n * E].view(n, E), lo)
    assert bool(out[n * E:plane].isnan().all()) and bool(out[plane + n * E:].isnan().all())


@pytest.mark.parametrize("step_ptr", [False, True])
@pytest.mark.parametrize("with_pe", [False, True])
@pytest.mark.parametrize("n,D", [(1, 64), (30, 256), (60, 516)])
def test_relu_posenc_bit_exact(n, D, with_pe, step_ptr):
    rng = np.random.default_rng(n * D + with_pe)
    P, pos = 30, 9
    x = rng.standard_normal((n, D), dtype=np.float32)
    pe = np.full((P, D), np.nan, dtype=np.float32)
    pe[pos] = rng.standard_normal(D, dtype=np.float32)
    scale = float(np.sqrt(D))
    val, sp = _step(step_ptr, 2, pos - 2)
    xd = torch.full((n * D + 3,), NAN, device="cuda")
    xd[:n * D] = _dev(x).view(-1)
    _call("espb_relu_posenc_f32", _ptr(xd), n, D, _ptr(_dev(pe)) if with_pe else None, val, _ptr(sp), scale)
    torch.cuda.synchronize()
    r = np.maximum(x, np.float32(0))
    got = xd[:n * D].view(n, D)
    if with_pe:
        assert _fma_or_not(got, r, scale, np.broadcast_to(pe[pos], (n, D)))
    else:
        assert _same_bits(got, r)
    assert bool(xd[n * D:].isnan().all())


# ====================================================================================================== weighted score sum, score tracking
@pytest.mark.parametrize("n", [1, 255, 256, 257, 50003])
def test_axpby_bit_exact(n):
    rng = np.random.default_rng(n)
    a = (rng.standard_normal(n) * 30).astype(np.float32)
    b = (rng.standard_normal(n) * 30).astype(np.float32)
    wa, wb = np.float32(0.7), np.float32(0.3)
    out = torch.full((n + 4,), NAN, device="cuda")
    _call("espb_axpby_f32", _ptr(_dev(a)), float(wa), _ptr(_dev(b)), float(wb), _ptr(out), n)
    torch.cuda.synchronize()
    assert _same_bits(out[:n], (wa * a) + (wb * b))
    assert bool(out[n:].isnan().all())


@pytest.mark.parametrize("step_ptr", [False, True])
@pytest.mark.parametrize("with_b", [False, True])
def test_track_scores_bit_exact(with_b, step_ptr):
    """new[ns] = prev[parent] + logp[parent][tok] where bp_parent[step][ns] >= 0, else 0; also recorded as hist[step][ns].  With logp_b NULL
    new_b / hist_b are left untouched."""
    rng = np.random.default_rng(3 + with_b)
    n, V, steps, step = 37, 50, 6, 4
    parent = rng.integers(0, n, n).astype(np.int32)
    tok = rng.integers(0, V, n).astype(np.int32)
    bp = np.full((steps, n), -7, dtype=np.int32)          # other steps' rows: reading one would zero the scores
    bp[step] = np.where(rng.random(n) < 0.3, -1, parent)
    ok = bp[step] >= 0
    lp = [np.full((n, V), np.nan, dtype=np.float32) for _ in range(2)]
    prev = [np.full(n, np.nan, dtype=np.float32) for _ in range(2)]
    for k in range(2):
        lp[k][parent[ok], tok[ok]] = rng.standard_normal(int(ok.sum()), dtype=np.float32) - 3
        prev[k][parent[ok]] = rng.standard_normal(int(ok.sum()), dtype=np.float32) * 20 - 40
    new = [torch.full((n,), NAN, device="cuda") for _ in range(2)]
    hist = [torch.full((steps, n), NAN, device="cuda") for _ in range(2)]
    val, sp = _step(step_ptr, 1, step - 1)
    _call("espb_track_scores_f32", _ptr(_dev(parent)), _ptr(_dev(tok)), _ptr(_dev(bp)), _ptr(_dev(lp[0])), _ptr(_dev(lp[1])) if with_b else None, V,
          _ptr(_dev(prev[0])), _ptr(_dev(prev[1])) if with_b else None, _ptr(new[0]), _ptr(new[1]), _ptr(hist[0]), _ptr(hist[1]), val, _ptr(sp), n)
    torch.cuda.synchronize()
    for k in range(2 if with_b else 1):
        ref = np.zeros(n, dtype=np.float32)
        ref[ok] = prev[k][parent[ok]] + lp[k][parent[ok], tok[ok]]
        assert _same_bits(new[k], ref)
        h = hist[k].cpu().numpy()
        assert _same_bits(h[step], ref)
        assert np.isnan(np.delete(h, step, axis=0)).all()
    if not with_b:
        assert bool(new[1].isnan().all()) and bool(hist[1].isnan().all())


# ====================================================================================================== LSTM LM operand gather
@pytest.mark.parametrize("step_ptr", [False, True])
@pytest.mark.parametrize("pos", [0, 1, 6])
@pytest.mark.parametrize("L", [1, 2, 3])
def test_rnnlm_gather_bit_exact(L, pos, step_ptr):
    """Layer 0's operand row is [emb(tok) | pad | parent h of layer 0 | pad], layer l's [input half (not written here) | parent h | pad];
    the parent is anc[s][pos - 1] in ring (pos - 1) & 1, and zeros at pos 0."""
    rng = np.random.default_rng(L * 10 + pos)
    n, V, E, Ep, H, Hp, anc_ld = 6, 40, 30, 32, 50, 52, 8
    tok = rng.integers(0, V, n).astype(np.int32)
    emb = np.full((V, E), np.nan, dtype=np.float32)
    emb[tok] = rng.standard_normal((n, E), dtype=np.float32)
    anc = rng.integers(0, n - 1, (n, anc_ld)).astype(np.int32)    # slot n - 1 is nobody's parent: its state stays NaN
    ring = np.full((2, L, n, Hp), np.nan, dtype=np.float32)        # the other ring and the pad columns must not be read
    par = anc[:, pos - 1] if pos > 0 else None
    if pos > 0:
        ring[(pos - 1) & 1, :, np.unique(par), :H] = rng.standard_normal((len(np.unique(par)), L, H), dtype=np.float32)
    kp0, kp1 = Ep + Hp, 2 * Hp
    total = 2 * n * kp0 + 2 * (L - 1) * n * kp1
    xs = torch.full((total + 4,), NAN, device="cuda")
    val, sp = _step(step_ptr, 0 if pos == 0 else 1, pos - (0 if pos == 0 else 1))
    _call("espb_rnnlm_gather_f32", _ptr(_dev(tok)), _ptr(_dev(emb)), E, Ep, _ptr(_dev(anc)), anc_ld, val, _ptr(sp), _ptr(_dev(ring)), L, n, H, Hp,
          _ptr(xs))
    torch.cuda.synchronize()
    ref = np.full(total + 4, np.nan, dtype=np.float32)

    def put(off, kp, col, vals):      # split [2][n][kp] operand at off, columns col.. of every row
        hi, lo = _split_np(vals)
        w = vals.shape[1]
        for s in range(n):
            ref[off + s * kp + col:off + s * kp + col + w] = hi[s]
            ref[off + n * kp + s * kp + col:off + n * kp + s * kp + col + w] = lo[s]

    put(0, kp0, 0, emb[tok])
    for l in range(L):
        h = ring[(pos - 1) & 1, l, par, :H] if pos > 0 else np.zeros((n, H), dtype=np.float32)
        if l == 0:
            put(0, kp0, Ep, h)
        else:
            put(2 * n * kp0 + 2 * (l - 1) * n * kp1, kp1, Hp, h)
    assert _same_bits(xs, ref)


# ====================================================================================================== device step counter, active count
def test_step_inc():
    step = torch.tensor([41, -5], dtype=torch.int32, device="cuda")
    _call("espb_step_inc_i32", _ptr(step))
    _call("espb_step_inc_i32", _ptr(step))
    torch.cuda.synchronize()
    assert step.tolist() == [43, -5]


@pytest.mark.parametrize("n", [0, 1, 257, 4096])
def test_count_active(n):
    rng = np.random.default_rng(n)
    act = rng.choice(np.array([0, 1, 2, -1], dtype=np.int32), n + 5, p=[0.5, 0.3, 0.1, 0.1])   # any nonzero value is active
    act[n:] = 1                                                                                 # past n: not counted
    out = torch.tensor([-99, -99], dtype=torch.int32, device="cuda")
    _call("espb_count_active_i32", _ptr(_dev(act)), n, _ptr(out))
    torch.cuda.synchronize()
    assert out.tolist() == [int((act[:n] != 0).sum()), -99]
