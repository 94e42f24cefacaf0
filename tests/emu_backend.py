"""TEST INFRASTRUCTURE: a torch-CPU emulation of the C-ABI entry points the encoder classes call, so that the HOST logic of
espnet_b200 (GEMM descriptors: strides / offsets / batch dims, buffer pitches, layouts, the order of kernels) can be tested on a box
without a GPU.  Each function restates the contract of the CUDA kernel of the same name (espnet_b200/csrc/*.cu; the GEMM follows
gemm_simt_kernel, which is itself the validator of the tensor-core kernels).  Nothing in the product imports this file; it is
installed by monkey-patching `call` / `ptr` / `gemm` inside the espnet_b200 modules for the duration of a test.
"""
import math

import torch

MASK = -8192  # 0xFFFFE000 as int32


def tf32_hi(x):
    return (x.contiguous().view(torch.int32) & MASK).view(torch.float32)


def tf32_lo(x, hi):
    return ((x - hi).contiguous().view(torch.int32) & MASK).view(torch.float32)


def _flat(t):
    assert t.is_contiguous()
    return t.view(-1)


def _store(flat, off, v, split, plane):
    if split:
        hi = tf32_hi(v)
        flat[off] = hi
        flat[off + plane] = tf32_lo(v, hi)
    else:
        flat[off] = v


def gemm(M, N, K, A, a_plane, lda, B, b_plane, ldb, C, ldc, *, c_plane=0, split_out=False, bias=None, R=None, ldr=0, alpha=1.0, act=0,
         nbx=1, nby=1, sa=(0, 0), sb=(0, 0), sc=(0, 0), sr=(0, 0), kob=0, a_mode=0, conv=(0, 0, 0), a_off=0, b_off=0, c_off=0, r_off=0,
         sbias_x=0, bias_off=0, band_t=0, force=None):
    """EspbGemmDesc semantics (gemm.cu: load_a / load_b / gemm_simt_kernel epilogue).  band_t only lets the kernels skip tiles nobody
    reads, so computing everything is a valid superset."""
    Af, Bf, Cf = _flat(A), _flat(B), _flat(C)
    m = torch.arange(M).view(M, 1)
    n = torch.arange(N).view(N, 1)
    k = torch.arange(K).view(1, K)
    rows, cols = torch.arange(M).view(M, 1), torch.arange(N).view(1, N)
    for by in range(nby):
        for bx in range(nbx):
            if a_mode == 0:
                ko, ki = (k // (kob * 32), k % (kob * 32)) if kob > 0 else (0, k)
                off = a_off + by * sa[1] + (bx + ko) * sa[0] + m * lda + ki
                Am = Af[off] + Af[off + a_plane]
            else:  # conv2 over [b][plane*4 + pt*2 + pf][F1h][T1h][C]
                t1h, f1h, cin = conv
                tap, c = k // cin, k % cin
                kt, kf = tap // 3, tap % 3
                par = (kt & 1) * 2 + (kf & 1)
                tt, ff = m + (kt >> 1), bx + (kf >> 1)
                ok = (tt < t1h) & (ff < f1h)
                sub = f1h * t1h * cin
                off = a_off + by * 8 * sub + (torch.clamp(ff, max=f1h - 1) * t1h + torch.clamp(tt, max=t1h - 1)) * cin + c
                Am = torch.where(ok, Af[off + par * sub] + Af[off + (4 + par) * sub], torch.zeros(()))
            offb = b_off + by * sb[1] + bx * sb[0] + n * ldb + k
            Bm = Bf[offb] + Bf[offb + b_plane]
            v = (Am.double() @ Bm.double().t()).float()
            if bias is not None:
                v = v + _flat(bias)[bias_off + bx * sbias_x + cols]
            if act == 1:
                v = torch.relu(v)
            elif act == 2:
                v = v / (1.0 + torch.exp(-v))
            v = v * alpha
            if R is not None:
                v = v + _flat(R)[r_off + by * sr[1] + bx * sr[0] + rows * ldr + cols]
            _store(Cf, c_off + by * sc[1] + bx * sc[0] + rows * ldc + cols, v, split_out, c_plane)
    return True


def ptr(t):
    return t


def _split_tf32(x, n, out, plane):
    _store(_flat(out), torch.arange(n), _flat(x)[:n], True, plane)


def _layernorm(x, rows, D, gamma, beta, eps, out_plain, out_split, split_plane):
    xr = _flat(x)[: rows * D].view(rows, D)
    mean = xr.sum(-1, keepdim=True) / D
    var = ((xr - mean) ** 2).sum(-1, keepdim=True) / D
    y = ((xr - mean) * (1.0 / torch.sqrt(var + eps)) * gamma + beta).reshape(-1)   # clone: out_plain may alias x
    if out_split is not None:
        _store(_flat(out_split), torch.arange(rows * D), y, True, split_plane)
    if out_plain is not None:
        _flat(out_plain)[: rows * D] = y


def _conv1_relu(feats, B, Tf, F, w, bias, C, out, T1, F1, T1h, F1h):
    x = feats.view(B, 1, Tf, F)
    y = torch.relu(torch.nn.functional.conv2d(x, w.view(C, 1, 3, 3), bias, stride=2))   # [B][C][T1][F1]
    sub = F1h * T1h * C
    of = _flat(out)
    b, c, t1, f1 = torch.meshgrid(torch.arange(B), torch.arange(C), torch.arange(T1), torch.arange(F1), indexing="ij")
    par = (t1 & 1) * 2 + (f1 & 1)
    off = b * 8 * sub + par * sub + ((f1 >> 1) * T1h + (t1 >> 1)) * C + c
    _store(of, off, y, True, 4 * sub)


def _qu_qv(qkv, qkv_plane, M, D, pos_u, pos_v, qu, qv, out_plane):
    qf = _flat(qkv)
    off = torch.arange(M).view(M, 1) * 3 * D + torch.arange(D).view(1, D)
    q = qf[off] + qf[off + qkv_plane]
    o = torch.arange(M * D).view(M, D)
    _store(_flat(qu), o, q + pos_u.view(1, D), True, out_plane)
    _store(_flat(qv), o, q + pos_v.view(1, D), True, out_plane)


def _v_transpose(qkv, qkv_plane, B, Tmax, D, H, lens, vt, vt_plane, Tp):
    qf, dk = _flat(qkv), D // H
    b, h, d, t = torch.meshgrid(torch.arange(B), torch.arange(H), torch.arange(dk), torch.arange(Tp), indexing="ij")
    ok = t < lens.view(B, 1, 1, 1).long()
    src = (b * Tmax + torch.clamp(t, max=Tmax - 1)) * 3 * D + 2 * D + h * dk + d
    v = torch.where(ok, qf[src] + qf[src + qkv_plane], torch.zeros(()))
    _store(_flat(vt), ((b * H + h) * dk + d) * Tp + t, v, True, vt_plane)


def _softmax_rows(scores, lens_rows, Tp, probs, plane):
    """scores [R][Tp] already scaled; keys >= len -> probability 0; split store."""
    Rn = scores.shape[0]
    j = torch.arange(Tp).view(1, Tp)
    ok = j < lens_rows.view(Rn, 1)
    s = torch.where(ok, scores, torch.full((), float("-inf")))
    p = torch.where(ok, torch.softmax(s, dim=-1), torch.zeros(()))
    _store(_flat(probs), torch.arange(Rn * Tp).view(Rn, Tp), p, True, plane)


def _relpos_softmax(ac, bd, B, H, T, Tp, Rp, lens, sqrt_dk, probs, plane):
    a = _flat(ac)[: B * H * T * Tp].view(B * H * T, Tp)
    bdv = _flat(bd)[: B * H * T * Rp].view(B * H * T, Rp)
    i = (torch.arange(B * H * T) % T).view(-1, 1)
    j = torch.arange(Tp).view(1, Tp)
    col = torch.clamp(T - 1 - i + j, max=Rp - 1)                      # rel_shift: bd[i][T-1-i+j]
    s = (a + torch.gather(bdv, 1, col)) / sqrt_dk
    _softmax_rows(s, lens.long().repeat_interleave(H * T), Tp, probs, plane)


def _masked_softmax(sc, B, H, T, Tp, lens, sqrt_dk, probs, plane):
    s = _flat(sc)[: B * H * T * Tp].view(B * H * T, Tp) / sqrt_dk
    _softmax_rows(s, lens.long().repeat_interleave(H * T), Tp, probs, plane)


def _flash_attn(q, q_off, q_plane, ldq, k, k_off, k_plane, ldk, vt, vt_plane, Tp, bd, Rp, lens, B, H, T, dk, out, out_plane, ldo):
    """flash_attn_kernel: out[b,i,h] = softmax_{j<len}((q.k + bd[b,h,i,T-1-i+j]) / sqrt(dk)) v; rows i >= len of an utterance are padding
    (zero for whole 256-row blocks beyond len, finite values otherwise -- compared only below len)."""
    qf, kf, vf, of = _flat(q), _flat(k), _flat(vt), _flat(out)
    bdv = _flat(bd)[: B * H * T * Rp].view(B, H, T, Rp) if bd is not None else None
    c = torch.arange(dk)
    for b in range(B):
        n = int(lens[b])
        rows = (b * T + torch.arange(T)).view(T, 1)
        for h in range(H):
            qo = q_off + rows * ldq + h * dk + c
            Q = qf[qo] + qf[qo + q_plane]
            ko = k_off + rows[:n] * ldk + h * dk + c
            K = kf[ko] + kf[ko + k_plane]
            vo = ((b * H + h) * dk + c.view(dk, 1)) * Tp + torch.arange(n).view(1, n)
            V = (vf[vo] + vf[vo + vt_plane]).t()
            S = Q @ K.t()
            if bdv is not None:
                i, j = torch.arange(T).view(T, 1), torch.arange(n).view(1, n)
                S = S + bdv[b, h][i, T - 1 - i + j]
            O = torch.softmax(S / math.sqrt(dk), dim=-1) @ V
            _store(of, rows * ldo + h * dk + c, O, True, out_plane)


def _glu_dwconv_bn_swish(y, B, Tmax, C, lens, dw_w, dw_b, K, bn_a, bn_b, out, out_plane):
    yv = _flat(y)[: B * Tmax * 2 * C].view(B, Tmax, 2 * C)
    t = torch.arange(Tmax).view(1, Tmax, 1)
    valid = t < lens.view(B, 1, 1).long()
    g = torch.where(valid, yv[..., :C] * (1.0 / (1.0 + torch.exp(-yv[..., C:]))), torch.zeros(()))
    z = torch.nn.functional.conv1d(g.transpose(1, 2), dw_w.view(C, 1, K), dw_b, padding=(K - 1) // 2, groups=C).transpose(1, 2)
    z = z * bn_a + bn_b
    z = z / (1.0 + torch.exp(-z))
    z = torch.where(valid, z, torch.zeros(()))
    _store(_flat(out), torch.arange(B * Tmax * C).view(B, Tmax, C), z, True, out_plane)


def _cbe_build_chunks(xs, N, Tt, D, nb, block, hop, pe, pos0, ctx0, scale, prev_addin, addin_out, chunks):
    x = _flat(xs)[: N * Tt * D].view(N, Tt, D)
    c = chunks.view(N, nb, block + 2, D)
    c.zero_()
    pev = pe.view(-1, D)
    sc = torch.tensor(scale, dtype=torch.float32)
    prev = prev_addin.view(N, D).clone() if prev_addin is not None else None
    for i in range(nb):
        cur = i * hop
        ln = min(block, Tt - cur)
        seg = x[:, cur:cur + ln]
        addin = (seg.sum(1) / ln) * sc + pev[ctx0 + i]
        c[:, i, 1:ln + 1] = seg * sc + pev[pos0 + cur: pos0 + cur + ln]
        c[:, i, block + 1] = addin
        c[:, i, 0] = addin if prev is None else prev
        prev = addin
    addin_out.view(N, D).copy_(prev)


def _cbe_ctx_propagate(x, N, nb, S, D, past_ctx, next_ctx, layer, L):
    xv = x.view(N, nb, S, D)
    last = xv[:, :, S - 1].clone()
    next_ctx.view(N, L, D)[:, layer] = last[:, nb - 1]
    xv[:, 0, 0] = past_ctx.view(N, L, D)[:, layer] if past_ctx is not None else last[:, 0]
    if nb > 1:
        xv[:, 1:, 0] = last[:, :-1]


def _zero_rows(x, row0, every, count, D, plane, nplanes):
    f = _flat(x)
    for q in range(nplanes):
        for k in range(count):
            o = q * plane + (row0 + k * every) * D
            f[o:o + D] = 0.0


def _gather_rows(src, N, src_rows, idx, nout, D, out):
    out.view(N, nout, D).copy_(_flat(src)[: N * src_rows * D].view(N, src_rows, D)[:, idx.view(-1)[:nout].long()])


_TABLE = {"espb_cbe_build_chunks_f32": _cbe_build_chunks, "espb_cbe_ctx_propagate_f32": _cbe_ctx_propagate, "espb_zero_rows_f32": _zero_rows,
          "espb_gather_rows_f32": _gather_rows, "espb_split_tf32_f32": _split_tf32, "espb_layernorm_f32": _layernorm, "espb_conv1_relu_f32": _conv1_relu, "espb_qu_qv_f32": _qu_qv,
          "espb_v_transpose_f32": _v_transpose, "espb_relpos_softmax_f32": _relpos_softmax, "espb_masked_softmax_f32": _masked_softmax,
          "espb_flash_attn_f32": _flash_attn, "espb_glu_dwconv_bn_swish_f32": _glu_dwconv_bn_swish}
calls = []   # names of the emulated entry points, in call order (tests can assert on the sequence)


def call(name, *args):
    if name not in _TABLE:
        raise NotImplementedError(f"emu_backend: {name} is not emulated")
    calls.append(name)
    _TABLE[name](*args)


def install(monkeypatch):
    """Route the encoder-side modules of espnet_b200 through the emulation (CPU tensors)."""
    import espnet_b200.encoder as enc
    import espnet_b200.ops as ops
    import espnet_b200.streaming_encoder as senc
    import espnet_b200.transformer_encoder as tenc

    del calls[:]
    monkeypatch.setattr(senc, "gemm", gemm, raising=True)
    for mod in (ops, enc, tenc, senc):
        monkeypatch.setattr(mod, "call", call, raising=True)
        monkeypatch.setattr(mod, "ptr", ptr, raising=True)
    monkeypatch.setattr(ops, "gemm", gemm, raising=True)
    monkeypatch.setattr(enc, "gemm", gemm, raising=True)
    monkeypatch.setattr(tenc, "gemm", gemm, raising=True)
    monkeypatch.setattr(ops, "new_split", lambda *shape, device="cpu": torch.zeros((2,) + tuple(shape), dtype=torch.float32), raising=True)
    monkeypatch.setattr(enc, "new_split", ops.new_split, raising=True)


# ------------------------------------------------------------------------------------------------ CTC head / decoder / search entry points
# Restated with plain loops (test sizes are a few utterances x a few beam slots x tens of frames).
LOGZERO = -10000000000.0


def _lae(a, b):
    m = max(a, b)
    return m + math.log(math.exp(a - m) + math.exp(b - m))


def _step(step_ptr):
    return int(step_ptr.view(-1)[0]) if step_ptr is not None else 0


def _log_softmax_rows(x, rows, ld, V):
    xv = torch.as_strided(x, (rows, V), (ld, 1), x.storage_offset())
    xv.copy_(torch.log_softmax(xv, dim=-1))


def _argmax_rows(x, rows, ld, V, out):
    xv = torch.as_strided(x, (rows, V), (ld, 1), x.storage_offset())
    _flat(out)[:rows] = torch.argmax(xv, dim=-1).to(torch.int32)


def _ctc_collapse(am, B, Tmax, lens, blank, out_ids, out_len):
    a, o = am.view(B, Tmax), out_ids.view(B, Tmax)
    for b in range(B):
        n = 0
        for t in range(int(lens[b])):
            v = int(a[b, t])
            if v != blank and (t == 0 or int(a[b, t - 1]) != v):
                o[b, n] = v
                n += 1
        out_len.view(-1)[b] = n


def _rows_topk(x, rows, ld, V, scale, k, ids, vals):
    xv = torch.as_strided(x, (rows, V), (ld, 1), x.storage_offset()) * scale
    for r in range(rows):
        i = torch.sort(-xv[r], stable=True).indices[:k]   # descending, ties (-inf included) -> lower index
        ids.view(-1)[r * k:(r + 1) * k] = i.to(torch.int32)
        vals.view(-1)[r * k:(r + 1) * k] = xv[r][i]


def _dec_embed(last_tok, emb, pe, pos, step_ptr, n, D, scale, x):
    p = pos + _step(step_ptr)
    x.view(n, D).copy_(emb[last_tok.view(-1)[:n].long()] * scale + pe[p])


def _dec_self_attn(qkv, kc, vc, anc, anc_ld, n, D, H, pos, step_ptr, max_pos, ctx, ctx_plane):
    pos = pos + _step(step_ptr)
    dk = D // H
    q3 = qkv.view(n, 3 * D)
    kc[pos].view(n, D).copy_(q3[:, D:2 * D])
    vc[pos].view(n, D).copy_(q3[:, 2 * D:])
    an = anc.view(n, anc_ld)
    out = torch.zeros(n, D)
    for s in range(n):
        rows = [int(an[s, j]) for j in range(pos)] + [s]
        K = torch.stack([kc[j].view(n, D)[rows[j]] for j in range(pos + 1)])     # [pos+1][D]
        Vv = torch.stack([vc[j].view(n, D)[rows[j]] for j in range(pos + 1)])
        for h in range(H):
            sl = slice(h * dk, (h + 1) * dk)
            sc = (K[:, sl] @ q3[s, sl]) / math.sqrt(dk)
            out[s, sl] = torch.softmax(sc, dim=0) @ Vv[:, sl]
    _store(_flat(ctx), torch.arange(n * D), out.view(-1), True, ctx_plane)


def _dec_src_attn(q, kmem, vmem, U, Tmax, lens, W, D, H, ctx, ctx_plane):
    dk = D // H
    qv, km, vm = q.view(U * W, D), kmem.view(U, H, Tmax, dk), vmem.view(U, H, Tmax, dk)
    out = torch.zeros(U * W, D)
    for u in range(U):
        T = int(lens[u])
        for h in range(H):
            sl = slice(h * dk, (h + 1) * dk)
            sc = (qv[u * W:(u + 1) * W, sl] @ km[u, h, :T].t()) / math.sqrt(dk)      # no memory mask beyond the utterance's own frames
            out[u * W:(u + 1) * W, sl] = torch.softmax(sc, dim=-1) @ vm[u, h, :T]
    _store(_flat(ctx), torch.arange(U * W * D), out.view(-1), True, ctx_plane)


def _x(logp, u, Tmax, V, token_major):
    """Returns f(t, c) reading the posterior of utterance u in either layout."""
    base = logp.view(-1)[u * Tmax * V:(u + 1) * Tmax * V]
    return (lambda t, c: float(base[c * Tmax + t])) if token_major else (lambda t, c: float(base[t * V + c]))


def _ctc_init_state(logp, U, Tmax, V, lens, blank, W, r, s_prev):
    rr = r.view(U * W, Tmax, 4)
    for s in range(U * W):
        u = s // W
        x, T, c = _x(logp, u, Tmax, V, 0), int(lens[u]), 0.0
        for t in range(Tmax):
            if t < T:
                c = float(torch.tensor(c, dtype=torch.float32) + torch.tensor(x(t, blank), dtype=torch.float32))
            rb = c if t < T else LOGZERO
            rr[s, t] = torch.tensor([LOGZERO, rb, _lae(LOGZERO, rb), 0.0])
        s_prev.view(-1)[s] = 0.0


def _ctc_extend_state(logp, T_new, V, blank, n, r_old, T_old, r_new):
    ro, rn, lp = r_old.reshape(-1)[: n * T_old * 4].view(n, T_old, 4), r_new.view(-1)[: n * T_new * 4].view(n, T_new, 4), logp.view(-1)[: T_new * V].view(T_new, V)
    for s in range(n):
        rn[s, :T_old] = ro[s]
        rb = ro[s, T_old - 1, 1].clone()
        for t in range(max(T_old, 1), T_new):
            rb = rb + lp[t, blank]
            rn[s, t] = torch.tensor([LOGZERO, float(rb), _lae(LOGZERO, float(rb)), 0.0])


def _transpose_tv(x, U, Tmax, V, xt):
    xt.view(U, V, Tmax).copy_(x.view(U, Tmax, V).transpose(1, 2))


def _log_psi(x, T, blank, eos, rp, c, last, out_len):
    if T <= 0:
        return LOGZERO
    if c == eos:
        return float(rp[T - 1, 2])
    if c == blank:
        return LOGZERO
    start = max(out_len, 1)
    terms = [(float(rp[t - 1, 1]) if c == last else float(rp[t - 1, 2])) + x(t, c) for t in range(start, T)]
    terms.append(x(0, c) if out_len == 0 else LOGZERO)
    return float(torch.logsumexp(torch.tensor(terms, dtype=torch.float64), dim=0))


def _ctc_score_cands(logp, U, Tmax, V, lens, blank, eos, W, r_prev, s_prev, last_tok, out_len, step_ptr, cand, P, part, psi, valid, token_major):
    out_len += _step(step_ptr)
    rp, cd = r_prev.view(U * W, Tmax, 4), cand.view(U * W, P)
    for s in range(U * W):
        u = s // W
        x = _x(logp, u, Tmax, V, token_major)
        for j in range(P + 1):
            c = int(cd[s, j]) if j < P else eos
            ok = 0 if (j == P and bool((cd[s] == eos).any())) else 1
            v = _log_psi(x, int(lens[u]), blank, eos, rp[s], c, int(last_tok.view(-1)[s]), out_len)
            i = s * (P + 1) + j
            psi.view(-1)[i], part.view(-1)[i], valid.view(-1)[i] = v, v - float(s_prev.view(-1)[s]), ok


def _ctc_score_dense(logp, U, Tmax, V, lens, blank, eos, W, r_prev, s_prev, last_tok, out_len, part):
    rp = r_prev.view(U * W, Tmax, 4)
    for s in range(U * W):
        u = s // W
        x = _x(logp, u, Tmax, V, 0)
        for c in range(V):
            part.view(-1)[s * V + c] = _log_psi(x, int(lens[u]), blank, eos, rp[s], c, int(last_tok.view(-1)[s]), out_len) - float(s_prev.view(-1)[s])


def _ctc_advance(logp, U, Tmax, V, lens, blank, eos, W, r_prev, parent, par_last_tok, new_tok, new_active, out_len, step_ptr, r_new, s_new,
                 token_major):
    out_len += _step(step_ptr)
    rp, ro = r_prev.view(-1, Tmax, 4), r_new.view(U * W, Tmax, 4)      # parents may come from a larger set of previous slots (scorer protocol)
    Z4 = torch.tensor([LOGZERO, LOGZERO, _lae(LOGZERO, LOGZERO), 0.0])
    for s in range(U * W):
        u, c, act = s // W, int(new_tok.view(-1)[s]), int(new_active.view(-1)[s])
        if not act or c == eos or c == blank:
            ro[s] = Z4
            s_new.view(-1)[s] = LOGZERO if (act and c == blank) else 0.0
            continue
        p, T = int(parent.view(-1)[s]), int(lens[u])
        x, last = _x(logp, u, Tmax, V, token_major), int(par_last_tok.view(-1)[p])
        start = max(out_len, 1)
        rn, rb = (x(0, c) if out_len == 0 else LOGZERO), LOGZERO
        ro[s] = Z4
        if start - 1 < T:      # a prefix longer than the encoder output keeps an all-logzero state (ctc_advance_kernel)
            ro[s, start - 1] = torch.tensor([rn, rb, _lae(rn, rb), 0.0])
        for t in range(start, T):
            phi = float(rp[p, t - 1, 1]) if c == last else float(rp[p, t - 1, 2])
            rn, rb = _lae(rn, phi) + x(t, c), _lae(rn, rb) + x(t, blank)
            ro[s, t] = torch.tensor([rn, rb, _lae(rn, rb), 0.0])
        s_new.view(-1)[s] = _log_psi(x, T, blank, eos, rp[p], c, last, out_len)


def _beam_select(score, sc_dec, sc_ctc, active, n_score, n_sc_dec, n_sc_ctc, n_active, n_last_tok, n_parent, bp_parent, bp_token, e_count,
                 e_step, e_slot, e_score, e_dec, e_ctc, ended_cap, best_at, best_all, utt_done, U, W, P, V, step, step_ptr, maxlen, minlen, eos,
                 w_dec, w_ctc, penalty, mode, cand_ids, cand_val, logp_dec, part, valid, end_detect, maxlen_cap):
    step += _step(step_ptr)
    f32 = lambda v: float(torch.tensor(v, dtype=torch.float32))  # noqa: E731
    w_dec, w_ctc, penalty = f32(w_dec), f32(w_ctc), f32(penalty)   # the kernel takes them as float
    PC = P + 1 if mode == 1 else P
    fl = lambda t: t.view(-1)  # noqa: E731
    for u in range(U):
        done = int(fl(utt_done)[u]) != 0
        tot = []
        for ci in range(W * PC):
            w, j = divmod(ci, PC)
            s, t = u * W + w, float("-inf")
            if not done and int(fl(active)[s]):
                if mode == 1:
                    if int(fl(valid)[s * PC + j]):
                        dec = float(fl(cand_val)[s * P + j]) if j < P else f32(w_dec * float(fl(logp_dec)[s * V + eos]))
                        t = f32(f32(f32(dec + penalty) + f32(w_ctc * float(fl(part)[s * PC + j]))) + float(fl(score)[s]))
                else:
                    t = f32(f32(float(fl(cand_val)[s * P + j]) + penalty) + float(fl(score)[s]))
            tot.append(t)
        mlen = int(fl(maxlen)[u])
        last_step, step_best = step == mlen - 1, float("-inf")
        for k in range(W):
            ns = u * W + k
            bp = step * U * W + ns
            best = max(tot) if tot else float("-inf")
            if best == float("-inf"):
                fl(n_active)[ns], fl(n_score)[ns], fl(n_sc_dec)[ns], fl(n_sc_ctc)[ns], fl(n_last_tok)[ns] = 0, 0.0, 0.0, 0.0, eos
                fl(n_parent)[ns], fl(bp_parent)[bp], fl(bp_token)[bp] = ns, -1, eos
                continue
            bidx = tot.index(best)               # ties -> lower flat index
            tot[bidx] = float("-inf")
            w, j = divmod(bidx, PC)
            s = u * W + w
            tok = eos if (mode == 1 and j == P) else int(fl(cand_ids)[s * P + j])
            dlogp = float(fl(logp_dec)[s * V + tok]) if mode != 2 else 0.0
            cpart = float(fl(part)[s * PC + j]) if mode == 1 else (float(fl(part)[s * V + tok]) if mode == 2 else 0.0)
            ndec, nctc = f32(float(fl(sc_dec)[s]) + dlogp), f32(float(fl(sc_ctc)[s]) + cpart)
            fl(bp_parent)[bp], fl(bp_token)[bp], fl(n_parent)[ns] = s, tok, s
            fl(n_score)[ns], fl(n_sc_dec)[ns], fl(n_sc_ctc)[ns], fl(n_last_tok)[ns] = best, ndec, nctc, tok
            ended = last_step or tok == eos
            fl(n_active)[ns] = 0 if ended else 1
            if ended and step >= int(fl(minlen)[u]):
                e = int(fl(e_count)[u])
                if e < ended_cap:
                    o = u * ended_cap + e
                    fl(e_step)[o], fl(e_slot)[o], fl(e_score)[o], fl(e_dec)[o], fl(e_ctc)[o] = step, ns, best, ndec, nctc
                    fl(e_count)[u] = e + 1
                step_best = max(step_best, best)
        if not done:
            if end_detect:
                if step < maxlen_cap:
                    fl(best_at)[u * maxlen_cap + step] = step_best
                ball = max(float(fl(best_all)[u]), step_best)
                fl(best_all)[u] = ball
                count = 0
                for m in range(3):
                    j = step - m - 2
                    if 0 <= j < maxlen_cap:
                        b = float(fl(best_at)[u * maxlen_cap + j])
                        if b > float("-inf") and b - ball < -10.0:
                            count += 1
                if count == 3:
                    fl(utt_done)[u] = 1
            if last_step:
                fl(utt_done)[u] = 1


def _anc_update(anc, n_anc, anc_ld, parent, pos, step_ptr, n):
    pos += _step(step_ptr)
    a, na = anc.view(n, anc_ld), n_anc.view(n, anc_ld)
    for s in range(n):
        p = int(parent.view(-1)[s])
        na[s, :pos] = a[p, :pos]
        na[s, pos] = p


def _step_inc(step):
    step.view(-1)[0] += 1


def _count_active(active, n, out):
    out.view(-1)[0] = int((active.view(-1)[:n] != 0).sum())


_TABLE.update({"espb_log_softmax_rows_f32": _log_softmax_rows, "espb_argmax_rows_f32": _argmax_rows, "espb_ctc_collapse_i32": _ctc_collapse,
               "espb_rows_topk_f32": _rows_topk, "espb_dec_embed_f32": _dec_embed, "espb_dec_self_attn_f32": _dec_self_attn,
               "espb_dec_src_attn_f32": _dec_src_attn, "espb_ctc_init_state_f32": _ctc_init_state, "espb_ctc_extend_state_f32": _ctc_extend_state, "espb_transpose_tv_f32": _transpose_tv,
               "espb_ctc_score_cands_f32": _ctc_score_cands, "espb_ctc_score_dense_f32": _ctc_score_dense, "espb_ctc_advance_f32": _ctc_advance,
               "espb_beam_select": _beam_select, "espb_anc_update_i32": _anc_update, "espb_step_inc_i32": _step_inc,
               "espb_count_active_i32": _count_active})


def _gather_rows_split(tok, emb, n, E, out, plane):
    _store(_flat(out), torch.arange(n * E).view(n, E), emb.view(-1, E)[tok.view(-1)[:n].long()], True, plane)


def _relu_posenc(x, n, D, pe, pos, step_ptr, scale):
    pos += _step(step_ptr)
    xv = _flat(x)[: n * D].view(n, D)
    v = torch.relu(xv)
    if pe is not None:
        v = v * torch.tensor(scale, dtype=torch.float32) + pe.view(-1, D)[pos]
    xv.copy_(v)


def _axpby(a, wa, b, wb, out, n):
    f = lambda w: torch.tensor(w, dtype=torch.float32)  # noqa: E731
    _flat(out)[:n] = f(wa) * _flat(a)[:n] + f(wb) * _flat(b)[:n]


def _track_scores(parent, tok, bp_parent, logp_a, logp_b, V, prev_a, prev_b, new_a, new_b, hist_a, hist_b, step, step_ptr, n):
    step += _step(step_ptr)
    for ns in range(n):
        ok = int(bp_parent.view(-1)[step * n + ns]) >= 0
        p, t = int(parent.view(-1)[ns]), int(tok.view(-1)[ns])
        for lp, prev, new, hist in ((logp_a, prev_a, new_a, hist_a), (logp_b, prev_b, new_b, hist_b)):
            if lp is None:
                continue
            v = (prev.view(-1)[p] + lp.view(-1)[p * V + t]) if ok else torch.tensor(0.0)
            new.view(-1)[ns] = v
            hist.view(-1)[step * n + ns] = v


_TABLE.update({"espb_gather_rows_split_f32": _gather_rows_split, "espb_relu_posenc_f32": _relu_posenc, "espb_axpby_f32": _axpby,
               "espb_track_scores_f32": _track_scores})


def install_search(monkeypatch):
    """install() + the CTC head, decoder and search modules; CUDA streams / graphs are taken out of the picture (host logic only)."""
    import contextlib

    import espnet_b200.ctc as ctc
    import espnet_b200.decoder as dec
    import espnet_b200.lm as lmmod
    import espnet_b200.search as search

    install(monkeypatch)
    for mod in (ctc, dec, search, lmmod):
        monkeypatch.setattr(mod, "call", call, raising=True)
        monkeypatch.setattr(mod, "ptr", ptr, raising=True)
    class NoStream:   # stands in for torch.cuda.Stream: ordering is trivially sequential on the host
        def wait_stream(self, other):
            pass

        def wait_event(self, ev):
            pass

    monkeypatch.setattr(search.BatchBeamSearch, "use_cuda_graphs", False, raising=True)
    monkeypatch.setattr(search.BatchBeamSearch, "_side_stream", lambda self, dev, g=0: None, raising=True)
    monkeypatch.setattr(search.BatchBeamSearch, "_group_stream", lambda self, dev, g: NoStream(), raising=True)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: NoStream(), raising=True)
    monkeypatch.setattr(torch.cuda, "stream", lambda s: contextlib.nullcontext(), raising=True)


# ------------------------------------------------------------------------------------------------ frontend / normalisation entry points
def _stft_logmel(wave, lens, B, L, hop, window, tw, twt, start, count, offset, weight, nnz, n_mels, out, Tf, partial):
    """frontend.cu: torch.stft semantics per utterance (own reflect padding), power, SPARSE mel filterbank exactly as the tables describe it,
    clamp 1e-10, log; frames >= 1 + len/hop are zero (window: 512 taps, already zero-padded around the centre for win_length < 512).  The per-block column sums go to block 0 (only their total is contractual)."""
    o = out.view(B, Tf, n_mels)
    o.zero_()
    if partial is not None:
        partial.zero_()
    for b in range(B):
        n = int(lens[b])
        spec = torch.stft(wave.view(B, L)[b, :n], 512, hop_length=hop, win_length=512, window=window, center=True, pad_mode="reflect",
                          normalized=False, onesided=True, return_complex=True)
        power = (spec.real ** 2 + spec.imag ** 2).t()          # [Tf_b][257]
        tf_b = 1 + n // hop
        assert power.shape[0] == tf_b
        for j in range(n_mels):
            s, c, w0 = int(start[j]), int(count[j]), int(offset[j])
            mel = (power[:, s:s + c] * weight[w0:w0 + c]).sum(-1) if c > 0 else torch.zeros(tf_b)
            o[b, :tf_b, j] = torch.log(torch.clamp(mel, min=1e-10))
        if partial is not None:
            partial.view(B, -1, n_mels)[b, 0] = o[b, :tf_b].sum(0)


def _utt_mvn_from_partial(feats, wave_lens, B, Tf_max, n_mels, hop, partial):
    f = feats.view(B, Tf_max, n_mels)
    for b in range(B):
        tf_b = 1 + int(wave_lens[b]) // hop
        f[b, :tf_b] -= partial.view(B, -1, n_mels)[b].sum(0) / tf_b


def _utt_mvn(feats, feat_lens, B, Tf_max, n_mels, ws):
    f = feats.view(B, Tf_max, n_mels)
    for b in range(B):
        n = int(feat_lens[b])
        f[b, :n] -= f[b, :n].sum(0) / n


def _global_mvn(feats, feat_lens, B, Tmax, D, mean, std, norm_means, norm_vars):
    f = feats.view(B, Tmax, D)
    for b in range(B):
        n = int(feat_lens[b])
        if norm_means:
            f[b] -= mean
        f[b, n:] = 0.0
        if norm_vars:
            f[b] /= std


_TABLE.update({"espb_stft_logmel_f32": _stft_logmel, "espb_utt_mvn_from_partial_f32": _utt_mvn_from_partial, "espb_utt_mvn_f32": _utt_mvn,
               "espb_global_mvn_f32": _global_mvn})


def install_frontend(monkeypatch):
    import espnet_b200.frontend as fe

    monkeypatch.setattr(fe, "call", call, raising=True)
    monkeypatch.setattr(fe, "ptr", ptr, raising=True)
