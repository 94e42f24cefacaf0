"""CPU: the RNN model family (VGGRNNEncoder / RNNEncoder / RNNDecoder) -- the float64 oracle against the reference fixtures
(tests/golden/rnn.npz), strict loading of reference state_dicts, the refused configurations, the registries, a model built from a
recipe-style config.yaml and checkpoint, and the C-ABI bindings of the new entry points."""
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import rnn_fixture as fx
from oracle import rnn as orn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("espb_vgg_conv1_relu_f32", "espb_vgg_pool_f32", "espb_lstm_rec_step_f32", "espb_rnn_proj_post_f32", "espb_att_loc_step_f32",
               "espb_drop_cand_i32")


@pytest.mark.parametrize("case", fx.ENC_CASES)
def test_oracle_encoder_vs_reference_fixture(case):
    z = fx.load()
    cls, conf, w, feats = fx.enc_case(case)
    out, trace = orn.rnn_encoder(feats[0].double(), orn.to(w), conf, cls)
    np.testing.assert_allclose(out.numpy(), z[f"{case}:out"][0], atol=1e-4, rtol=0)
    names = (["vgg"] if cls == "vgg_rnn" else []) + [f"layer{i}" for i in range(len(trace) - (cls == "vgg_rnn"))]
    for nm, t in zip(names, trace):
        np.testing.assert_allclose(t.numpy(), z[f"{case}:{nm}"].reshape(t.shape), atol=1e-4, rtol=0, err_msg=nm)
    assert out.shape[0] == int(z[f"{case}:olens"][0])


@pytest.mark.parametrize("case", fx.ENC_CASES)
def test_encoder_state_dict_loads_strictly(case):
    enc, _ = fx.build_encoder(case)
    _, _, w, _ = fx.enc_case(case)
    assert sorted(enc.state_dict()) == sorted(w)


@pytest.mark.parametrize("model", ["base", "ctxres"])
def test_model_from_recipe_config_and_checkpoint(tmp_path, model):
    """ASRTask.build_model_from_file path: config.yaml (encoder: vgg_rnn, decoder: rnn) + checkpoint -> every reference key loads."""
    from espnet_b200.asr_inference import build_model_from_file

    cfg, ckpt = fx.write_model_files(tmp_path, model)
    m, args = build_model_from_file(cfg, ckpt, device="cpu")
    w = fx.model_weights(model)
    sd = m.state_dict()
    assert sorted(k for k in sd if not k.startswith("frontend.")) == sorted(k for k in w if not k.startswith("frontend."))
    for k, v in w.items():
        if k in sd:
            assert torch.equal(sd[k], v), k
    assert type(m.encoder).__name__ == "VGGRNNEncoder" and type(m.decoder).__name__ == "RNNDecoder"
    assert m.decoder.context_residual == (model == "ctxres")


def test_registries():
    import espnet_b200
    from espnet_b200 import integration

    assert espnet_b200.encoder_choices["vgg_rnn"] is espnet_b200.VGGRNNEncoder
    assert espnet_b200.encoder_choices["rnn"] is espnet_b200.RNNEncoder
    assert espnet_b200.decoder_choices["rnn"] is espnet_b200.RNNDecoder
    assert integration.NAMES["encoder"]["b200_vgg_rnn"] == "VGGRNNEncoder"
    assert integration.NAMES["encoder"]["b200_rnn"] == "RNNEncoder"
    assert integration.NAMES["decoder"]["b200_rnn"] == "RNNDecoder"


def test_refused_configurations():
    import espnet_b200

    for cls in (espnet_b200.VGGRNNEncoder, espnet_b200.RNNEncoder):
        with pytest.raises(NotImplementedError):
            cls(80, rnn_type="gru")
        with pytest.raises(ValueError):
            cls(80, rnn_type="rnn_tanh")
    with pytest.raises(NotImplementedError):
        espnet_b200.VGGRNNEncoder(80, in_channel=3)
    dec = dict(vocab_size=10, encoder_output_size=8, hidden_size=8, att_conf=dict(adim=8, aconv_chans=2, aconv_filts=3))
    espnet_b200.RNNDecoder(**dec)
    bad = [dict(rnn_type="gru"), dict(replace_sos=True), dict(num_encs=2), dict(sampling_probability=0.1),
           dict(att_conf=dict(atype="dot")), dict(att_conf=dict(atype="location2d")), dict(att_conf=dict(han_mode=True)),
           dict(att_conf=dict(han_dim=16)), dict(att_conf=dict(num_att=2))]
    for kw in bad:
        with pytest.raises(NotImplementedError):
            espnet_b200.RNNDecoder(**dict(dec, **kw))
    with pytest.raises(ValueError):
        espnet_b200.RNNDecoder(**dict(dec, rnn_type="rnn"))
    with pytest.raises(TypeError):
        espnet_b200.RNNDecoder(**dict(dec, att_conf=dict(no_such_option=1)))


def test_decoder_parameter_names_match_reference():
    """The reference RNNDecoder's state_dict names (embed, decoder.{k}.*, output, att_list.0.*) as the fixture records them."""
    import espnet_b200

    cfg = fx.model_config("ctxres")
    dec = espnet_b200.RNNDecoder(vocab_size=len(cfg["token_list"]), encoder_output_size=cfg["encoder_conf"]["output_size"], **cfg["decoder_conf"])
    w = {k[len("decoder."):]: v for k, v in fx.model_weights("ctxres").items() if k.startswith("decoder.")}
    dec.load_state_dict(w, strict=True)


def test_oracle_decoder_step_properties():
    """The oracle decoder step: log-probabilities normalise, attention weights are a distribution, the first step uses uniform weights."""
    cfg = fx.model_config("base")
    w = orn.to({k[len("decoder."):]: v for k, v in fx.model_weights("base").items() if k.startswith("decoder.")})
    d = orn.OracleRNNDecoder(w, cfg["decoder_conf"]["num_layers"])
    enc = torch.randn(7, cfg["encoder_conf"]["output_size"], dtype=torch.float64)
    logp, st = d.score(len(cfg["token_list"]) - 1, None, enc)
    assert abs(float(logp.exp().sum()) - 1) < 1e-12 and abs(float(st[2].sum()) - 1) < 1e-12
    logp2, st2 = d.score(3, st, enc)
    assert abs(float(logp2.exp().sum()) - 1) < 1e-12 and not torch.equal(st2[2], st[2])


def test_new_entry_points_are_declared_and_bound():
    from espnet_b200 import lib

    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "espnet_b200.h")).read(), flags=re.S)
    for sym in NEW_SYMBOLS:
        assert sym in lib._SIGS and re.search(r"\bint\s+" + sym + r"\s*\(", src), sym
    assert len(lib._SIGS["espb_drop_cand_i32"]) == 5 and len(lib._SIGS["espb_att_loc_step_f32"]) == 28 and len(lib._SIGS["espb_lstm_rec_step_f32"]) == 16


# ------------------------------------------------------------------------------------------------ host logic through the kernel emulation
@pytest.mark.parametrize("case", fx.ENC_CASES)
def test_encoder_host_logic_vs_reference_fixture(case, monkeypatch):
    """VGGRNNEncoder / RNNEncoder.forward with the C-ABI entry points emulated (tests/emu_rnn.py): GEMM descriptors of the implicit-GEMM
    convs, the per-step recurrence GEMMs and the strided projection GEMMs, buffer pitches and layouts, against the reference fixture."""
    import emu_rnn

    emu_rnn.install(monkeypatch)
    z = fx.load()
    enc, feats = fx.build_encoder(case)
    enc.trace = []
    out, olens, _ = enc(feats, torch.tensor([feats.shape[1]]))
    np.testing.assert_allclose(out[0].numpy(), z[f"{case}:out"][0], atol=1e-4, rtol=0)
    assert int(olens[0]) == int(z[f"{case}:olens"][0])
    names = (["vgg"] if case.startswith("vgg") else []) + [k.split(":")[1] for k in sorted(z.files) if k.startswith(f"{case}:layer")]
    assert len(enc.trace) == len(names)
    for nm, t in zip(names, enc.trace):
        np.testing.assert_allclose(t[0].numpy(), z[f"{case}:{nm}"].reshape(t[0].shape), atol=1e-4, rtol=0, err_msg=nm)


@pytest.mark.parametrize("case", ["vgg_blstmp", "rnn_sub"])
def test_encoder_host_logic_ragged_batch_equals_single(case, monkeypatch):
    import emu_rnn

    emu_rnn.install(monkeypatch)
    enc, feats = fx.build_encoder(case)
    g = torch.Generator().manual_seed(9)
    T = feats.shape[1]
    lens = [T, T - 6, 3]
    xs = torch.randn(len(lens), T, 80, generator=g)
    out, olens, _ = enc(xs, torch.tensor(lens))
    out = out.clone()
    for i, L in enumerate(lens):
        o1, ol1, _ = enc(xs[i:i + 1, :L], torch.tensor([L]))
        assert int(olens[i]) == int(ol1[0])
        torch.testing.assert_close(out[i, :int(ol1[0])], o1[0], atol=1e-5, rtol=0)
        assert torch.all(out[i, int(ol1[0]):] == 0)


@pytest.mark.parametrize("context_residual", [False, True])
def test_decoder_host_logic_vs_oracle(context_residual, monkeypatch):
    """RNNDecoder.init_memory / step with the entry points emulated: 2 utterances (lengths 7, 3) x 2 slots over 4 positions with reordered
    ancestors, log-probabilities, h / c rings and attention weights against OracleRNNDecoder (float64); widths 10 / 14 exercise the padded
    operand columns."""
    import emu_rnn

    from espnet_b200 import RNNDecoder, ops

    emu_rnn.install(monkeypatch)
    torch.manual_seed(5)
    U, W, Tm, E, H, V, L, P = 2, 2, 7, 14, 10, 23, 2, 4
    n = U * W
    dec = RNNDecoder(V, E, num_layers=L, hidden_size=H, context_residual=context_residual,
                     att_conf=dict(adim=16, aconv_chans=3, aconv_filts=4)).eval()
    o = orn.OracleRNNDecoder(orn.to(dec.state_dict()), L, context_residual)
    lens = torch.tensor([7, 3])
    g = torch.Generator().manual_seed(6)
    enc = torch.randn(U, Tm, E, generator=g)
    st = dec.init_memory(ops.split_from(enc.view(U * Tm, E)), U, Tm, lens.to(torch.int32), n, P)
    anc = torch.zeros(n, P, dtype=torch.int32)
    prev = [None] * n
    for pos in range(P):
        tok = torch.randint(0, V, (n,), generator=g)
        if pos:
            anc[:, pos - 1] = torch.tensor([(s // W) * W + (s + pos) % W for s in range(n)], dtype=torch.int32)
        logp = dec.step(st, pos, tok.to(torch.int32), anc).double()
        cur = []
        for s in range(n):
            u, Lu = s // W, int(lens[s // W])
            lp, ns = o.score(int(tok[s]), prev[int(anc[s, pos - 1])] if pos else None, enc[u, :Lu].double())
            cur.append(ns)
            torch.testing.assert_close(logp[s], lp, atol=5e-5, rtol=0)
            for k in range(L):
                torch.testing.assert_close(st["h"][pos & 1, k, s, :H].double(), ns[0][k], atol=2e-5, rtol=0)
                torch.testing.assert_close(st["c"][pos & 1, k, s, :H].double(), ns[1][k], atol=2e-5, rtol=0)
            torch.testing.assert_close(st["a"][pos & 1, s, :Lu].double(), ns[2], atol=2e-5, rtol=0)
        prev = cur


# ------------------------------------------------------------------------------------------------ float64 references of the kernels
# Each takes the values the kernel reads (fp32 inputs as float64, hi + lo of split operands) and returns the result with a per-element error
# bound of the kernel's fp32 arithmetic, u = 2^-24.  CUDA's expf and tanhf are within 2 ulp (<= 4u relative), logf within 1 ulp, and a value
# stored split (hi + lo, each with 10 explicit mantissa bits) is within 2^-20 = 16u of the fp32 result.  tests/test_gpu_rnn.py compares the
# kernels with these; test_tolerances_catch_plausible_bugs below shows the bounds are tight enough to see the bugs named there.  Saturated
# gates and peaked weights reach values below fp32's smallest normal 2^-126, which keep no relative precision: the bounds add 2^-126
# absolute where that happens.
U32 = 2.0 ** -24
TINY = 2.0 ** -126


def _over(diff, tol):
    """max diff / tol (diff > 0 where tol == 0 counts as infinitely over)."""
    return (diff / tol.clamp_min(1e-300)).max().item()


def vgg_conv1_ref(x, w, b, L):
    """conv1_1 + ReLU (espb_vgg_conv1_relu_f32) of one utterance x [T][F] with rows t >= L zero, w [C][9], b [C] -> (v, tol) [C][T][F].
    Per element 9 fmaf and the bias add, each within u of the partial sums' magnitude sum_k |w_k x_k| + |b|, then the split store."""
    C = w.shape[0]
    x = x.clone()
    x[L:] = 0
    v = torch.relu(F.conv2d(x[None, None], w.view(C, 1, 3, 3), b, padding=1))[0]
    mag = F.conv2d(x.abs()[None, None], w.abs().view(C, 1, 3, 3), b.abs(), padding=1)[0]
    v[:, L:] = 0
    return v, 10 * U32 * mag + 16 * U32 * v.abs()


def vgg_pool_ref(x, L, ceil=True):
    """2x2 max-pool of x [C][T][F] over its rows t < L (espb_vgg_pool_f32, ceil mode) -> (v [C][To][Fo], tol): the max is exact, so the
    tolerance is the split store.  ceil=False restates a pool in floor mode (odd T or F lose their last row or column)."""
    C, T, Fr = x.shape
    To, Fo = (T + 1) // 2, (Fr + 1) // 2
    r = F.max_pool2d(x[None, :, :L], 2, stride=2, ceil_mode=ceil)[0]
    v = x.new_zeros(C, To, Fo)
    v[:, :r.shape[1], :r.shape[2]] = r
    return v, 16 * U32 * v.abs()


def _sig(x):
    s = torch.sigmoid(x)
    return s, s * (1 - s)


def lstm_step_ref(xg, hg, cp, order=(0, 1, 2, 3)):
    """One LSTM cell step (espb_lstm_rec_step_f32): gates xg [..][4H] (+ hg, None at the first step, where c starts at 0), c_prev cp
    [..][H] as the kernel holds it -> (h, c, tol_h, tol_c).  order restates a gate layout bug ((1, 0, 2, 3): i and f swapped).
    Error per element: the gate sum xg + hg rounds once (u |x|, moved by sigma' = s (1 - s) or tanh' = 1 - tanh^2); sigmoid
    1 / (1 + expf(-x)) is within 6u relative (expf, the add, the divide), tanhf within 4u; c' = s_f c + s_i tanh(g) rounds twice; h' =
    s_o tanhf(c') once more; h (and y) are stored split (16u), c plain."""
    x = xg if hg is None else xg + hg
    dx = torch.zeros_like(x) if hg is None else U32 * x.abs()
    gi, gf, gg, go = (x.chunk(4, dim=-1)[k] for k in order)
    di, df, dg, do = (dx.chunk(4, dim=-1)[k] for k in order)
    cp = torch.zeros_like(gi) if hg is None else cp
    (si, si_d), (sf, sf_d), (so, so_d) = _sig(gi), _sig(gf), _sig(go)
    tg = torch.tanh(gg)
    e_si, e_sf, e_so = 6 * U32 * si + si_d * di, 6 * U32 * sf + sf_d * df, 6 * U32 * so + so_d * do
    e_tg = 4 * U32 * tg.abs() + (1 - tg * tg) * dg
    c = sf * cp + si * tg
    e_c = e_sf * cp.abs() + e_si * tg.abs() + si * e_tg + 2 * U32 * ((sf * cp).abs() + (si * tg).abs())
    tc = torch.tanh(c)
    h = so * tc
    e_h = e_so * tc.abs() + so * (4 * U32 * tc.abs() + (1 - tc * tc) * e_c) + 17 * U32 * h.abs() + 4 * TINY
    return h, c, e_h, e_c + 4 * TINY


def att_loc_ref(eh, dz, cw, wt, gv, gb, enc, prev, L, tap=0, len_off=0):
    """AttLoc of one slot (espb_att_loc_step_f32) from the values the kernel reads: eh [>= L][A] = mlp_enc(enc) + bias, dz [A] = mlp_dec(z),
    cw [chans][2 filts + 1], wt [chans][A] (mlp_att.weight^T), gv [A], gb, enc [>= L][E] (hi + lo), prev [L] the previous weights (the
    uniform 1/L of the first step as the fp32 value the kernel forms) -> (a [L], ctx [E], tol_a, tol_ctx).  OracleRNNDecoder.att
    (oracle/rnn.py) computes the same from the model weights; test_att_loc_ref_is_the_oracle checks that.
    tap / len_off restate bugs: the location conv reads prev one tap late; the softmax runs over L + len_off frames.
    Error, per frame t: the conv (K = 2 filts + 1 fmaf) within K u sum_k |w prev|; loc = sum_c wt conv (chans fmaf) within chans u
    sum_c |wt conv| plus the conv errors through |wt|; the two adds into the tanh argument u (|loc| + |eh| + |dz|) each; tanhf 4u; the energy
    (ceil(A / 32) fmaf per lane, 5 shuffle adds, + gb) within (ceil(A / 32) + 6) u (sum_a |gv tanh| + |gb|), doubled by the scaling 2.
    A weight a_t = exp(x_t - m) / sum is off relatively by its own energy error and the weighted mean of all of them (through the sum),
    u |x_t - m| for the subtraction, 4u for expf (in its own term and, weighted, in the sum's), and (ceil(L / 256) + 12) u for the block sum (per-thread adds, two 5-step shuffle
    trees), 1 / sum and the product.  The context
    (hi + lo added, then L fmaf in sequence) is within sum_t tol_a |enc| + (L + 1) u sum_t a |enc|, plus 16u for its split store.  Weights
    whose exponential underflows (peaked energies) are within 2^-126."""
    K, A = cw.shape[1], wt.shape[1]
    filts = (K - 1) // 2
    Lw = L + len_off
    pv = prev.new_zeros(Lw)
    pv[:min(L, Lw)] = prev[:min(L, Lw)]
    pp = F.pad(pv, (filts - tap, filts + tap))[None, None]
    conv = F.conv1d(pp, cw[:, None])[0].t()                              # [Lw][chans]
    e_conv = K * U32 * F.conv1d(pp.abs(), cw.abs()[:, None])[0].t()
    loc = conv @ wt
    e_loc = wt.shape[0] * U32 * (conv.abs() @ wt.abs()) + e_conv @ wt.abs()
    arg = loc + eh[:Lw] + dz
    e_arg = e_loc + 2 * U32 * (loc.abs() + eh[:Lw].abs() + dz.abs())
    th = torch.tanh(arg)
    e_th = 4 * U32 * th.abs() + (1 - th * th) * e_arg
    x = 2 * (th @ gv + gb)
    e_x = 2 * (e_th @ gv.abs() + (-(-A // 32) + 6) * U32 * (th.abs() @ gv.abs() + abs(float(gb))))
    a = torch.softmax(x, 0)
    xm = (x - x.max()).abs()
    rho = e_x + (a * e_x).sum() + U32 * (xm + (a * xm).sum()) + (20 - (-Lw // 256)) * U32
    ta = a * rho + TINY
    en = enc[:Lw]
    ctx = a @ en
    tc = ta @ en.abs() + (Lw + 1) * U32 * (a @ en.abs()) + 16 * U32 * ctx.abs() + TINY
    return a, ctx, ta, tc


def _att_case(A, E, chans, filts, Tmax, seed, peaked=False):
    """Seeded weights and inputs of one AttLoc slot at the given shape, and its OracleRNNDecoder; gvec scaled by 60 when peaked (2e spans
    hundreds)."""
    g = torch.Generator().manual_seed(seed)
    H = 16
    w = {"att_list.0.mlp_enc.weight": torch.randn(A, E, generator=g) / E ** 0.5, "att_list.0.mlp_enc.bias": 0.1 * torch.randn(A, generator=g),
         "att_list.0.mlp_dec.weight": torch.randn(A, H, generator=g) / H ** 0.5, "att_list.0.mlp_att.weight": torch.randn(A, chans, generator=g),
         "att_list.0.loc_conv.weight": torch.randn(chans, 1, 1, 2 * filts + 1, generator=g) / 4,
         "att_list.0.gvec.weight": torch.randn(1, A, generator=g) / A ** 0.5 * (60 if peaked else 1),
         "att_list.0.gvec.bias": 0.1 * torch.randn(1, generator=g)}
    enc = torch.randn(Tmax, E, generator=g)
    z = torch.randn(H, generator=g)
    return w, enc, z, g


def _att_dev_inputs(w, enc, z):
    """The values the attention kernel reads, from the model weights: eh, dz rounded to fp32 as the GEMMs deliver them (float64 here)."""
    eh = (enc.double() @ w["att_list.0.mlp_enc.weight"].double().t() + w["att_list.0.mlp_enc.bias"].double()).float()
    dz = (w["att_list.0.mlp_dec.weight"].double() @ z.double()).float()
    chans = w["att_list.0.mlp_att.weight"].shape[1]
    return dict(eh=eh, dz=dz, cw=w["att_list.0.loc_conv.weight"].view(chans, -1).contiguous(), wt=w["att_list.0.mlp_att.weight"].t().contiguous(),
                gv=w["att_list.0.gvec.weight"].view(-1).contiguous(), gb=w["att_list.0.gvec.bias"].contiguous())


def test_att_loc_ref_is_the_oracle():
    """att_loc_ref over mlp_enc(enc) and mlp_dec(z) in float64 is OracleRNNDecoder.att, first step and a later one."""
    w, enc, z, g = _att_case(40, 24, 3, 5, 30, seed=1)
    o = orn.OracleRNNDecoder(orn.to(w), 1)
    x = {k: v.double() for k, v in dict(eh=enc.double() @ w["att_list.0.mlp_enc.weight"].double().t() + w["att_list.0.mlp_enc.bias"].double(),
                                        dz=w["att_list.0.mlp_dec.weight"].double() @ z.double()).items()}
    d = {k: v.double() for k, v in _att_dev_inputs(w, enc, z).items()}
    L = 23
    for prev in (None, torch.softmax(torch.randn(L, generator=g, dtype=torch.float64), 0)):
        c_o, a_o = o.att(enc[:L].double(), z.double(), prev)
        p = torch.full((L,), 1.0 / L, dtype=torch.float64) if prev is None else prev
        a, c, _, _ = att_loc_ref(x["eh"], x["dz"], d["cw"], d["wt"], d["gv"], d["gb"], enc.double(), p, L)
        torch.testing.assert_close(a, a_o, atol=1e-12, rtol=0)
        torch.testing.assert_close(c, c_o, atol=1e-12, rtol=0)


def test_tolerances_catch_plausible_bugs():
    """On the CPU, from the float64 references above: each plausible bug moves the reference by more than 10x the tolerance the GPU tests
    of tests/test_gpu_rnn.py use, at a shape they run.
    * LSTM i and f gates swapped (H 320, B 16, gates randn and +-60);
    * the location conv one tap late, and the softmax over len + 1 frames (AttLoc at adim 1024, 10 channels, 100 taps, Tmax 750, len 57,
      previous weights of a later step);
    * the pool in floor mode (C 128, odd F 41 and T 53)."""
    g = torch.Generator().manual_seed(0)
    H = 320
    xg = torch.randn(16, 4 * H, generator=g, dtype=torch.float64) * 2
    xg[:, ::3] = 60 * torch.sign(xg[:, ::3])
    hg = torch.randn(16, 4 * H, generator=g).double()
    cp = torch.randn(16, H, generator=g).double()
    h, c, th, tcl = lstm_step_ref(xg, hg, cp)
    h2, c2, _, _ = lstm_step_ref(xg, hg, cp, order=(1, 0, 2, 3))
    assert float(th.max()) < 1e-5 and _over((h2 - h).abs(), th) > 10 and _over((c2 - c).abs(), tcl) > 10

    A, E, chans, filts, Tmax, L = 1024, 1024, 10, 100, 750, 57
    w, enc, z, g = _att_case(A, E, chans, filts, Tmax, seed=2)
    d = {k: v.double() for k, v in _att_dev_inputs(w, enc, z).items()}
    prev = torch.softmax(3 * torch.randn(L, generator=g, dtype=torch.float64), 0).float().double()
    args = (d["eh"], d["dz"], d["cw"], d["wt"], d["gv"], d["gb"], enc.double(), prev, L)
    a, ctx, ta, tc = att_loc_ref(*args)
    for bug in (dict(tap=1), dict(len_off=1)):
        a2, ctx2, _, _ = att_loc_ref(*args, **bug)
        assert _over((a2[:L] - a).abs(), ta) > 10, bug
        assert _over((ctx2 - ctx).abs(), tc) > 10, bug

    x = torch.rand(128, 53, 41, generator=g, dtype=torch.float64)
    v, tol = vgg_pool_ref(x, 53)
    v2, _ = vgg_pool_ref(x, 53, ceil=False)
    assert _over((v2 - v).abs(), tol) > 10
