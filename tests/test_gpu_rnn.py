"""-m gpu: the RNN model family on the CUDA path -- each new kernel against float64 torch (espb_vgg_conv1_relu_f32, espb_vgg_pool_f32,
espb_lstm_rec_step_f32, espb_rnn_proj_post_f32, espb_att_loc_step_f32), the encoders against the reference fixtures layer by layer, a ragged
batch against single-utterance calls, the whole Speech2Text against the reference's n-best lists, the reference's own BeamSearch driving
RNNDecoder.score, and bin_asr_inference from config and checkpoint files.

Tolerances as tests/test_gpu_subsampling.py: encoder outputs atol 1e-4, n-best sequences identical and scores within rtol 1e-4."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import rnn_fixture as fx
import test_rnn_host as rh
from oracle import rnn as orn

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _hl(a):
    return a[0] + a[1]


def test_vgg_conv1_and_pool_kernels_vs_float64():
    """conv1_1 with per-utterance zero padding into the bordered split layout; pool (odd extents, ragged lengths) into both layouts."""
    from espnet_b200 import ops

    g = torch.Generator().manual_seed(0)
    B, T, Fr, C = 3, 23, 13, 64
    lens = torch.tensor([23, 17, 1])
    fe = torch.randn(B, T, Fr, generator=g)
    w, b = torch.randn(C, 1, 3, 3, generator=g) / 3, 0.1 * torch.randn(C, generator=g)
    dev = [t.cuda() for t in (fe, w.view(C, 9), b, lens.to(torch.int32))]
    a = torch.full((B, 2, Fr + 2, T + 2, C), 7.0, device="cuda")
    ops.call("espb_vgg_conv1_relu_f32", ops.ptr(dev[0]), B, T, Fr, ops.ptr(dev[3]), ops.ptr(dev[1]), ops.ptr(dev[2]), C, ops.ptr(a), T)
    got = (a[:, 0] + a[:, 1]).cpu().double()            # [B][Fp][Tp][C]
    for i in range(B):
        L = int(lens[i])
        x = torch.zeros(1, 1, T, Fr, dtype=torch.float64)
        x[0, 0, :L] = fe[i, :L].double()
        ref = torch.relu(F.conv2d(x, w.double(), b.double(), padding=1))[0]   # [C][T][F]
        ref[:, L:] = 0
        exp = torch.zeros(Fr + 2, T + 2, C, dtype=torch.float64)
        exp[1:-1, 1:-1] = ref.permute(2, 1, 0)
        torch.testing.assert_close(got[i], exp, atol=1e-5, rtol=1e-5)
    # pool: x [B][F][T][C] plain with valid rows t < len
    x = torch.rand(B, Fr, T, C, generator=g)
    xd = x.cuda()
    Fo, To = (Fr + 1) // 2, (T + 1) // 2
    for pool, flat in ((1, 0), (0, 0), (1, 1)):
        Fe, Te = (Fo if pool else Fr), (To if pool else T)
        if flat:
            out = torch.full((2, B * Te, C * Fe), 7.0, device="cuda")
            plane = B * Te * C * Fe
        else:
            out = torch.full((B, 2, Fe + 2, Te + 2, C), 7.0, device="cuda")
            plane = (Fe + 2) * (Te + 2) * C
        ops.call("espb_vgg_pool_f32", ops.ptr(xd), B, Fr, T, C, ops.ptr(dev[3]), pool, flat, ops.ptr(out), plane)
        for i in range(B):
            L = int(lens[i])
            xi = x[i].permute(2, 1, 0)[None].double()[:, :, :L]    # [1][C][L][F]
            r = F.max_pool2d(xi, 2, stride=2, ceil_mode=True)[0] if pool else xi[0]
            OL = (L + 1) // 2 if pool else L
            full = torch.zeros(C, Te, Fe, dtype=torch.float64)
            full[:, :OL] = r
            if flat:
                got = _hl(out).cpu().double().view(B, Te, C * Fe)[i]
                exp = full.transpose(0, 1).reshape(Te, C * Fe)
            else:
                got = (out[i, 0] + out[i, 1]).cpu().double()
                exp = torch.zeros(Fe + 2, Te + 2, C, dtype=torch.float64)
                exp[1:-1, 1:-1] = full.permute(2, 1, 0)
            torch.testing.assert_close(got, exp, atol=1e-6, rtol=1e-6)


@pytest.mark.parametrize("ndir", [1, 2])
def test_lstm_rec_step_kernel_vs_float64(ndir):
    """A whole (B)LSTM layer driven step by step (the h W_hh^T product from float64 torch), ragged lengths, both directions."""
    from espnet_b200 import ops

    g = torch.Generator().manual_seed(ndir)
    B, T, H, Hp = 3, 9, 13, 16
    lens = torch.tensor([9, 4, 1])
    xg = torch.randn(B, T, ndir * 4 * H, generator=g)
    whh = torch.randn(ndir, 4 * H, H, generator=g) / 4
    xgd, l32 = xg.cuda(), lens.to(torch.int32).cuda()
    h = torch.zeros(2, ndir, B, Hp, device="cuda")
    c = torch.zeros(ndir, B, H, device="cuda")
    hg = torch.zeros(ndir, B, 4 * H, device="cuda")
    y = torch.full((2, B * T, ndir * H), 7.0, device="cuda")
    for s in range(T):
        if s:
            hh = _hl(h)[:, :, :H].double()
            hg.copy_(torch.einsum("dbk,dgk->dbg", hh, whh.double().cuda()).float())
        ops.call("espb_lstm_rec_step_f32", ops.ptr(xgd), ops.ptr(hg), ops.ptr(l32), s, B, T, H, Hp, ndir, ops.ptr(h), ndir * B * Hp, ops.ptr(c),
                 ops.ptr(y), B * T * ndir * H, ndir * H)
    got = _hl(y).cpu().double().view(B, T, ndir * H)
    for i in range(B):
        L = int(lens[i])
        exp = torch.zeros(T, ndir * H, dtype=torch.float64)
        for d in range(ndir):
            hh, cc = torch.zeros(H, dtype=torch.float64), torch.zeros(H, dtype=torch.float64)
            for t in (range(L - 1, -1, -1) if d else range(L)):
                gt = xg[i, t, d * 4 * H:(d + 1) * 4 * H].double() + whh[d].double() @ hh
                ig, fg, gg, og = gt.chunk(4)
                cc = torch.sigmoid(fg) * cc + torch.sigmoid(ig) * torch.tanh(gg)
                hh = torch.sigmoid(og) * torch.tanh(cc)
                exp[t, d * H:(d + 1) * H] = hh
        torch.testing.assert_close(got[i], exp, atol=2e-5, rtol=0)


def test_rnn_proj_post_kernel_vs_float64():
    from espnet_b200 import ops

    g = torch.Generator().manual_seed(3)
    B, T, D, ldo = 2, 5, 7, 8
    lens = torch.tensor([5, 2])
    x = torch.randn(B, T, D, generator=g)
    for act in (0, 1):
        xd = x.cuda()
        out = torch.full((2, B * T, ldo), 7.0, device="cuda")
        ops.call("espb_rnn_proj_post_f32", ops.ptr(xd), B, T, D, ops.ptr(lens.to(torch.int32).cuda()), act, 1, ops.ptr(out), B * T * ldo, ldo)
        exp = torch.tanh(x.double()) if act else x.double()
        exp[1, 2:] = 0
        torch.testing.assert_close(xd.cpu().double(), exp, atol=1e-6, rtol=0)
        torch.testing.assert_close(_hl(out)[:, :D].cpu().double().view(B, T, D), exp, atol=1e-6, rtol=0)
        assert torch.all(out[:, :, D:] == 7.0)


def test_att_loc_step_kernel_vs_float64():
    """AttLoc for 3 utterances (lengths 11, 1, 6) x 2 slots: the uniform first step, then a step whose parents are reordered through the
    ancestor table; weights, context and the ring against the float64 oracle."""
    from espnet_b200 import ops

    g = torch.Generator().manual_seed(4)
    U, W, Tm, A, E, H, chans, filts = 3, 2, 11, 24, 10, 12, 3, 4
    n = U * W
    lens = torch.tensor([11, 1, 6])
    enc = torch.randn(U, Tm, E, generator=g)
    w = {"att_list.0.mlp_enc.weight": torch.randn(A, E, generator=g) / 3, "att_list.0.mlp_enc.bias": 0.1 * torch.randn(A, generator=g),
         "att_list.0.mlp_dec.weight": torch.randn(A, H, generator=g) / 3, "att_list.0.mlp_att.weight": torch.randn(A, chans, generator=g),
         "att_list.0.loc_conv.weight": torch.randn(chans, 1, 1, 2 * filts + 1, generator=g),
         "att_list.0.gvec.weight": torch.randn(1, A, generator=g) / 3, "att_list.0.gvec.bias": 0.1 * torch.randn(1, generator=g)}
    o = orn.OracleRNNDecoder(orn.to(w), 1)
    enc_h = (enc @ w["att_list.0.mlp_enc.weight"].t() + w["att_list.0.mlp_enc.bias"]).cuda()
    enc_split = ops.split_from(enc.cuda().view(U * Tm, E))
    ring = torch.full((2, n, Tm), 7.0, device="cuda")
    out = torch.zeros(2, n, E + 4, device="cuda")
    out2 = torch.zeros(2, n, E, device="cuda")
    anc = torch.tensor([[0, 0], [0, 1], [3, 0], [3, 2], [5, 4], [4, 5]], dtype=torch.int32).cuda()   # pos 1 parents: anc[s][0]
    dev = dict(lens=lens.to(torch.int32).cuda(), cw=w["att_list.0.loc_conv.weight"].view(chans, -1).contiguous().cuda(),
               wt=w["att_list.0.mlp_att.weight"].t().contiguous().cuda(), gv=w["att_list.0.gvec.weight"].view(-1).cuda(),
               gb=w["att_list.0.gvec.bias"].cuda())
    prev = [None] * n
    for pos in (0, 1):
        z = torch.randn(n, H, generator=g)
        dec_z = (z @ w["att_list.0.mlp_dec.weight"].t()).cuda()
        ops.call("espb_att_loc_step_f32", ops.ptr(enc_h), ops.ptr(enc_split), U * Tm * E, ops.ptr(dev["lens"]), W, Tm, A, E, ops.ptr(dec_z),
                 ops.ptr(dev["cw"]), chans, filts, ops.ptr(dev["wt"]), ops.ptr(dev["gv"]), ops.ptr(dev["gb"]), ops.ptr(anc), 2, pos, None,
                 ops.ptr(ring), n, ops.ptr(out[0, 0, 4:]), n * (E + 4), E + 4, ops.ptr(out2), n * E, E)
        cur = []
        for s in range(n):
            u, L = s // W, int(lens[s // W])
            p = None if pos == 0 else prev[int(anc[s, 0])]
            cexp, aexp = o.att(enc[u, :L].double(), z[s].double(), p)
            cur.append(aexp)
            torch.testing.assert_close(ring[pos & 1, s, :L].cpu().double(), aexp, atol=2e-6, rtol=0)
            assert torch.all(ring[pos & 1, s, L:] == 0)
            torch.testing.assert_close(_hl(out)[s, 4:].cpu().double(), cexp, atol=2e-5, rtol=0)
            torch.testing.assert_close(_hl(out2)[s].cpu().double(), cexp, atol=2e-5, rtol=0)
        prev = cur


def test_drop_cand_kernel():
    from espnet_b200 import ops

    valid = torch.ones(5, 7, dtype=torch.int32, device="cuda")
    ops.call("espb_drop_cand_i32", ops.ptr(valid), 5, 7, 6)
    exp = torch.ones(5, 7, dtype=torch.int32)
    exp[:, 6] = 0
    assert torch.equal(valid.cpu(), exp)


@pytest.mark.parametrize("context_residual", [False, True])
def test_decoder_steps_vs_float64_oracle(context_residual):
    """RNNDecoder.init_memory / step for 3 utterances (lengths 9, 1, 6) x 2 slots over 5 positions, each slot's parent drawn among its
    utterance's slots through the ancestor table, against OracleRNNDecoder.score in float64: log-probabilities, every layer's h and c, and
    the attention weights.  Widths 10 / 14 exercise the padded operand columns; with context_residual the output layer reads [z_L; c]."""
    from espnet_b200 import RNNDecoder, ops

    torch.manual_seed(5)
    U, W, Tm, E, H, V, L, P = 3, 2, 9, 14, 10, 23, 2, 5
    n = U * W
    dec = RNNDecoder(V, E, num_layers=L, hidden_size=H, context_residual=context_residual,
                     att_conf=dict(adim=16, aconv_chans=3, aconv_filts=4)).cuda().eval()
    o = orn.OracleRNNDecoder(orn.to({k: v.cpu() for k, v in dec.state_dict().items()}), L, context_residual)
    lens = torch.tensor([9, 1, 6])
    g = torch.Generator().manual_seed(6)
    enc = torch.randn(U, Tm, E, generator=g)
    st = dec.init_memory(ops.split_from(enc.cuda().view(U * Tm, E)), U, Tm, lens.to(torch.int32).cuda(), n, P)
    anc = torch.zeros(n, P, dtype=torch.int32)
    prev = [None] * n
    for pos in range(P):
        tok = torch.randint(0, V, (n,), generator=g)
        if pos:
            anc[:, pos - 1] = torch.tensor([(s // W) * W + int(torch.randint(0, W, (1,), generator=g)) for s in range(n)], dtype=torch.int32)
        logp = dec.step(st, pos, tok.to(torch.int32).cuda(), anc.cuda()).cpu().double()
        cur = []
        for s in range(n):
            u, Lu = s // W, int(lens[s // W])
            parent = prev[int(anc[s, pos - 1])] if pos else None
            lp, ns = o.score(int(tok[s]), parent, enc[u, :Lu].double())
            cur.append(ns)
            torch.testing.assert_close(logp[s], lp, atol=5e-5, rtol=0)
            for k in range(L):
                torch.testing.assert_close(st["h"][pos & 1, k, s, :H].cpu().double(), ns[0][k], atol=2e-5, rtol=0)
                torch.testing.assert_close(st["c"][pos & 1, k, s, :H].cpu().double(), ns[1][k], atol=2e-5, rtol=0)
            torch.testing.assert_close(st["a"][pos & 1, s, :Lu].cpu().double(), ns[2], atol=2e-5, rtol=0)
            assert torch.all(st["a"][pos & 1, s, Lu:] == 0)
        prev = cur


@pytest.mark.parametrize("case", fx.ENC_CASES)
def test_encoder_layers_vs_reference_fixture(case):
    z = fx.load()
    enc, feats = fx.build_encoder(case, "cuda")
    enc.trace = []
    out, olens, _ = enc(feats.cuda(), torch.tensor([feats.shape[1]]))
    np.testing.assert_allclose(out[0].cpu().numpy(), z[f"{case}:out"][0], atol=TOL, rtol=0)
    assert int(olens[0]) == int(z[f"{case}:olens"][0])
    names = (["vgg"] if case.startswith("vgg") else []) + [k.split(":")[1] for k in sorted(z.files) if k.startswith(f"{case}:layer")]
    assert len(enc.trace) == len(names)
    for nm, t in zip(names, enc.trace):
        np.testing.assert_allclose(t[0].cpu().numpy(), z[f"{case}:{nm}"].reshape(t[0].shape), atol=TOL, rtol=0, err_msg=nm)


@pytest.mark.parametrize("case", fx.ENC_CASES)
def test_ragged_batch_equals_single(case):
    enc, feats = fx.build_encoder(case, "cuda")
    g = torch.Generator().manual_seed(9)
    T = feats.shape[1]
    lens = [T, T - 6, 3, T - 1]
    xs = torch.randn(len(lens), T, 80, generator=g).cuda()
    out, olens, _ = enc(xs, torch.tensor(lens))
    out = out.clone()
    for i, L in enumerate(lens):
        o1, ol1, _ = enc(xs[i:i + 1, :L], torch.tensor([L]))
        assert int(olens[i]) == int(ol1[0])
        torch.testing.assert_close(out[i, :int(ol1[0])], o1[0], atol=1e-5, rtol=0)
        assert torch.all(out[i, int(ol1[0]):] == 0)


def _s2t(tmp_path, dn):
    from espnet_b200 import Speech2Text

    model, kw, lm, hyps = fx.decode(dn)
    cfg, ckpt = fx.write_model_files(tmp_path, model)
    if lm:
        kw["lm_train_config"], kw["lm_file"] = fx.write_lm_files(tmp_path, lm)
    return Speech2Text(asr_train_config=cfg, asr_model_file=ckpt, device="cuda", **kw), hyps


def _check(hyps, ref):
    """n-best sequences identical, scores within rtol TOL."""
    assert len(hyps) == len(ref)
    for h, (yseq, score) in zip(hyps, ref):
        assert h.yseq.tolist() == yseq
        assert abs(float(h.score) - score) <= TOL * max(1.0, abs(score))


@pytest.mark.parametrize("dn", fx.DECODES)
def test_speech2text_vs_reference_fixture(tmp_path, dn):
    """The reference decodes this model with its non-batch BeamSearch (<eos> only from within the pre-beam); ctc_weight 0.3 / 0.5 / 1.0,
    context_residual, LSTM and Transformer LM fusion, alone and inside a ragged batch."""
    s2t, hyps = _s2t(tmp_path, dn)
    wave = torch.from_numpy(fx.load()["s2t:wave"])
    _check([r[3] for r in s2t(wave)], hyps)
    g = torch.Generator().manual_seed(1)
    out = s2t.batch_decode([0.1 * torch.randn(9000, generator=g), wave, 0.1 * torch.randn(15000, generator=g)])
    _check([r[3] for r in out[1]], hyps)


def test_reference_beam_search_drives_rnn_decoder_score(tmp_path):
    """The reference's own non-batch BeamSearch with our RNNDecoder (ScorerInterface.score / init_state / select_state) and the reference's
    CTCPrefixScorer over our encoder output reproduces the reference n-best of ctc_weight 0.5."""
    import os
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    from oracle import install_ref

    if not install_ref.available():
        pytest.skip("oracle/_ref is absent")
    install_ref.activate()
    from espnet2.legacy.nets.beam_search import BeamSearch
    from espnet2.legacy.nets.scorers.ctc import CTCPrefixScorer
    from espnet2.legacy.nets.scorers.length_bonus import LengthBonus

    s2t, hyps = _s2t(tmp_path, "ctc05")
    m = s2t.asr_model
    wave = torch.from_numpy(fx.load()["s2t:wave"]).cuda()
    enc, _ = m.encode(wave[None], torch.tensor([wave.shape[0]]))

    class _CTC(torch.nn.Module):   # the reference CTCPrefixScorer needs ctc.log_softmax (float64 math on the host from here)
        def log_softmax(self, x):
            w = fx.model_weights("base")
            return torch.log_softmax(x.double().cpu() @ w["ctc.ctc_lo.weight"].double().t() + w["ctc.ctc_lo.bias"].double(), dim=-1).float()

    from espnet_b200 import integration

    V = m.vocab_size
    cfg = fx.model_config("base")
    dec = integration.register()["decoder"]["b200_rnn"](vocab_size=V, encoder_output_size=cfg["encoder_conf"]["output_size"],
                                                        **cfg["decoder_conf"])
    dec.load_state_dict(m.decoder.state_dict(), strict=True)
    dec = dec.cuda().eval()
    bs = BeamSearch(scorers=dict(decoder=dec, ctc=CTCPrefixScorer(_CTC(), m.eos), length_bonus=LengthBonus(V)),
                    weights=dict(decoder=0.5, ctc=0.5, length_bonus=0.0), beam_size=4, vocab_size=V, sos=m.sos, eos=m.eos,
                    token_list=m.token_list, pre_beam_score_key="full")
    _check(bs(x=enc[0], maxlenratio=0.0, minlenratio=0.0), hyps)


def test_bin_asr_inference_from_config_and_checkpoint(tmp_path):
    """bin_asr_inference over a wav.scp with the recipe-style config and checkpoint: the 1- and 2-best token ids and scores are the
    reference's for the same 16-bit PCM."""
    import wave as wavmod

    from espnet_b200.bin_asr_inference import main

    z = fx.load()
    _, _, _, hyps = fx.decode("cli")
    cfg, ckpt = fx.write_model_files(tmp_path, "base")
    with wavmod.open(str(tmp_path / "a.wav"), "wb") as f:
        f.setnchannels(1); f.setsampwidth(2); f.setframerate(16000); f.writeframes(z["cli:pcm"].tobytes())
    (tmp_path / "wav.scp").write_text(f"a {tmp_path / 'a.wav'}\n")
    main(["--output_dir", str(tmp_path / "dec"), "--data_path_and_name_and_type", f"{tmp_path / 'wav.scp'},speech,sound",
          "--asr_train_config", cfg, "--asr_model_file", ckpt, "--beam_size", "4", "--ctc_weight", "0.5", "--nbest", "2"])
    for k in (1, 2):
        tok = (tmp_path / f"dec/{k}best_recog/token_int").read_text().split()
        assert tok[0] == "a" and tok[1:] == [str(t) for t in hyps[k - 1][0][1:-1]]
        score = float((tmp_path / f"dec/{k}best_recog/score").read_text().split()[1])
        assert abs(score - hyps[k - 1][1]) <= TOL * abs(hyps[k - 1][1])


# ================================================================================ kernels at recipe shapes, tile edges and refusals
# Against the float64 references of tests/test_rnn_host.py (vgg_conv1_ref, vgg_pool_ref, lstm_step_ref, att_loc_ref), fed the values the
# kernels read; each returns a per-element bound of the kernel's fp32 arithmetic, derived in its docstring, and err <= bound is asserted
# everywhere.  Outputs start as NaN: what a kernel must not write keeps its NaN bits.
NAN = float("nan")
NAN_BITS = int(np.float32(NAN).view(np.int32))


def _nan_bits(t):
    return bool((t.view(torch.int32) == NAN_BITS).all())


def _within(got, ref, tol, what):
    err = (got - ref).abs()
    assert bool((err <= tol).all()), f"{what}: max err {err.max().item():.3e}, worst err/tol {(err / tol.clamp_min(1e-300)).max().item():.2f}"


def _refused(name, args, match, *untouched):
    from espnet_b200 import ops

    with pytest.raises(RuntimeError, match=match):
        ops.call(name, *args)
    torch.cuda.synchronize()
    for t in untouched:
        assert _nan_bits(t) if t.is_floating_point() else bool((t == 1).all())


@pytest.mark.parametrize("B,Tf,T,Fr,C,lens", [(3, 3000, 3000, 83, 64, [3000, 1, 1237]), (2, 1001, 1000, 80, 96, [999, 1]),
                                             (2, 301, 301, 80, 256, [301, 150])])
def test_vgg_conv1_recipe_shapes(B, Tf, T, Fr, C, lens):
    """F 83 (fbank + pitch) and 80; T up to 3000 with lengths 1 and odd ones; T < Tf_max (the feature rows past T are not read); C 96 (two
    channel groups per 256-thread block, 64 threads idle) and C 256 (one time step per block)."""
    from espnet_b200 import ops

    g = torch.Generator().manual_seed(T + C)
    fe = torch.randn(B, Tf, Fr, generator=g)
    fe[:, T:] = NAN                                    # rows T..Tf_max-1 are never read
    w, b = torch.randn(C, 9, generator=g) / 3, 0.1 * torch.randn(C, generator=g)
    fe_d, w_d, b_d, l_d = fe.cuda(), w.cuda(), b.cuda(), torch.tensor(lens, dtype=torch.int32).cuda()
    out = torch.full((B, 2, Fr + 2, T + 2, C), NAN, device="cuda")
    ops.call("espb_vgg_conv1_relu_f32", ops.ptr(fe_d), B, Tf, Fr, ops.ptr(l_d), ops.ptr(w_d), ops.ptr(b_d), C, ops.ptr(out), T)
    for i, L in enumerate(lens):
        got = (out[i, 0].double() + out[i, 1].double())
        v, tol = rh.vgg_conv1_ref(fe_d[i, :T].double().nan_to_num(0.0), w_d.double(), b_d.double(), L)
        exp, et = torch.zeros_like(got), torch.zeros_like(got)
        exp[1:-1, 1:-1], et[1:-1, 1:-1] = v.permute(2, 1, 0), tol.permute(2, 1, 0)
        _within(got, exp, et, f"conv1 T{T} F{Fr} C{C} utt {i}")
    del out
    torch.cuda.empty_cache()


@pytest.mark.parametrize("B,Fr,T,C,lens", [(4, 41, 53, 128, [53, 1, 20, 27]), (3, 83, 2999, 64, [2999, 1, 1501])])
@pytest.mark.parametrize("pool,flat", [(1, 0), (1, 1), (0, 0)])
def test_vgg_pool_layouts_odd_extents(B, Fr, T, C, lens, pool, flat):
    """Pool (ceil mode over the valid rows) or copy into the bordered split layout, and pool into the flat [B * To][C * Fo] rows the BLSTM
    reads, at C 128 with odd F and T and at the F 83 / T 2999 input extents."""
    from espnet_b200 import ops

    g = torch.Generator().manual_seed(T * 7 + pool + 2 * flat)
    x = torch.rand(B, Fr, T, C, generator=g)
    xd, l_d = x.cuda(), torch.tensor(lens, dtype=torch.int32).cuda()
    Fe, Te = ((Fr + 1) // 2, (T + 1) // 2) if pool else (Fr, T)
    if flat:
        out = torch.full((2, B * Te, C * Fe), NAN, device="cuda")
        plane = B * Te * C * Fe
    else:
        out = torch.full((B, 2, Fe + 2, Te + 2, C), NAN, device="cuda")
        plane = (Fe + 2) * (Te + 2) * C
    ops.call("espb_vgg_pool_f32", ops.ptr(xd), B, Fr, T, C, ops.ptr(l_d), pool, flat, ops.ptr(out), plane)
    for i, L in enumerate(lens):
        xi = xd[i].permute(2, 1, 0).double()                # [C][T][F]
        if pool:
            v, tol = rh.vgg_pool_ref(xi, L)
        else:
            v = xi.clone()
            v[:, L:] = 0
            tol = 16 * rh.U32 * v.abs()
        if flat:
            got = (out[0].double() + out[1].double()).view(B, Te, C * Fe)[i]
            exp, et = v.transpose(0, 1).reshape(Te, C * Fe), tol.transpose(0, 1).reshape(Te, C * Fe)
        else:
            got = out[i, 0].double() + out[i, 1].double()
            exp, et = torch.zeros_like(got), torch.zeros_like(got)
            exp[1:-1, 1:-1], et[1:-1, 1:-1] = v.permute(2, 1, 0), tol.permute(2, 1, 0)
        _within(got, exp, et, f"pool {pool} flat {flat} T{T} utt {i}")


def test_vgg_refusals():
    from espnet_b200 import ops

    fe, w, b = torch.zeros(1, 8, 5, device="cuda"), torch.zeros(257 * 9, device="cuda"), torch.zeros(257, device="cuda")
    lens = torch.tensor([8], dtype=torch.int32).cuda()
    out = torch.full((2 * 7 * 10 * 257,), NAN, device="cuda")
    base = dict(T=8, F=5, C=64)
    for bad in (dict(C=0), dict(C=257), dict(T=9), dict(F=0)):
        a = dict(base, **bad)
        _refused("espb_vgg_conv1_relu_f32", (ops.ptr(fe), 1, 8, a["F"], ops.ptr(lens), ops.ptr(w), ops.ptr(b), a["C"], ops.ptr(out), a["T"]),
                 "vgg_conv1_relu: need", out)
    x = torch.zeros(5 * 8 * 64, device="cuda")
    for bad in (dict(F=0), dict(T=0), dict(C=0), dict(C=-3), dict(F=-1)):
        a = dict(base, **bad)
        _refused("espb_vgg_pool_f32", (ops.ptr(x), 1, a["F"], a["T"], a["C"], ops.ptr(lens), 1, 0, ops.ptr(out), 7 * 10 * 64),
                 "vgg_pool: need", out)


def _lstm_lens(B, T, g):
    return [T, T - 1, 1] + torch.randint(1, T + 1, (B - 3,), generator=g).tolist()


@pytest.mark.parametrize("H,Hp", [(320, 320), (1024, 1024), (333, 336)])
@pytest.mark.parametrize("ndir", [1, 2])
def test_lstm_rec_step_recipe_widths(H, Hp, ndir):
    """The (B)LSTM recurrence at the recipes' widths 320 and 1024 and at H 333 < Hp 336, B 16 with ragged lengths {T, T - 1, 1, ..}, gate
    pre-activations randn and +-60 (saturated sigmoid and tanh), y rows ldy > ndir * H.  Each step against lstm_step_ref fed the gates,
    the h W_hh^T product and the c the kernel holds; the pad columns of h (H..Hp) and of y (ndir * H..ldy) keep their NaN, and y rows
    t >= len are +0."""
    from espnet_b200 import ops

    g = torch.Generator().manual_seed(H * ndir)
    B, T = 16, 7
    lens = _lstm_lens(B, T, g)
    xg = torch.randn(B, T, ndir * 4 * H, generator=g) * 2
    sat = torch.rand(B, T, ndir * 4 * H, generator=g) < 0.3
    xg[sat] = 60 * torch.sign(xg[sat])
    whh = (torch.randn(ndir, 4 * H, H, generator=g) / H ** 0.5).double().cuda()
    ldy = ndir * H + 3
    xgd, l32 = xg.cuda(), torch.tensor(lens, dtype=torch.int32).cuda()
    h = torch.full((2, ndir, B, Hp), NAN, device="cuda")
    c = torch.full((ndir, B, H), NAN, device="cuda")
    hg = torch.zeros(ndir, B, 4 * H, device="cuda")
    y = torch.full((2, B * T, ldy), NAN, device="cuda")
    L = torch.tensor(lens).cuda()
    bi = torch.arange(B, device="cuda")
    for s in range(T):
        if s:
            hg.copy_(torch.einsum("dbk,dgk->dbg", _hl(h)[:, :, :H].double(), whh).float())
        c_prev = c.double()
        ops.call("espb_lstm_rec_step_f32", ops.ptr(xgd), ops.ptr(hg), ops.ptr(l32), s, B, T, H, Hp, ndir, ops.ptr(h), ndir * B * Hp,
                 ops.ptr(c), ops.ptr(y), B * T * ldy, ldy)
        yv = _hl(y.double()).view(B, T, ldy)
        for d in range(ndir):
            act = s < L
            t = torch.where(act, (L - 1 - s) if d else torch.full_like(L, s), 0)
            xs = xgd[bi, t, d * 4 * H:(d + 1) * 4 * H].double()
            hr, cr, th, tc = rh.lstm_step_ref(xs, None if s == 0 else hg[d].double(), c_prev[d])
            what = f"H{H} ndir{ndir} s{s} d{d}"
            _within(_hl(h.double())[d, act, :H], hr[act], th[act], what + " h")
            _within(c[d, act].double(), cr[act], tc[act], what + " c")
            _within(yv[bi, t, d * H:(d + 1) * H][act], hr[act], th[act], what + " y")
    assert _nan_bits(h[..., H:]) and _nan_bits(y[..., ndir * H:])
    for b, n in enumerate(lens):
        assert not bool(y[:, b * T + n:(b + 1) * T, :ndir * H].ne(0).any()), f"utterance {b}: y rows past len not 0"


def test_lstm_rec_step_refusals():
    from espnet_b200 import ops

    H = 8
    xg, hg = torch.zeros(2 * 4 * 2 * H, device="cuda"), torch.zeros(2 * 2 * 4 * H, device="cuda")
    lens = torch.tensor([2], dtype=torch.int32).cuda()
    h, c, y = (torch.full((n,), NAN, device="cuda") for n in (2 * 2 * H, 2 * H, 2 * 2 * 2 * H))
    base = dict(s=0, H=H, Hp=H, ndir=2, ldy=2 * H)
    for bad in (dict(Hp=H - 1), dict(ndir=3), dict(ndir=0), dict(ldy=2 * H - 1), dict(s=-1)):
        a = dict(base, **bad)
        _refused("espb_lstm_rec_step_f32", (ops.ptr(xg), ops.ptr(hg), ops.ptr(lens), a["s"], 1, 2, a["H"], a["Hp"], a["ndir"], ops.ptr(h),
                                            2 * H, ops.ptr(c), ops.ptr(y), 2 * 2 * H, a["ldy"]), "lstm_rec_step: need", h, c, y)


@pytest.mark.parametrize("act", [0, 1])
@pytest.mark.parametrize("write_plain,with_out", [(0, True), (1, False)])
def test_rnn_proj_post_modes(act, write_plain, with_out):
    """write_plain = 0 with out: x bit-unchanged; out = NULL with write_plain = 1: x in place only.  D = 13 (not a multiple of 4) with
    ldo = 16: the pad columns keep their NaN."""
    from espnet_b200 import ops

    g = torch.Generator().manual_seed(act + 2 * write_plain)
    B, T, D, ldo = 3, 5, 13, 16
    lens = [5, 2, 1]
    x = torch.randn(B, T, D, generator=g)
    xd, l_d = x.cuda(), torch.tensor(lens, dtype=torch.int32).cuda()
    out = torch.full((2, B * T, ldo), NAN, device="cuda")
    ops.call("espb_rnn_proj_post_f32", ops.ptr(xd), B, T, D, ops.ptr(l_d), act, write_plain, ops.ptr(out) if with_out else None,
             B * T * ldo, ldo)
    exp = torch.tanh(x.double()) if act else x.double()
    for b, n in enumerate(lens):
        exp[b, n:] = 0
    tol = (5 * rh.U32) * exp.abs()                            # tanhf 4u and its fp32 rounding; the identity is exact
    if write_plain:
        _within(xd.cpu().double(), exp, tol, "x in place")
    else:
        assert torch.equal(xd.cpu().view(torch.int32), x.view(torch.int32))
    if with_out:
        _within(_hl(out.double())[:, :D].cpu().view(B, T, D), exp, tol + 16 * rh.U32 * exp.abs(), "out")
        assert _nan_bits(out[:, :, D:])
    else:
        assert _nan_bits(out)


def test_rnn_proj_post_refusal():
    from espnet_b200 import ops

    x = torch.randn(2, 3, 8, device="cuda")
    x0 = x.clone()
    l_d = torch.tensor([3, 1], dtype=torch.int32).cuda()
    out = torch.full((2, 6, 8), NAN, device="cuda")
    _refused("espb_rnn_proj_post_f32", (ops.ptr(x), 2, 3, 8, ops.ptr(l_d), 1, 1, ops.ptr(out), 48, 7), "rnn_proj_post: need ldo >= D", out)
    assert torch.equal(x, x0)
    ops.call("espb_rnn_proj_post_f32", ops.ptr(x), 2, 3, 8, ops.ptr(l_d), 1, 1, None, 0, 7)   # ldo is not read without out
    torch.cuda.synchronize()
    assert bool(x[1, 1:].eq(0).all()) and not torch.equal(x, x0)


@pytest.mark.parametrize("j", [0, 4])
def test_drop_cand_several_blocks(j):
    from espnet_b200 import ops

    n, PC = 600, 5
    valid = torch.ones(n, PC, dtype=torch.int32, device="cuda")
    ops.call("espb_drop_cand_i32", ops.ptr(valid), n, PC, j)
    exp = torch.ones(n, PC, dtype=torch.int32)
    exp[:, j] = 0
    assert torch.equal(valid.cpu(), exp)
    for bad in (-1, PC):
        v = torch.ones(n, PC, dtype=torch.int32, device="cuda")
        _refused("espb_drop_cand_i32", (ops.ptr(v), n, PC, bad), r"drop_cand: need 0 <= j < PC", v)


def _att_setup(A, E, chans, filts, Tmax, lens, W, seed, peaked):
    """Weights, encoder states (split) and device operands of AttLoc for len(lens) utterances x W slots."""
    from espnet_b200 import ops

    w, _, _, g = rh._att_case(A, E, chans, filts, 1, seed, peaked)
    U = len(lens)
    enc = torch.randn(U, Tmax, E, generator=g)
    d = rh._att_dev_inputs(w, enc, torch.zeros(16))
    enc_split = ops.split_from(enc.cuda().view(U * Tmax, E))
    dev = {k: v.cuda() for k, v in d.items() if k != "dz"}
    dev["lens"] = torch.tensor(lens, dtype=torch.int32).cuda()
    return dict(w=w, g=g, enc_split=enc_split, enc_v=_hl(enc_split.double()).view(U, Tmax, E), dev=dev, U=U, W=W, n=U * W, Tmax=Tmax,
                A=A, E=E, chans=chans, filts=filts, lens=lens)


def _att_call(st, dz, anc, pos, step, ring, out, out_ld, out2):
    from espnet_b200 import ops

    dv, n, E = st["dev"], st["n"], st["E"]
    ops.call("espb_att_loc_step_f32", ops.ptr(dv["eh"]), ops.ptr(st["enc_split"]), st["U"] * st["Tmax"] * E, ops.ptr(dv["lens"]), st["W"],
             st["Tmax"], st["A"], E, ops.ptr(dz), ops.ptr(dv["cw"]), st["chans"], st["filts"], ops.ptr(dv["wt"]), ops.ptr(dv["gv"]),
             ops.ptr(dv["gb"]), ops.ptr(anc), anc.shape[1], pos, ops.ptr(step), ops.ptr(ring), n, ops.ptr(out), n * out_ld, out_ld,
             ops.ptr(out2), 0 if out2 is None else n * E, E)


def _att_check(st, dz, prev_ring, anc, pos, ring, out, what):
    """Every slot's new ring row and context against att_loc_ref, fed the parent's ring row the kernel read (1/len in fp32 at pos 0)."""
    dv, E = st["dev"], st["E"]
    ring_c = ring[pos & 1].double()
    ctx = _hl(out.double())
    for s in range(st["n"]):
        u = s // st["W"]
        L = st["lens"][u]
        prev = (torch.full((L,), float(np.float32(1.0) / np.float32(L)), dtype=torch.float64, device="cuda") if pos == 0
                else prev_ring[int(anc[s, pos - 1])][:L].double())
        a, c, ta, tc = rh.att_loc_ref(dv["eh"][u].double(), dz[s].double(), dv["cw"].double(), dv["wt"].double(), dv["gv"].double(),
                                      dv["gb"].double(), st["enc_v"][u], prev, L)
        _within(ring_c[s, :L], a, ta, f"{what} pos {pos} slot {s} weights")
        assert not bool(ring[pos & 1, s, L:].ne(0).any()), f"{what} pos {pos} slot {s}: weights past len not 0"
        _within(ctx[s, :E], c, tc, f"{what} pos {pos} slot {s} context")


@pytest.mark.parametrize("A,E,chans,filts,Tmax,peaked", [(1024, 1024, 10, 100, 750, False), (320, 320, 10, 100, 1500, False),
                                                          (320, 320, 10, 100, 750, True)])
def test_att_loc_step_recipe_shapes(A, E, chans, filts, Tmax, peaked):
    """AttLoc at the aishell RNN recipe's adim 1024 (10 channels, 100 taps: about 76 KiB of shared memory at Tmax 750, 30 s of audio) and
    at adim 320 with Tmax 1500 (about 70 KiB), both above the 48 KiB default, and a peaked case (gvec x 60, 2e spans hundreds).  Lengths
    Tmax, 1, 57 (< filts) and Tmax - 1, W = 4 slots each; positions 0, 1, 2 with parents reordered through the ancestor table; out_ld = E + 5
    (pad columns keep their NaN), out2 at position 0 only (bitwise out); position 1 again as pos 0 + *step_ptr = 1 is bitwise position 1."""
    lens = [Tmax, 1, 57, Tmax - 1]
    st = _att_setup(A, E, chans, filts, Tmax, lens, 4, seed=A + Tmax + peaked, peaked=peaked)
    n, W, g = st["n"], st["W"], st["g"]
    anc = torch.tensor([[(s // W) * W + (3 * s + 1) % W, (s // W) * W + (s + 2) % W] for s in range(n)], dtype=torch.int32).cuda()
    ring = torch.full((2, n, Tmax), NAN, device="cuda")
    out_ld = E + 5
    outs = [torch.full((2, n, out_ld), NAN, device="cuda") for _ in range(3)]
    out2 = torch.full((2, n, E), NAN, device="cuda")
    wdec = st["w"]["att_list.0.mlp_dec.weight"].double()
    prev_ring = None
    what = f"A{A} Tmax{Tmax}{' peaked' if peaked else ''}"
    for pos in range(3):
        dz = (torch.randn(n, wdec.shape[1], generator=g, dtype=torch.float64) @ wdec.t()).float().cuda()
        _att_call(st, dz, anc, pos, None, ring, outs[pos], out_ld, out2 if pos == 0 else None)
        torch.cuda.synchronize()
        if pos == 0:
            assert _nan_bits(ring[1]), "position 0 wrote the other ring half"
            assert torch.equal(out2, outs[0][:, :, :st["E"]])
        _att_check(st, dz, prev_ring, anc, pos, ring, outs[pos], what)
        assert _nan_bits(outs[pos][:, :, st["E"]:])
        if pos == 1:
            snap = ring[1].clone()
            again = torch.full_like(outs[1], NAN)
            step = torch.ones(1, dtype=torch.int32, device="cuda")
            _att_call(st, dz, anc, 0, step, ring, again, out_ld, None)
            torch.cuda.synchronize()
            assert torch.equal(again.view(torch.int32), outs[1].view(torch.int32)) and torch.equal(ring[1], snap), "step_ptr"
        prev_ring = ring[pos & 1].clone()


def test_att_loc_step_largest_shared_memory():
    """adim 1024, 10 channels, 100 taps: Tmax 3969 is the largest whose shared memory (4 (12 Tmax + 200 + 10240) bytes plus the 132-byte
    reduction buffer) fits the 227 KiB a block may use; it runs and is right.  Tmax 3970 is refused before any launch."""
    st = _att_setup(1024, 64, 10, 100, 3969, [3969, 1], 1, seed=3, peaked=False)
    wdec = st["w"]["att_list.0.mlp_dec.weight"].double()
    dz = (torch.randn(2, wdec.shape[1], generator=st["g"], dtype=torch.float64) @ wdec.t()).float().cuda()
    anc = torch.zeros(2, 1, dtype=torch.int32, device="cuda")
    ring = torch.full((2, 2, 3969), NAN, device="cuda")
    out = torch.full((2, 2, 64), NAN, device="cuda")
    _att_call(st, dz, anc, 0, None, ring, out, 64, None)
    torch.cuda.synchronize()
    _att_check(st, dz, None, anc, 0, ring, out, "Tmax 3969")


@pytest.mark.parametrize("bad,match", [(dict(Tmax=3970), "too large for shared memory"), (dict(Tmax=5000), "too large for shared memory"),
                                       (dict(W=5), "W > 0 dividing n"), (dict(out_ld=63), "out_ld"), (dict(filts=-1), "filts >= 0")])
def test_att_loc_step_refusals(bad, match):
    """Each bad argument is refused with a message before any launch: ring and out keep their NaN."""
    from espnet_b200 import ops

    a = dict(A=1024, E=64, chans=10, filts=100, Tmax=64, W=4, out_ld=64)
    a.update(bad)
    n = 12
    f = lambda k: torch.zeros(k, device="cuda")   # noqa: E731
    eh, enc, dz, cw, wt, gv, gb = f(3 * a["Tmax"] * a["A"]), f(2 * 3 * a["Tmax"] * 64), f(n * a["A"]), f(10 * 201), f(10 * a["A"]), f(a["A"]), f(1)
    lens = torch.full((3,), 5, dtype=torch.int32, device="cuda")
    anc = torch.zeros(n, 2, dtype=torch.int32, device="cuda")
    ring = torch.full((2, n, a["Tmax"]), NAN, device="cuda")
    out = torch.full((2, n, 64), NAN, device="cuda")
    _refused("espb_att_loc_step_f32", (ops.ptr(eh), ops.ptr(enc), 3 * a["Tmax"] * 64, ops.ptr(lens), a["W"], a["Tmax"], a["A"], a["E"],
                                       ops.ptr(dz), ops.ptr(cw), a["chans"], a["filts"], ops.ptr(wt), ops.ptr(gv), ops.ptr(gb), ops.ptr(anc), 2,
                                       0, None, ops.ptr(ring), n, ops.ptr(out), n * 64, a["out_ld"], None, 0, 64), match, ring, out)
