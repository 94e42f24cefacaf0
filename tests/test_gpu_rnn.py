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
