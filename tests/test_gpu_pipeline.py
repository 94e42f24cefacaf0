"""-m gpu parity tests: CUDA path (through the C-ABI library) vs the golden fixtures and the CPU oracle.

Tolerances (fp32 path, error-compensated 3xTF32 GEMMs): features atol 5e-4 on log-mel; encoder outputs / CTC logits
atol 1e-4 on O(1) activations with the default GEMM (chunked fp32 promotion) and the FFMA GEMM, 5e-4 with the
plain kernel that accumulates all of K in the tensor core; CTC-greedy token ids bit-exact; beam-search
token sequences identical and scores within rtol 2e-4 (the reference's own cached-vs-uncached decoder
tolerance is rtol 1e-4, test/espnet2/legacy/test_transformer_decode.py:9).
"""
import os

import numpy as np
import pytest
import torch

import oracle
from oracle import encoder as OE
from oracle import frontend as OF
from golden_util import DEC_NAMES, decode_params, decode_results, load
from gpu_util import build_cuda_model, random_weights, refbuild, speech2text

pytestmark = pytest.mark.gpu

GEMM_MODES = [m for m in os.environ.get("ESPB_TEST_GEMM_MODES", "simt,tc,tc2").split(",") if m]


@pytest.fixture(params=GEMM_MODES)
def gemm_mode(request):
    from espnet_b200 import ops

    old = ops.gemm_mode()
    ops.set_gemm_mode(request.param)
    yield request.param
    ops.set_gemm_mode(old)


def enc_tol(mode=None):
    """Encoder / logits tolerance by GEMM kernel (see the module docstring)."""
    from espnet_b200 import ops

    return 5e-4 if (mode or ops.gemm_mode()) == "tc" else 1e-4


def _maxerr(a, b):
    return (a.double().cpu() - torch.as_tensor(b).double()).abs().max().item()


def test_library_loaded_and_device():
    import ctypes

    from espnet_b200 import lib

    l = lib.load()
    ma, mi = ctypes.c_int(), ctypes.c_int()
    assert l.espb_device_sm(ctypes.byref(ma), ctypes.byref(mi)) == 0
    assert (ma.value, mi.value) == (9, 0), "sm_90a library needs an H100-class (compute capability 9.0) GPU"


@pytest.mark.parametrize("lens", [[12000], [16000, 16000, 16000], [20000, 9000, 13333, 4000]])
def test_frontend_and_mvn_vs_oracle(lens):
    import espnet_b200

    fe, mvn = espnet_b200.DefaultFrontend().cuda(), espnet_b200.UtteranceMVN()
    waves = [refbuild.waveform(10 + i, n) for i, n in enumerate(lens)]
    L = max(lens)
    batch = torch.zeros(len(lens), L)
    for i, w in enumerate(waves):
        batch[i, : lens[i]] = w
    feats, flens = fe(batch.cuda(), torch.tensor(lens))
    assert flens.tolist() == [1 + n // 128 for n in lens]
    raw = feats.clone()
    norm, _ = mvn(feats, flens)
    melmat = fe.logmel.melmat.cpu()
    for i, w in enumerate(waves):
        ref = OF.log_mel(OF.stft_power(w), melmat)
        tf = ref.shape[0]
        e = _maxerr(raw[i, :tf], ref)
        assert e < 5e-4, f"log-mel max abs err {e}"
        assert raw[i, tf:].abs().max().item() == 0 if tf < raw.shape[1] else True
        e = _maxerr(norm[i, :tf], OF.utterance_mvn(ref))
        assert e < 5e-4, f"mvn max abs err {e}"


@pytest.mark.parametrize("hop,win_length,window", [(160, None, "hann"), (160, 400, "hann"), (100, 320, "hamming"), (75, 512, None), (256, 512, "hann")])
def test_frontend_other_hop_and_window_vs_oracle(hop, win_length, window):
    """hop_length / win_length / window generality of the fused kernel (e.g. the hop-160 Conformer recipe,
    egs2/librispeech/asr1/conf/tuning/train_asr_conformer10_hop_length160.yaml:37-38): ragged batch against the oracle (= torch.stft)."""
    import espnet_b200

    fe, mvn = espnet_b200.DefaultFrontend(hop_length=hop, win_length=win_length, window=window).cuda(), espnet_b200.UtteranceMVN()
    lens = [21000, 9001, 16000]
    waves = [refbuild.waveform(30 + i, n) for i, n in enumerate(lens)]
    batch = torch.zeros(len(lens), max(lens))
    for i, w in enumerate(waves):
        batch[i, : lens[i]] = w
    feats, flens = fe(batch.cuda(), torch.tensor(lens))
    assert flens.tolist() == [1 + n // hop for n in lens]
    raw = feats.clone()
    norm, _ = mvn(feats, flens)
    melmat = fe.logmel.melmat.cpu()
    for i, w in enumerate(waves):
        ref = OF.log_mel(OF.stft_power(w, hop=hop, win_length=win_length, window=window), melmat)
        tf = ref.shape[0]
        e = _maxerr(raw[i, :tf], ref)
        assert e < 5e-4, f"log-mel max abs err {e}"
        assert (raw[i, tf:].abs().max().item() == 0) if tf < raw.shape[1] else True
        assert _maxerr(norm[i, :tf], OF.utterance_mvn(ref)) < 5e-4


def test_standalone_mvn_kernel():
    import espnet_b200

    x = torch.randn(3, 50, 80)
    lens = torch.tensor([50, 31, 7])
    y, _ = espnet_b200.UtteranceMVN()(x.clone().cuda(), lens)
    for b in range(3):
        ref = OF.utterance_mvn(x[b, : lens[b]])
        assert _maxerr(y[b, : lens[b]], ref) < 1e-5


@pytest.mark.parametrize("case", ["tiny", "small"])
def test_encoder_vs_golden(case, gemm_mode):
    z, cfg, w = load(case)
    model, _ = build_cuda_model(cfg, w)
    feats = torch.from_numpy(z["feats_norm"]).unsqueeze(0).cuda()
    model.encoder.trace = []
    enc, olens, _ = model.encoder(feats, torch.tensor([feats.shape[1]]))
    torch.cuda.synchronize()
    errs = [_maxerr(t[0], z[f"layer{i}"]) for i, t in enumerate(model.encoder.trace)]
    print(f"[{case}/{gemm_mode}] per-stage max abs err:", ["%.2e" % e for e in errs])
    assert olens.tolist() == [z["enc"].shape[0]]
    tol = enc_tol(gemm_mode)
    assert max(errs) < tol, errs
    e = _maxerr(enc[0], z["enc"])
    print(f"[{case}/{gemm_mode}] encoder out max abs err {e:.3e}")
    assert e < tol
    lg = model.ctc.logits(enc, model.enc_split(enc))
    e = _maxerr(lg[0], z["ctc_logits"])
    print(f"[{case}/{gemm_mode}] ctc logits max abs err {e:.3e}")
    assert e < tol
    lp = model.ctc.log_softmax(enc)
    assert _maxerr(lp[0], z["ctc_logp"]) < tol
    assert model.ctc.argmax(enc)[0].cpu().tolist() == z["ctc_argmax"].tolist()


@pytest.mark.parametrize("case", ["tiny", "small"])
def test_ctc_greedy_bit_exact_vs_golden(case, gemm_mode):
    z, cfg, w = load(case)
    s2t = speech2text(cfg, w, beam_size=2, ctc_weight=0.3)
    ids = s2t.ctc_greedy([z["wave"]])
    assert ids[0] == z["ctc_greedy"].tolist()


def test_encoder_batch_and_ragged_vs_oracle(gemm_mode):
    """Equal-length batch and ragged batch both reproduce per-utterance (batch-1) results of the oracle."""
    cfg = dict(d_model=128, heads=4, ff=256, enc_layers=2, dec_layers=1, vocab=300, kernel=31)
    w = random_weights(cfg, seed=5)
    s2t = speech2text(cfg, w, beam_size=2, ctc_weight=0.3)
    o = oracle.OracleSpeech2Text(cfg, w, beam_size=2, ctc_weight=0.3)
    for lens in ([24000] * 3, [40000, 17000, 29000, 8000], [96000, 51000, 70001]):   # the last: rows longer than 128 keys (smem softmax), ragged
        waves = [refbuild.waveform(50 + i, n) for i, n in enumerate(lens)]
        speech, sl = s2t._to_batch(waves)
        enc, elens = s2t.asr_model.encode(speech, sl)
        greedy = s2t.ctc_greedy(waves)
        for i, wv in enumerate(waves):
            ref = o.encode(wv)
            assert int(elens[i]) == ref.shape[0]
            e = _maxerr(enc[i, : ref.shape[0]], ref)
            print(f"[{gemm_mode}] lens={lens} utt{i} enc max abs err {e:.3e}")
            assert e < enc_tol(gemm_mode)
            am, ids = OE.ctc_greedy(ref, o.w)
            logits = OE.ctc_logits(ref, o.w)
            top2 = logits.topk(2, dim=-1)[0]
            margin = (top2[:, 0] - top2[:, 1]).min().item()
            if margin > 20 * e:  # margin-aware: only demand identity when the oracle's own top-2 gap exceeds the measured error
                assert greedy[i] == ids.tolist()


@pytest.mark.parametrize("case", ["tiny", "small"])
@pytest.mark.parametrize("dn", DEC_NAMES)
def test_beam_search_vs_golden(case, dn, gemm_mode):
    z, cfg, w = load(case)
    s2t = speech2text(cfg, w, nbest=10, **decode_params(z, dn))
    res = s2t(z["wave"])
    gold = decode_results(z, dn)
    got = [(r[3].yseq.tolist(), r[3].score) for r in res]
    print(f"[{case}/{dn}/{gemm_mode}] got", got[:3], "gold", [(g[0], g[1]) for g in gold[:3]])
    assert len(res) == len(gold)
    for (_, _, _, h), (yseq, score, scores) in zip(res, gold):
        assert h.yseq.tolist() == yseq
        assert abs(h.score - score) <= 2e-4 * max(1.0, abs(score))
        for k, ref in zip(("decoder", "ctc", "length_bonus"), scores):
            if not np.isnan(ref):
                assert abs(h.scores[k] - ref) <= 2e-4 * max(1.0, abs(ref)), (k, h.scores[k], ref)


def test_batched_beam_search_vs_oracle(gemm_mode):
    """Several utterances decoded in one device-resident search == oracle run per utterance (ragged lengths)."""
    cfg = dict(d_model=64, heads=4, ff=128, enc_layers=2, dec_layers=2, vocab=60, kernel=15)
    w = random_weights(cfg, seed=7)
    kw = dict(beam_size=5, ctc_weight=0.3, maxlenratio=-10.0, nbest=5)
    s2t = speech2text(cfg, w, **kw)
    o = oracle.OracleSpeech2Text(cfg, w, **kw)
    lens = [16000, 9000, 12345]
    waves = [refbuild.waveform(70 + i, n) for i, n in enumerate(lens)]
    res = s2t.batch_decode(waves)
    for i, wv in enumerate(waves):
        ref = o(wv)
        assert len(res[i]) == len(ref)
        for a, b in zip(res[i], ref):
            assert a[3].yseq.tolist() == b[3].yseq.tolist()
            assert abs(a[3].score - b[3].score) <= 2e-4 * max(1.0, abs(b[3].score))


def test_too_short_utterance_raises():
    import espnet_b200

    z, cfg, w = load("tiny")
    s2t = speech2text(cfg, w, beam_size=2, ctc_weight=0.3)
    with pytest.raises(espnet_b200.TooShortUttError):
        s2t(torch.zeros(700))


def test_config0_ctc_greedy_8x5s_vs_oracle():
    """BASELINE.json configs[0]: Conformer 4L/256d/4h (ff 2048, kernel 31), V=5000, CTC-greedy, 8 x 5 s -- token ids bit-exact against the
    CPU oracle (identity is demanded for every utterance whose smallest top-2 logit gap exceeds 20x the measured logit error)."""
    torch.set_num_threads(min(16, torch.get_num_threads()))
    cfg = dict(d_model=256, heads=4, ff=2048, enc_layers=4, dec_layers=1, vocab=5000, kernel=31)
    w = random_weights(cfg, seed=0)
    s2t = speech2text(cfg, w, beam_size=2, ctc_weight=0.3)
    o = oracle.OracleSpeech2Text(cfg, w, beam_size=2, ctc_weight=0.3)
    waves = [refbuild.waveform(i, 80000) for i in range(8)]
    got = s2t.ctc_greedy(waves)
    speech, sl = s2t._to_batch(waves)
    enc, elens = s2t.asr_model.encode(speech, sl)
    lg = s2t.asr_model.ctc.logits(enc)
    checked = 0
    for i, wv in enumerate(waves):
        ref_enc = o.encode(wv)
        ref_lg = OE.ctc_logits(ref_enc, o.w)
        err = _maxerr(lg[i, : ref_lg.shape[0]], ref_lg)
        top2 = ref_lg.topk(2, dim=-1)[0]
        margin = (top2[:, 0] - top2[:, 1]).min().item()
        _, ids = OE.ctc_greedy(ref_enc, o.w)
        print(f"utt{i}: logit max abs err {err:.2e}, min top-2 margin {margin:.2e}, tokens {len(ids)}")
        assert err < 2 * enc_tol()          # logits of a V=5000 head on O(1) encoder outputs
        if margin > 20 * err:
            assert got[i] == ids.tolist()
            checked += 1
        else:  # frames inside the error band may flip: demand identity of all frames whose own margin is safe
            am_ref = ref_lg.argmax(-1)
            am_got = lg[i, : ref_lg.shape[0]].argmax(-1).cpu()
            safe = (top2[:, 0] - top2[:, 1]) > 20 * err
            assert bool((am_ref[safe] == am_got[safe]).all())
    print(f"{checked}/8 utterances compared for exact token identity")


def test_config1_like_joint_decode_vs_oracle():
    """Conformer (4L/256d) + 2L decoder, V=5000, joint CTC/attention beam 10 on 2 x 5 s, first 6 steps: identical n-best sequences."""
    torch.set_num_threads(min(16, torch.get_num_threads()))
    cfg = dict(d_model=256, heads=4, ff=1024, enc_layers=2, dec_layers=2, vocab=5000, kernel=31)
    w = random_weights(cfg, seed=3)
    kw = dict(beam_size=10, ctc_weight=0.3, maxlenratio=-6.0, nbest=3)
    s2t = speech2text(cfg, w, **kw)
    o = oracle.OracleSpeech2Text(cfg, w, **kw)
    waves = [refbuild.waveform(100 + i, 80000) for i in range(2)]
    res = s2t.batch_decode(waves)
    for i, wv in enumerate(waves):
        ref = o(wv)
        assert len(res[i]) == len(ref)
        for a, b in zip(res[i], ref):
            print(a[3].yseq.tolist(), a[3].score, b[3].score)
            assert a[3].yseq.tolist() == b[3].yseq.tolist()
            assert abs(a[3].score - b[3].score) <= 2e-4 * max(1.0, abs(b[3].score))


@pytest.mark.parametrize("heads,beam,ctc_weight", [(2, 20, 0.3), (8, 20, 0.3), (2, 32, 0.5), (8, 24, 0.0), (2, 20, 1.0)])
def test_wide_beam_vs_oracle(heads, beam, ctc_weight):
    """Beams wider than one cross-attention slot group (the reference default is beam 20): d_k = 64 takes the tensor-core
    cross-attention, d_k = 16 the FFMA one; n-best identical to the oracle."""
    cfg = dict(d_model=128, heads=heads, ff=256, enc_layers=2, dec_layers=2, vocab=80, kernel=15)
    w = random_weights(cfg, seed=11)
    kw = dict(beam_size=beam, ctc_weight=ctc_weight, maxlenratio=-8.0, nbest=5)
    s2t = speech2text(cfg, w, **kw)
    o = oracle.OracleSpeech2Text(cfg, w, **kw)
    waves = [refbuild.waveform(40 + i, n) for i, n in enumerate([16000, 11000])]
    res = s2t.batch_decode(waves)
    for i, wv in enumerate(waves):
        ref = o(wv)
        assert len(res[i]) == len(ref)
        for a, b in zip(res[i], ref):
            assert a[3].yseq.tolist() == b[3].yseq.tolist()
            assert abs(a[3].score - b[3].score) <= 2e-4 * max(1.0, abs(b[3].score))


def test_long_utterance_90s_ragged_batch_vs_oracle():
    """Maximum-size edge: a 90-s utterance (T = 2812 encoder frames: several key tiles beyond anything else in the suite, a 5623-column rel-pos
    band, the cross-attention and CTC recursions over 2812 frames) batched with a 2-s one; encoder output per utterance (atol 1e-4) and the joint
    beam-4 n-best of the first 5 steps vs the oracle."""
    torch.set_num_threads(min(16, torch.get_num_threads()))
    cfg = dict(d_model=128, heads=2, ff=256, enc_layers=2, dec_layers=1, vocab=60, kernel=15)
    w = random_weights(cfg, seed=21)
    kw = dict(beam_size=4, ctc_weight=0.3, maxlenratio=-5.0, nbest=2)
    s2t = speech2text(cfg, w, **kw)
    o = oracle.OracleSpeech2Text(cfg, w, **kw)
    waves = [refbuild.waveform(300, 90 * 16000), refbuild.waveform(301, 2 * 16000)]
    speech = torch.zeros(2, 90 * 16000)
    for i, wv in enumerate(waves):
        speech[i, : wv.numel()] = wv
    lens = torch.tensor([wv.numel() for wv in waves])
    enc, olens = s2t.asr_model.encode(speech.cuda(), lens.cuda())
    assert olens.tolist() == [2812, 62]
    for i, wv in enumerate(waves):
        ref_enc = o.encode(wv)
        got = enc[i, : int(olens[i])].cpu()
        assert got.shape == ref_enc.shape
        err = float((got - ref_enc).abs().max())
        print(f"utt {i}: T {int(olens[i])}, encoder max abs err {err:.2e}")
        assert err < 1e-4
    res = s2t.batch_decode(waves)
    for i, wv in enumerate(waves):
        ref = o(wv)
        assert len(res[i]) == len(ref)
        for a, b in zip(res[i], ref):
            assert a[3].yseq.tolist() == b[3].yseq.tolist()
            assert abs(a[3].score - b[3].score) <= 2e-4 * max(1.0, abs(b[3].score))


def test_beam_wider_than_64_is_refused():
    z, cfg, w = load("tiny")
    with pytest.raises(NotImplementedError):
        speech2text(cfg, w, beam_size=65, ctc_weight=0.3)


@pytest.mark.parametrize("beam,ctc_weight", [(60, 0.3), (40, 0.0), (48, 1.0)])
def test_beam_up_to_64_vs_oracle(beam, ctc_weight):
    """Beams beyond one warp of slots (the reference's Librispeech decode_asr.yaml uses beam 60, egs2/librispeech/asr1/conf/decode_asr.yaml:1-3):
    block-wide beam selection, pre-beam of 1.5 * beam candidates, four cross-attention slot groups; n-best identical to the oracle."""
    cfg = dict(d_model=128, heads=2, ff=256, enc_layers=2, dec_layers=2, vocab=150, kernel=15)
    w = random_weights(cfg, seed=13)
    kw = dict(beam_size=beam, ctc_weight=ctc_weight, maxlenratio=-6.0, nbest=8)
    s2t = speech2text(cfg, w, **kw)
    o = oracle.OracleSpeech2Text(cfg, w, **kw)
    waves = [refbuild.waveform(60 + i, n) for i, n in enumerate([14000, 9000])]
    res = s2t.batch_decode(waves)
    for i, wv in enumerate(waves):
        ref = o(wv)
        assert len(res[i]) == len(ref)
        for a, b in zip(res[i], ref):
            assert a[3].yseq.tolist() == b[3].yseq.tolist()
            assert abs(a[3].score - b[3].score) <= 2e-4 * max(1.0, abs(b[3].score))


def test_global_mvn_bit_exact_vs_reference_fixture(tmp_path):
    """GlobalMVN (espnet2/layers/global_mvn.py) for all four (norm_means, norm_vars) settings, npz and Kaldi-style stats files."""
    import os

    import espnet_b200

    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gmvn.npz"))
    stats = {k: z["stats_" + k] for k in ("count", "sum", "sum_square")}
    f_npz, f_npy = str(tmp_path / "stats.npz"), str(tmp_path / "stats.npy")
    np.savez(f_npz, **stats)
    kaldi = np.zeros((2, 81))
    kaldi[0, :80], kaldi[1, :80], kaldi[0, 80] = stats["sum"], stats["sum_square"], stats["count"]
    np.save(f_npy, kaldi)
    for f in (f_npz, f_npy):
        for nm in (1, 0):
            for nv in (1, 0):
                m = espnet_b200.GlobalMVN(f, norm_means=bool(nm), norm_vars=bool(nv)).cuda()
                x = torch.from_numpy(z["x"]).cuda()
                y, ol = m(x, torch.from_numpy(z["ilens"]).cuda())
                assert y.data_ptr() == x.data_ptr()
                np.testing.assert_array_equal(y.cpu().numpy(), z[f"y_m{nm}_v{nv}"])
                assert ol.tolist() == z["ilens"].tolist()


def test_speech2text_with_global_mvn_vs_oracle(tmp_path):
    """normalize: global_mvn in the model config (espnet2/tasks/asr.py normalize_choices) -- greedy ids and encoder output vs the oracle."""
    import argparse

    import espnet_b200

    cfg = dict(d_model=64, heads=4, ff=128, enc_layers=2, dec_layers=1, vocab=50, kernel=15)
    rng = np.random.RandomState(3)
    data = rng.randn(500, 80) * 2.0 - 3.0
    stats = dict(count=np.array(500), sum=data.sum(0), sum_square=(data * data).sum(0))
    f = str(tmp_path / "feats_stats.npz")
    np.savez(f, **stats)
    y = refbuild.model_yaml(cfg)
    y["normalize"], y["normalize_conf"] = "global_mvn", dict(stats_file=f)
    args = argparse.Namespace(**y)
    torch.manual_seed(5)
    model = espnet_b200.build_model(args)
    w = {k: v.detach().clone() for k, v in model.state_dict().items()}
    assert "normalize.mean" in w and "normalize.std" in w
    model = model.cuda().eval()
    wave = refbuild.waveform(9, 14000)
    speech = wave[None].cuda()
    enc, elens = model.encode(speech, torch.tensor([wave.numel()]).cuda())
    feats = OF.frontend_forward(wave, w["frontend.logmel.melmat"])
    mean, std = OF.global_mvn_stats(stats)
    fn = OF.global_mvn(feats[None], torch.tensor([feats.shape[0]]), mean, std)[0]
    ref = OE.conformer_encode(fn, w, cfg["heads"], cfg["enc_layers"])
    assert _maxerr(enc[0, : ref.shape[0]], ref) < enc_tol()


@pytest.mark.parametrize("groups", [2, 3])
def test_utterance_groups_on_streams_match_single_group(groups):
    """Large batches are searched as independent utterance groups on separate streams (own state / workspace / CUDA graphs);
    the n-best lists must be those of the single-group search, and of the oracle."""
    cfg = dict(d_model=64, heads=4, ff=128, enc_layers=2, dec_layers=2, vocab=60, kernel=15)
    w = random_weights(cfg, seed=7)
    kw = dict(beam_size=5, ctc_weight=0.3, maxlenratio=-12.0, nbest=5)
    s2t = speech2text(cfg, w, **kw)
    lens = [16000, 9000, 12345, 14000, 8000, 15000, 10000]
    waves = [refbuild.waveform(70 + i, n) for i, n in enumerate(lens)]
    bs = s2t.beam_search
    bs.group_min_utts, bs.n_groups = 10 ** 9, 1
    single = s2t.batch_decode(waves)
    bs.group_min_utts, bs.n_groups = 2, groups
    for _ in range(2):   # second call replays the groups' cached CUDA graphs
        grouped = s2t.batch_decode(waves)
        assert len(grouped) == len(single) == len(waves)
        for a, b in zip(grouped, single):
            assert [h[3].yseq.tolist() for h in a] == [h[3].yseq.tolist() for h in b]
            for ha, hb in zip(a, b):
                assert abs(ha[3].score - hb[3].score) <= 1e-5 * max(1.0, abs(hb[3].score))
    o = oracle.OracleSpeech2Text(cfg, w, **kw)
    for i in (0, 4, 6):
        ref = o(waves[i])
        assert [h[3].yseq.tolist() for h in grouped[i]] == [h[3].yseq.tolist() for h in ref]


def test_cli_inference_writes_reference_style_result_dir(tmp_path):
    """espnet_b200.bin_asr_inference.inference (asr_inference.py:711-906): wav.scp in, {n}best_recog/{token,token_int,score} out, batch 2,
    a too-short utterance replaced by the reference's placeholder; tokens equal the direct API's."""
    import wave as wavmod

    from espnet_b200.bin_asr_inference import inference

    z, cfg, w = load("tiny")
    s2t = speech2text(cfg, w, beam_size=3, ctc_weight=0.3, maxlenratio=-6.0, nbest=2)
    lines = []
    waves = {"a": refbuild.waveform(1, 9000), "b": refbuild.waveform(2, 12000), "short": torch.zeros(600), "c": refbuild.waveform(3, 8000)}
    for k, x in waves.items():
        pcm = (x.clamp(-1, 1) * 32767).round().to(torch.int16).numpy()
        with wavmod.open(str(tmp_path / f"{k}.wav"), "wb") as f:
            f.setnchannels(1); f.setsampwidth(2); f.setframerate(16000); f.writeframes(pcm.tobytes())
        lines.append(f"{k} {tmp_path / (k + '.wav')}")
        waves[k] = torch.from_numpy(pcm.astype("float32") / 32768.0)
    (tmp_path / "wav.scp").write_text("\n".join(lines) + "\n")
    out = inference(str(tmp_path / "decode"), [(str(tmp_path / "wav.scp"), "speech", "sound")], batch_size=2, nbest=2, speech2text=s2t)
    tok = dict(ln.split(maxsplit=1) if " " in ln.strip() else (ln.strip(), "") for ln in (tmp_path / "decode/1best_recog/token_int").read_text().splitlines())
    assert set(tok) == {"a", "b", "short", "c"} and tok["short"].strip() == "2"
    for k in ("a", "b", "c"):
        ref = s2t(waves[k])
        assert tok[k].split() == [str(t) for t in ref[0][2]]
        assert out[k][0][3].yseq.tolist() == ref[0][3].yseq.tolist()
    assert (tmp_path / "decode/2best_recog/score").exists()
