"""-m gpu: the E-Branchformer encoder on the CUDA path -- GELU in the GEMM epilogue, the CSGU and merge kernels against torch, the
encoder against the reference fixtures and the oracle, the whole Speech2Text, and the LibriSpeech-recipe shape
(egs2/librispeech/asr1/conf/tuning/train_asr_e_branchformer.yaml: 17 blocks, d 512, h 8, cgmlp 3072, macaron FFN 1024, kernels 31 / 31).

Tolerances as tests/test_gpu_large.py: encoder outputs atol 1e-4, n-best sequences identical and scores within rtol 2e-4."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from golden_util import DEC_NAMES, GOLDEN_DIR, decode_params, decode_results, load

sys.path.insert(0, GOLDEN_DIR)
import refbuild  # noqa: E402
import refbuild_ebf  # noqa: E402

pytestmark = pytest.mark.gpu
TOL = 1e-4


@pytest.fixture(autouse=True, scope="module")
def _ebf_yaml():
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(refbuild, "model_yaml", refbuild_ebf.model_yaml)
        yield


def _enc_fixture(tag):
    z = np.load(os.path.join(GOLDEN_DIR, "ebranchformer_enc.npz"))
    cfg = dict(zip(z[f"{tag}:cfg_keys"].tolist(), (int(v) for v in z[f"{tag}:cfg_vals"])))
    return z, cfg, refbuild_ebf.fixture_weights(z, prefix=f"{tag}:")


def _encoder(cfg, w):
    import espnet_b200

    enc = espnet_b200.EBranchformerEncoder(80, **refbuild_ebf.encoder_conf(cfg))
    enc.load_state_dict({k[len("encoder."):]: v for k, v in w.items()}, strict=True)
    return enc.cuda().eval()


# ---------------------------------------------------------------------------------------------------------------- GELU epilogue
@pytest.mark.parametrize("mode", ["tc", "tc2", "simt"])
@pytest.mark.parametrize("M,N,K", [(937, 3072, 512), (200, 130, 96), (64, 256, 128)])
def test_gelu_epilogue(mode, M, N, K):
    from espnet_b200 import ops

    torch.manual_seed(M + N + K)
    a, b = torch.randn(M, K, device="cuda"), torch.randn(N, K, device="cuda") / K ** 0.5
    bias = torch.randn(N, device="cuda")
    ref = F.gelu((a.double() @ b.double().t() + bias.double()))
    out = torch.full((M, N), float("nan"), device="cuda")
    assert ops.linear(ops.split_from(a), ops.split_from(b), out, bias=bias, act=ops.ACT_GELU, force=mode) == (mode != "simt")
    assert (out.double() - ref).abs().max().item() < 3e-5
    # column-offset write into a wider buffer (ldc != N): columns outside [N0, N0 + N) stay untouched
    N0, ldc = 32, N + 64
    wide = torch.full((M, ldc), 7.0, device="cuda")
    ops.gemm(M, N, K, ops.split_from(a), M * K, K, ops.split_from(b), N * K, K, wide, ldc, bias=bias, act=ops.ACT_GELU, c_off=N0, force=mode)
    assert (wide[:, N0:N0 + N].double() - ref).abs().max().item() < 3e-5
    assert bool((wide[:, :N0] == 7.0).all()) and bool((wide[:, N0 + N:] == 7.0).all())


# ---------------------------------------------------------------------------------------------------------------- CSGU / merge kernels
LENS = [5, 200, 150]       # T < K, T > 128 (several time tiles), a ragged third


def _masked(x, lens):
    t = torch.arange(x.shape[1], device=x.device).view(1, -1, 1)
    return torch.where(t < torch.tensor(lens, device=x.device).view(-1, 1, 1), x, torch.zeros((), device=x.device))


def _dw(x, w, b):
    C, K = w.shape
    return F.conv1d(x.transpose(1, 2), w.view(C, 1, K), b, padding=(K - 1) // 2, groups=C).transpose(1, 2)


@pytest.mark.parametrize("K", [3, 7, 15, 31, 63, 127])   # 63 / 127: the run-time-K tile kernel at its widest halo
@pytest.mark.parametrize("Uh", [96, 200, 1536])
def test_csgu_kernel_vs_torch(K, Uh):
    from espnet_b200.lib import call, ptr

    g = torch.Generator(device="cuda").manual_seed(K * 1000 + Uh)
    B, T = len(LENS), max(LENS)
    h = torch.randn(B, T, 2 * Uh, device="cuda", generator=g)
    ln_g, ln_b = 1 + 0.3 * torch.randn(Uh, device="cuda", generator=g), 0.3 * torch.randn(Uh, device="cuda", generator=g)
    w, b = torch.randn(Uh, K, device="cuda", generator=g) / K ** 0.5, torch.randn(Uh, device="cuda", generator=g)
    lens = torch.tensor(LENS, dtype=torch.int32, device="cuda")
    stats = torch.empty(B * T, 2, device="cuda")
    out = torch.full((2, B * T, Uh), float("nan"), device="cuda")
    call("espb_csgu_f32", ptr(h), B, T, 2 * Uh, ptr(lens), ptr(ln_g), ptr(ln_b), 1e-12, ptr(w), ptr(b), K, ptr(stats), ptr(out), B * T * Uh)
    torch.cuda.synchronize()
    hd = h.double()
    gate = _masked(F.layer_norm(hd[..., Uh:], (Uh,), ln_g.double(), ln_b.double(), 1e-12), LENS)
    ref = _masked(hd[..., :Uh] * _dw(gate, w.double(), b.double()), LENS)
    got = (out[0] + out[1]).view(B, T, Uh)
    assert (got.double() - ref).abs().max().item() < 2e-5 * max(1.0, ref.abs().max().item())
    for i, n in enumerate(LENS):
        assert bool((out[:, i * T + n:(i + 1) * T] == 0).all())


@pytest.mark.parametrize("K", [3, 7, 15, 31, 63, 127])   # 63 / 127: the run-time-K tile kernel at its widest halo
@pytest.mark.parametrize("C2", [128, 200, 1024])
def test_merge_kernel_vs_torch(K, C2):
    from espnet_b200.lib import call, ptr

    g = torch.Generator(device="cuda").manual_seed(K * 1000 + C2)
    B, T = len(LENS), max(LENS)
    cat = torch.randn(B, T, C2, device="cuda", generator=g)
    w, b = torch.randn(C2, K, device="cuda", generator=g) / K ** 0.5, torch.randn(C2, device="cuda", generator=g)
    lens = torch.tensor(LENS, dtype=torch.int32, device="cuda")
    out = torch.full((2, B * T, C2), float("nan"), device="cuda")
    call("espb_merge_dwconv_f32", ptr(cat), B, T, C2, ptr(lens), ptr(w), ptr(b), K, ptr(out), B * T * C2)
    torch.cuda.synchronize()
    x = _masked(cat.double(), LENS)
    ref = _masked(x + _dw(x, w.double(), b.double()), LENS)
    got = (out[0] + out[1]).view(B, T, C2)
    assert (got.double() - ref).abs().max().item() < 2e-5 * max(1.0, ref.abs().max().item())
    for i, n in enumerate(LENS):
        assert bool((out[:, i * T + n:(i + 1) * T] == 0).all())


# ---------------------------------------------------------------------------------------------------------------- encoder
@pytest.mark.parametrize("mode", ["tc2", "simt"])
@pytest.mark.parametrize("tag", ["A", "B"])
def test_encoder_vs_reference_fixture(tag, mode, monkeypatch):
    """A: d_k 64 -> fused attention (tc2); B: d_k 16 -> materialised attention, no FFN, merge kernel 3.  simt: every GEMM on FFMA."""
    from espnet_b200 import ops

    monkeypatch.setattr(ops, "_GEMM_MODE", mode)
    z, cfg, w = _enc_fixture(tag)
    enc = _encoder(cfg, w)
    enc.trace = []
    feats = torch.from_numpy(z[f"{tag}:feats"])[None].cuda()
    out, olens, _ = enc(feats, torch.tensor([feats.shape[1]]).cuda())
    assert int(olens[0]) == int(z[f"{tag}:olens"][0]) == out.shape[1]
    for i in range(1, cfg["enc_layers"] + 1):
        err = float((enc.trace[i][0].cpu() - torch.from_numpy(z[f"{tag}:layer{i}"])).abs().max())
        print(f"{tag} {mode} layer {i} max abs err {err:.3e}")
        assert err < TOL
    assert float((out[0].cpu() - torch.from_numpy(z[f"{tag}:out"])).abs().max()) < TOL


@pytest.mark.parametrize("tag", ["A", "B"])
def test_encoder_ragged_batch_vs_oracle(tag):
    from oracle.e_branchformer import ebranchformer_encode

    _, cfg, w = _enc_fixture(tag)
    enc = _encoder(cfg, w)
    g = torch.Generator().manual_seed(3)
    lens = [700, 233, 480, 47]            # T = 174, 57, 119, 11: halos of both convs cross the utterance ends
    feats = torch.randn(len(lens), max(lens), 80, generator=g)
    out, olens, _ = enc(feats.cuda(), torch.tensor(lens).cuda())
    for i, n in enumerate(lens):
        ref = ebranchformer_encode(feats[i, :n], w, cfg["heads"], cfg["enc_layers"])
        T = ref.shape[0]
        assert int(olens[i]) == T
        e = float((out[i, :T].cpu() - ref).abs().max())
        print(f"{tag} utt{i} (T={T}) max abs err {e:.3e}")
        assert e < TOL
        assert not bool(out[i, T:].any())


def test_speech2text_vs_reference_fixture():
    from gpu_util import speech2text

    z, cfg, _ = load("ebf")
    w = refbuild_ebf.fixture_weights(z)
    s2t = speech2text(cfg, w, beam_size=2, ctc_weight=0.3)
    wave = torch.from_numpy(z["wave"])
    speech, sl = s2t._to_batch([wave])
    enc, _ = s2t.asr_model.encode(speech, sl)
    assert float((enc[0].cpu() - torch.from_numpy(z["enc"])).abs().max()) < TOL
    assert s2t.ctc_greedy([wave])[0] == z["ctc_greedy"].tolist()
    for dn in DEC_NAMES:
        res = speech2text(cfg, w, nbest=10, **decode_params(z, dn))(z["wave"])
        gold = decode_results(z, dn)
        assert len(res) == len(gold), dn
        for (_, _, _, h), (yseq, score, _) in zip(res, gold):
            assert h.yseq.tolist() == yseq, dn
            assert abs(h.score - score) <= 2e-4 * max(1.0, abs(score))


# ---------------------------------------------------------------------------------------------------------------- recipe shape
RECIPE = dict(d_model=512, heads=8, ff=1024, enc_layers=17, dec_layers=6, vocab=5000, cgmlp=3072, cgmlp_kernel=31, merge_kernel=31,
              use_ffn=1, macaron=1, encoder="e_branchformer")


@pytest.fixture(scope="module")
def recipe(_ebf_yaml):
    from gpu_util import random_weights

    torch.set_num_threads(min(16, torch.get_num_threads()))
    w = random_weights(RECIPE, seed=0)
    waves = [refbuild.waveform(400 + i, n) for i, n in enumerate([480000, 480000, 240000])]
    return w, waves


def _maxerr(a, b):
    return (a.double().cpu() - torch.as_tensor(b).double()).abs().max().item()


def test_recipe_encoder_and_ctc_greedy_vs_oracle(recipe):
    from gpu_util import speech2text
    from oracle import encoder as OE
    from oracle.e_branchformer import EBranchformerSpeech2Text

    w, waves = recipe
    s2t = speech2text(RECIPE, w, beam_size=10, ctc_weight=0.3)
    o = EBranchformerSpeech2Text(RECIPE, w, beam_size=10, ctc_weight=0.3)
    speech, sl = s2t._to_batch(waves)
    enc, elens = s2t.asr_model.encode(speech, sl)
    lg = s2t.asr_model.ctc.logits(enc, s2t.asr_model.enc_split(enc))
    greedy = s2t.ctc_greedy(waves)
    assert elens.tolist() == [937, 937, 468]
    for i, wv in enumerate(waves):
        ref = o.encode(wv)
        e = _maxerr(enc[i, : ref.shape[0]], ref)
        ref_lg = OE.ctc_logits(ref, o.w)
        el = _maxerr(lg[i, : ref.shape[0]], ref_lg)
        top2 = ref_lg.topk(2, dim=-1)[0]
        gap = top2[:, 0] - top2[:, 1]
        print(f"utt{i} T={ref.shape[0]}: encoder max abs err {e:.3e}, logits max abs err {el:.3e}, min top-2 margin {gap.min().item():.3e}")
        assert e < TOL
        assert el < 2e-4
        _, ids = OE.ctc_greedy(ref, o.w)
        if gap.min().item() > 20 * el:
            assert greedy[i] == ids.tolist()
        safe = gap > 20 * el
        assert bool((ref_lg.argmax(-1)[safe] == lg[i, : ref.shape[0]].argmax(-1).cpu()[safe]).all())
        assert int(safe.sum()) > 0.9 * ref.shape[0]


def test_recipe_joint_beam10_vs_oracle(recipe):
    from gpu_util import speech2text
    from oracle.e_branchformer import EBranchformerSpeech2Text

    w, waves = recipe
    kw = dict(beam_size=10, ctc_weight=0.3, maxlenratio=-8.0, nbest=5)
    res = speech2text(RECIPE, w, **kw).batch_decode(waves)
    o = EBranchformerSpeech2Text(RECIPE, w, **kw)
    for i in (0, 2):
        ref = o(waves[i])
        assert len(res[i]) == len(ref) > 0
        for a, b in zip(res[i], ref):
            assert a[3].yseq.tolist() == b[3].yseq.tolist()
            assert abs(a[3].score - b[3].score) <= 2e-4 * max(1.0, abs(b[3].score))
