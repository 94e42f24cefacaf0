"""-m gpu: the Branchformer encoder on the CUDA path -- the learned_ave pooling and the branch-merge kernels against float64 torch, the
encoder against the reference fixtures (concat, learned_ave, fixed_ave, one-branch layers) and the oracle, the whole Speech2Text, and the
LibriSpeech-recipe shape (egs2/librispeech/asr1/conf/tuning/train_asr_branchformer_hop_length160_e18_linear3072.yaml: 18 blocks, d 512, h 8,
cgmlp 3072, kernel 31, concat).

Tolerances as tests/test_gpu_large.py: encoder outputs atol 1e-4, n-best sequences identical and scores within rtol 2e-4."""
import math
import os
import sys

import numpy as np
import pytest
import torch

from golden_util import DEC_NAMES, GOLDEN_DIR, decode_params, decode_results, load

sys.path.insert(0, GOLDEN_DIR)
import refbuild  # noqa: E402
import refbuild_bf  # noqa: E402

pytestmark = pytest.mark.gpu
TOL = 1e-4
TAGS = ["A", "B", "C", "D", "E"]


@pytest.fixture(autouse=True, scope="module")
def _bf_yaml():
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(refbuild, "model_yaml", refbuild_bf.model_yaml)
        yield


def _enc_fixture(tag):
    z = np.load(os.path.join(GOLDEN_DIR, "branchformer_enc.npz"))
    cfg = dict(zip(z[f"{tag}:cfg_keys"].tolist(), (int(v) for v in z[f"{tag}:cfg_vals"])))
    return z, cfg, z[f"{tag}:cgmlp_weight"].tolist(), refbuild_bf.fixture_weights(z, prefix=f"{tag}:")


def _encoder(cfg, cw, w):
    import espnet_b200

    enc = espnet_b200.BranchformerEncoder(80, **refbuild_bf.encoder_conf(cfg, cw))
    enc.load_state_dict({k[len("encoder."):]: v for k, v in w.items()}, strict=True)
    return enc.cuda().eval()


# ---------------------------------------------------------------------------------------------------------------- pool / merge kernels
def _ragged(B, T, seed):
    """B lengths in [1, T]: 1, 31, 32, 33 (around the 32-row chunk), T, then random."""
    g = torch.Generator().manual_seed(seed)
    fixed = [1, 31, 32, 33, T, 7][:B]
    return [min(v, T) for v in fixed] + torch.randint(1, T + 1, (B - len(fixed),), generator=g).tolist()


def _pool_ref(x1, x2, lens, pool_w, pool_b, wt_w, wt_b):
    """branchformer_encoder.py:221-266 in float64, per utterance over its own rows."""
    D = x1.shape[-1]
    out = []
    for b, n in enumerate(lens):
        wk = []
        for k, x in enumerate((x1, x2)):
            xb = x[b, :n].double()
            s = (xb @ pool_w[k].double() + pool_b[k].double()) / math.sqrt(D)
            wk.append(torch.softmax(s, 0) @ xb @ wt_w[k].double() + wt_b[k].double())
        out.append(torch.softmax(torch.stack(wk), 0))
    return torch.stack(out)


@pytest.mark.parametrize("B,T,D", [(1, 1, 64), (3, 45, 128), (6, 97, 256), (64, 937, 512), (17, 300, 1024)])
def test_branch_pool_kernel_vs_float64(B, T, D):
    from espnet_b200.lib import call, ptr

    lens = _ragged(B, T, B * T + D) if B > 1 else [T]
    g = torch.Generator(device="cuda").manual_seed(B + T + D)
    cat = torch.randn(B, T, 2 * D, device="cuda", generator=g)
    cat[..., D:] = 0.5 * cat[..., D:] + 0.3          # the branches differ in scale and mean
    for b, n in enumerate(lens):
        cat[b, n:] = float("nan")                    # padded rows must not reach the pooling
    pool_w = torch.randn(2, D, device="cuda", generator=g) * 2.0
    pool_b = torch.randn(2, device="cuda", generator=g)
    wt_w = torch.randn(2, D, device="cuda", generator=g) / D ** 0.5
    wt_b = torch.tensor([1.5, -1.5], device="cuda")  # merge weights far from 0.5 / 0.5: a swapped branch shows
    part = torch.full((B * 2 * ((T + 31) // 32) * (D + 2),), float("nan"), device="cuda")
    mw = torch.full((B, 2), float("nan"), device="cuda")
    x1, x2 = cat[..., :D], cat[..., D:]
    call("espb_branch_pool_f32", ptr(x1), ptr(x2), 2 * D, B, T, D, ptr(torch.tensor(lens, dtype=torch.int32, device="cuda")), ptr(pool_w),
         ptr(pool_b), ptr(wt_w), ptr(wt_b), ptr(part), ptr(mw))
    torch.cuda.synchronize()
    ref = _pool_ref(x1.cpu(), x2.cpu(), lens, pool_w.cpu(), pool_b.cpu(), wt_w.cpu(), wt_b.cpu())
    err = (mw.double().cpu() - ref).abs().max().item()
    print(f"B {B} T {T} D {D}: merge weights max abs err {err:.2e}, min |w1 - w2| {(ref[:, 0] - ref[:, 1]).abs().min().item():.2f}")
    assert err < 1e-5
    assert (ref[:, 0] - ref[:, 1]).abs().mean().item() > 0.3


@pytest.mark.parametrize("learned", [True, False])
@pytest.mark.parametrize("B,T,D", [(1, 1, 64), (5, 77, 128), (64, 937, 512)])
def test_branch_merge_kernel_bitwise(B, T, D, learned):
    """Both products rounded before the add: the hi / lo planes are the tf32 split of torch's float32 w1 * x1 + w2 * x2, bit for bit."""
    from emu_backend import tf32_hi, tf32_lo
    from espnet_b200.lib import call, ptr

    g = torch.Generator(device="cuda").manual_seed(B * T + D + learned)
    M = B * T
    cat = torch.randn(M, 2 * D, device="cuda", generator=g)
    if learned:
        a = torch.rand(B, device="cuda", generator=g) * 0.3
        mw = torch.stack([a, 1 - a], 1).contiguous()          # w1 in [0, 0.3), w2 = 1 - w1
        w1, w2 = mw[:, :1].repeat_interleave(T, 0), mw[:, 1:].repeat_interleave(T, 0)
        c1 = c2 = 0.0
    else:
        mw, c1, c2 = None, 1.0 - 0.3, 0.3                      # fixed_ave: Python doubles, rounded once to float32
        w1, w2 = torch.tensor(c1, dtype=torch.float32, device="cuda"), torch.tensor(c2, dtype=torch.float32, device="cuda")
    out = torch.full((2, M, D), float("nan"), device="cuda")
    call("espb_branch_merge_f32", ptr(cat), ptr(cat[:, D:]), 2 * D, M, D, T, ptr(mw), c1, c2, ptr(out), M * D)
    torch.cuda.synchronize()
    y = (w1 * cat[:, :D]) + (w2 * cat[:, D:])
    hi = tf32_hi(y.cpu())
    assert torch.equal(out[0].cpu().view(torch.int32), hi.view(torch.int32))
    assert torch.equal(out[1].cpu().view(torch.int32), tf32_lo(y.cpu(), hi).view(torch.int32))
    y64 = w1.double() * cat[:, :D].double() + w2.double() * cat[:, D:].double()
    assert ((out[0] + out[1]).double() - y64).abs().max().item() < 1e-6 * max(1.0, y64.abs().max().item())


# ---------------------------------------------------------------------------------------------------------------- encoder
@pytest.mark.parametrize("mode", ["tc2", "simt"])
@pytest.mark.parametrize("tag", TAGS)
def test_encoder_vs_reference_fixture(tag, mode, monkeypatch):
    """A / E: d_k 64 -> fused attention (tc2); B / C / D: d_k 16 -> materialised attention.  simt: every GEMM on FFMA."""
    from espnet_b200 import ops

    monkeypatch.setattr(ops, "_GEMM_MODE", mode)
    z, cfg, cw, w = _enc_fixture(tag)
    enc = _encoder(cfg, cw, w)
    enc.trace = []
    feats = torch.from_numpy(z[f"{tag}:feats"])[None].cuda()
    out, olens, _ = enc(feats, torch.tensor([feats.shape[1]]).cuda())
    assert int(olens[0]) == int(z[f"{tag}:olens"][0]) == out.shape[1]
    for i in range(1, cfg["enc_layers"] + 1):
        err = float((enc.trace[i][0].cpu() - torch.from_numpy(z[f"{tag}:layer{i}"])).abs().max())
        print(f"{tag} {mode} layer {i} max abs err {err:.3e}")
        assert err < TOL
    assert float((out[0].cpu() - torch.from_numpy(z[f"{tag}:out"])).abs().max()) < TOL


@pytest.mark.parametrize("tag", TAGS)
def test_encoder_ragged_batch_vs_oracle(tag):
    """Lengths 7 (one encoder frame) to 700 feature frames; learned_ave pooling sees each utterance's own frames only."""
    from oracle.branchformer import branchformer_encode

    _, cfg, cw, w = _enc_fixture(tag)
    with torch.no_grad():
        for k in w:
            if "weight_proj" in k:
                w[k] = w[k] * 8.0              # merge weights far from 0.5 / 0.5
    enc = _encoder(cfg, cw, w)
    g = torch.Generator().manual_seed(3)
    lens = [700, 233, 7, 480, 47, 135]
    feats = torch.randn(len(lens), max(lens), 80, generator=g)
    out, olens, _ = enc(feats.cuda(), torch.tensor(lens).cuda())
    for i, n in enumerate(lens):
        ref = branchformer_encode(feats[i, :n], w, cfg["heads"], cfg["enc_layers"], cw)
        T = ref.shape[0]
        assert int(olens[i]) == T
        e = float((out[i, :T].cpu() - ref).abs().max())
        print(f"{tag} utt{i} (T={T}) max abs err {e:.3e}")
        assert e < TOL
        assert not bool(out[i, T:].any())


def test_speech2text_vs_reference_fixture():
    from gpu_util import speech2text

    z, cfg, _ = load("bf")
    w = refbuild_bf.fixture_weights(z)
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
RECIPE = dict(d_model=512, heads=8, ff=2048, enc_layers=18, dec_layers=6, vocab=5000, cgmlp=3072, cgmlp_kernel=31, merge=0, use_attn=1,
              use_cgmlp=1, encoder="branchformer")


def _maxerr(a, b):
    return (a.double().cpu() - torch.as_tensor(b).double()).abs().max().item()


def test_recipe_encoder_and_ctc_logits_vs_oracle():
    from gpu_util import random_weights, speech2text
    from oracle import encoder as OE
    from oracle.branchformer import BranchformerSpeech2Text

    torch.set_num_threads(min(16, torch.get_num_threads()))
    w = random_weights(RECIPE, seed=0)
    waves = [refbuild.waveform(500 + i, n) for i, n in enumerate([480000, 480000, 240000])]
    s2t = speech2text(RECIPE, w, beam_size=10, ctc_weight=0.3)
    o = BranchformerSpeech2Text(RECIPE, w)
    speech, sl = s2t._to_batch(waves)
    enc, elens = s2t.asr_model.encode(speech, sl)
    lg = s2t.asr_model.ctc.logits(enc, s2t.asr_model.enc_split(enc))
    assert elens.tolist() == [937, 937, 468]
    for i, wv in enumerate(waves):
        ref = o.encode(wv)
        e = _maxerr(enc[i, : ref.shape[0]], ref)
        el = _maxerr(lg[i, : ref.shape[0]], OE.ctc_logits(ref, o.w))
        print(f"utt{i} T={ref.shape[0]}: encoder max abs err {e:.3e}, logits max abs err {el:.3e}")
        assert e < TOL
        assert el < 2e-4
