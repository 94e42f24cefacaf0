"""-m gpu: the conv2d2 / conv2d6 / conv2d8 input layers on the CUDA path -- the phase-split conv1 kernel, the implicit-GEMM convolutions of
EspbGemmDesc.a_mode 1..3 and the phase re-layout against float64 torch in every GEMM mode, the nine (encoder, input layer) cases against the
reference fixtures layer by layer, ragged batches against single-utterance calls, the whole Speech2Text of a conv2d6 Conformer against the
reference's n-best lists, and the ReazonSpeech recipe shape (egs2/reazonspeech/asr1/conf/train_asr_conformer.yaml: Conformer 12 blocks,
d 512, h 8, conv2d6) against the oracle.

Tolerances as tests/test_gpu_large.py and tests/test_gpu_zz_next.py: encoder outputs atol 1e-4, n-best sequences identical and scores within
rtol 1e-4."""
import math

import pytest
import torch
import torch.nn.functional as F

from golden_util import DEC_NAMES, decode_params, decode_results, load
from gpu_util import random_weights, refbuild, speech2text
from oracle.subsampling import SubsamplingSpeech2Text
from subsampling_fixture import PAIRS, build_encoder, feats, load_case, oracle_encode

import refbuild_ebf  # noqa: E402  (tests/golden is on sys.path after subsampling_fixture)
import refbuild_subsampling  # noqa: E402

pytestmark = pytest.mark.gpu
TOL = 1e-4


@pytest.fixture(autouse=True)
def _input_layer_yaml(monkeypatch):
    refbuild_subsampling.install(monkeypatch)   # model yaml with cfg["input_layer"]


def _unphase(a, s, T, Fr):
    """[B][plane*s*s + (t%s)*s + (f%s)][Fh][Th][C] (hi + lo) -> [B][C][T][F]."""
    B, _, Fh, Th, C = a.shape
    v = (a[:, : s * s] + a[:, s * s:]).view(B, s, s, Fh, Th, C)   # [B][pt][pf][fh][th][C]
    v = v.permute(0, 5, 4, 1, 3, 2).reshape(B, C, Th * s, Fh * s)   # t = th*s + pt, f = fh*s + pf
    return v[:, :, :T, :Fr]


@pytest.mark.parametrize("mode", ["tc", "tc2", "simt"])
@pytest.mark.parametrize("C", [32, 512])
@pytest.mark.parametrize("input_layer", ["conv2d", "conv2d2", "conv2d6", "conv2d8"])
def test_conv_stack_vs_float64(mode, C, input_layer):
    """conv1 into the phases of the next stride, each implicit-GEMM conv, and (conv2d8) the re-layout between them; T_f 63 / F 47 give
    conv1 extents 31 x 23, which no stride divides."""
    from espnet_b200 import ops
    from espnet_b200.layers import _A_MODE, SUBSAMPLING

    geo = SUBSAMPLING[input_layer]
    B, Tf, Fin = 2, 63, 47
    g = torch.Generator().manual_seed(C + len(input_layer))
    fe = torch.randn(B, Tf, Fin, generator=g)
    w1, b1 = torch.randn(C, 1, 3, 3, generator=g) / 3, 0.1 * torch.randn(C, generator=g)
    ref = torch.relu(F.conv2d(fe.double()[:, None], w1.double(), b1.double(), stride=2))
    T1, F1 = ref.shape[2:]
    s = geo[0][1]
    Th, Fh = -(-T1 // s), -(-F1 // s)
    a = torch.zeros(B, 2 * s * s, Fh, Th, C, device="cuda")
    dev = [t.cuda() for t in (fe, w1.view(C, 9), b1)]   # referenced until the launch is enqueued
    ops.call("espb_conv1_relu_phase_f32", ops.ptr(dev[0]), B, Tf, Fin, ops.ptr(dev[1]), ops.ptr(dev[2]), C, ops.ptr(a), T1, F1, s, Th, Fh)
    assert (_unphase(a, s, T1, F1).double().cpu() - ref).abs().max().item() < 1e-5
    for i, (k, s) in enumerate(geo):
        K = k * k * C
        w, b = torch.randn(C, C, k, k, generator=g) / math.sqrt(K), 0.1 * torch.randn(C, generator=g)
        ref = torch.relu(F.conv2d(ref, w.double(), b.double(), stride=s))
        To, Fo = ref.shape[2:]
        c = torch.full((2, B, Fo, To, C), float("nan"), device="cuda")
        used_tc = ops.gemm(To, C, K, a, 0, 0, ops.split_from(w.permute(0, 2, 3, 1).reshape(C, K).cuda()), C * K, K, c, C,
                           c_plane=B * Fo * To * C, split_out=True, bias=b.cuda(), act=ops.ACT_RELU, nbx=Fo, nby=B, sc=(To * C, Fo * To * C),
                           a_mode=_A_MODE[(k, s)], conv=(Th, Fh, C), force=mode)
        assert used_tc == (mode != "simt")
        err = ((c[0] + c[1]).permute(0, 3, 2, 1).double().cpu() - ref).abs().max().item()
        print(f"{input_layer} conv {i + 2} (k {k}, s {s}) C {C} {mode}: max abs err {err:.3e}")
        # tc accumulates all of K inside the tensor core: its error grows with K (tests/test_gpu_gemm.py: _tol)
        assert err < (TOL + 1e-7 * K if mode == "tc" else TOL)
        if i + 1 < len(geo):
            s = geo[i + 1][1]
            Th, Fh = -(-To // s), -(-Fo // s)
            a = torch.zeros(B, 2 * s * s, Fh, Th, C, device="cuda")
            ops.call("espb_phase_split_f32", ops.ptr(c), B * Fo * To * C, B, Fo, To, C, s, Th, Fh, ops.ptr(a))
            assert torch.equal(_unphase(a, s, To, Fo), (c[0] + c[1]).permute(0, 3, 2, 1))


@pytest.mark.parametrize("encoder,input_layer", PAIRS)
def test_encoder_vs_reference_fixture(encoder, input_layer):
    z, tag, cfg, w = load_case(encoder, input_layer)
    enc = build_encoder(encoder, input_layer, cfg, w).cuda()
    enc.trace = []
    x = feats(z, tag)[None].cuda()
    out, olens, _ = enc(x, torch.tensor([x.shape[1]]).cuda())
    assert int(olens[0]) == int(z[f"{tag}olens"][0]) == out.shape[1]
    for i in range(cfg["enc_layers"] + 1):
        err = float((enc.trace[i][0].cpu() - torch.from_numpy(z[f"{tag}layer{i}"])).abs().max())
        print(f"{encoder} {input_layer} layer {i} max abs err {err:.3e}")
        assert err < TOL
    assert float((out[0].cpu() - torch.from_numpy(z[f"{tag}out"])).abs().max()) < TOL


@pytest.mark.parametrize("encoder,input_layer,lens", [
    ("conformer", "conv2d6", [11, 301, 130, 257, 64]),    # the minimum, then residues 1, 4, 5, 4 modulo 6
    ("transformer", "conv2d8", [15, 347, 170, 260]),      # the minimum, then residues 3, 2, 4 modulo 8
    ("e_branchformer", "conv2d8", [230, 15, 99]),
    ("e_branchformer", "conv2d2", [7, 180, 95]),
])
def test_ragged_batch_equals_single_utterances(encoder, input_layer, lens):
    z, tag, cfg, w = load_case(encoder, input_layer)
    enc = build_encoder(encoder, input_layer, cfg, w).cuda()
    g = torch.Generator().manual_seed(9)
    x = torch.zeros(len(lens), max(lens), 80)
    for i, n in enumerate(lens):
        x[i, :n] = torch.randn(n, 80, generator=g)
    out, olens, _ = enc(x.cuda(), torch.tensor(lens).cuda())
    out = out.cpu()
    for i, n in enumerate(lens):
        alone, ol, _ = enc(x[i:i + 1, :n].cuda(), torch.tensor([n]).cuda())
        T = int(ol[0])
        assert T == int(olens[i]) >= 1
        e_alone = float((out[i, :T] - alone[0].cpu()).abs().max())
        ref, _ = oracle_encode(encoder, input_layer, cfg, w, x[i, :n])
        e_ref = float((out[i, :T] - ref).abs().max())
        print(f"{encoder} {input_layer} utt{i} (T_f {n}, T {T}): vs alone {e_alone:.3e}, vs oracle {e_ref:.3e}")
        assert e_alone < 2e-5 and e_ref < TOL


def test_conv2d6_conformer_speech2text_vs_reference_fixture():
    z, cfg, _ = load("subsampling_s2t")
    w = refbuild_ebf.fixture_weights(z)
    cfg["input_layer"] = str(z["input_layer"])
    wave = torch.from_numpy(z["wave"])
    s2t = speech2text(cfg, w, beam_size=2, ctc_weight=0.3)
    speech, sl = s2t._to_batch([wave])
    enc, _ = s2t.asr_model.encode(speech, sl)
    assert float((enc[0].cpu() - torch.from_numpy(z["enc"])).abs().max()) < TOL
    assert s2t.ctc_greedy([wave])[0] == z["ctc_greedy"].tolist()
    for dn in DEC_NAMES:
        res = speech2text(cfg, w, nbest=10, **decode_params(z, dn))(z["wave"])
        gold = decode_results(z, dn)
        assert len(res) == len(gold) > 0, dn
        for (_, _, _, h), (yseq, score, _) in zip(res, gold):
            assert h.yseq.tolist() == yseq, dn
            assert abs(float(h.score) - score) <= 1e-4 * max(1.0, abs(score)), (dn, float(h.score), score)


REAZON = dict(d_model=512, heads=8, ff=2048, enc_layers=12, dec_layers=6, vocab=5000, kernel=31, input_layer="conv2d6")


def test_reazonspeech_shape_vs_oracle():
    """The ReazonSpeech Conformer (12 blocks, d 512, h 8, conv2d6) on 2 x 30 s + 15 s: encoder output per utterance and the joint
    CTC/attention beam-10 n-best of the first 8 steps against the oracle."""
    torch.set_num_threads(min(16, torch.get_num_threads()))
    w = random_weights(REAZON, seed=0)
    waves = [refbuild.waveform(300 + i, n) for i, n in enumerate([480000, 480000, 240000])]
    kw = dict(beam_size=10, ctc_weight=0.3, maxlenratio=-8.0, nbest=5)
    s2t = speech2text(REAZON, w, **kw)
    o = SubsamplingSpeech2Text(REAZON, w, **kw)
    speech, sl = s2t._to_batch(waves)
    enc, elens = s2t.asr_model.encode(speech, sl)
    assert elens.tolist() == [624, 624, 311]
    for i, wv in enumerate(waves):
        ref = o.encode(wv)
        e = float((enc[i, : ref.shape[0]].cpu() - ref).abs().max())
        print(f"utt{i} T={ref.shape[0]}: encoder max abs err {e:.3e}")
        assert ref.shape[0] == int(elens[i]) and e < TOL
    res = s2t.batch_decode(waves)
    for i in (0, 2):
        ref = o(waves[i])
        assert len(res[i]) == len(ref) > 0
        for a, b in zip(res[i], ref):
            assert a[3].yseq.tolist() == b[3].yseq.tolist()
            assert abs(a[3].score - b[3].score) <= 2e-4 * max(1.0, abs(b[3].score))
