"""-m gpu: intermediate and self-conditioned CTC on the CUDA path -- espb_softmax_rows_split_f32 against a float64 softmax, the Conformer
(fused and materialised attention) and Transformer encoders against the reference fixtures (every intermediate output and the output),
ragged batches against single-utterance calls, Speech2Text's n-best against the reference's (joint and CTC-only without a decoder),
ctc_greedy, and bin_asr_inference from a saved config and checkpoint.

Tolerances as tests/test_gpu_subsampling.py: encoder outputs atol 1e-4, n-best sequences identical and scores within rtol 1e-4."""
import math

import numpy as np
import pytest
import torch
import yaml

from golden_util import DEC_NAMES, decode_params, decode_results
from gpu_util import refbuild, speech2text
from interctc_fixture import CASES, build, feats, load_case, load_model_fixture, oracle
import refbuild_interctc  # noqa: E402  (tests/golden is on sys.path after interctc_fixture)

pytestmark = pytest.mark.gpu
TOL = 1e-4


@pytest.fixture(autouse=True)
def _interctc_yaml(monkeypatch):
    refbuild_interctc.install(monkeypatch)   # model yaml with cfg["ic_a"], cfg["ic_b"], cfg["ic_cond"], cfg["no_decoder"]


def _pitch(n):
    return (n + 31) // 32 * 32


@pytest.mark.parametrize("V", [1, 64, 37, 257, 2048, 2049, 5000, 5121, 8192, 8193, 50001])
def test_softmax_rows_split_vs_float64(V):
    """Row softmax into the hi / lo planes: every thread-count residue and each register-resident width (V <= 2048, 5120, 8192) and the
    three-pass kernel above.  Columns beyond V are NaN in the input, the output starts as NaN; hi has tf32 precision, hi + lo is the
    softmax, columns V..ldo-1 are +0 in both planes and rows beyond `rows` stay NaN."""
    from espnet_b200 import ops

    rows, ld = 7, V + 5
    ldo = _pitch(V) + (32 if V == 257 else 0)   # one case with a pitch wider than needed
    g = torch.Generator().manual_seed(V)
    x = torch.full((rows, ld), float("nan"))
    x[:, :V] = 4 * torch.randn(rows, V, generator=g)
    x[3, :V] = 0.0                              # uniform row
    x[4, : min(V, 3)] = 60.0                    # one or a few dominant logits
    x = x.cuda()
    out = torch.full((2, rows + 2, ldo), float("nan"), device="cuda")
    ops.call("espb_softmax_rows_split_f32", ops.ptr(x), rows, ld, V, ops.ptr(out), out[0].numel(), ldo)
    torch.cuda.synchronize()
    o = out.cpu()
    hi, lo = o[0, :rows], o[1, :rows]
    xd = x.cpu()[:, :V].double()
    ref = torch.softmax(xd, dim=-1)
    # p = expf(d) / s with d = x - max rounded to float32 (an error of up to |d| 2^-24 in the exponent, the same in the float32 torch
    # softmax), expf within 2 ulp, the block sum of V positive terms within (V / 256 + 8) ulp plus the p-weighted exponent errors of its
    # terms, one rounding in the division
    d = (xd - xd.max(dim=-1, keepdim=True).values).abs()
    tol = 2.0 ** -24 * (V / 256 + 16 + d + (ref * d).sum(-1, keepdim=True))
    err = ((hi[:, :V].double() + lo[:, :V].double()) - ref).abs() / ref.clamp_min(1e-30)
    print(f"V {V}: max rel err {float(err.max()):.3e}, max err / bound {float((err / tol).max()):.3f}")
    assert bool((err <= tol).all())
    assert bool(((hi.view(torch.int32) & 0x1FFF) == 0).all()) and bool(((lo.view(torch.int32) & 0x1FFF) == 0).all())
    assert bool((hi[:, V:] == 0).all()) and bool((lo[:, V:] == 0).all())
    assert not bool(torch.signbit(hi[:, V:]).any()) and not bool(torch.signbit(lo[:, V:]).any())
    assert bool(o[:, rows:].isnan().all())


def test_softmax_rows_split_refusals():
    from espnet_b200 import ops

    x = torch.randn(4, 64, device="cuda")
    out = torch.full((2, 4, 64), float("nan"), device="cuda")
    for rows, ld, V, plane, ldo in ((4, 64, 0, 256, 64), (4, 32, 64, 256, 64), (4, 64, 64, 256, 48), (4, 64, 64, 256, 32), (4, 64, 64, 255, 64),
                                    (-1, 64, 64, 256, 64)):
        with pytest.raises(RuntimeError, match="softmax_rows_split"):
            ops.call("espb_softmax_rows_split_f32", ops.ptr(x), rows, ld, V, ops.ptr(out), plane, ldo)
    assert bool(out.isnan().all())


@pytest.mark.parametrize("case", CASES)
def test_encoder_vs_reference_fixture(case):
    z, tag, cfg, idx, w = load_case(case)
    enc, ctc = build(cfg, w, "cuda")
    x = feats(z, tag)[None].cuda()
    (out, inter), olens, _ = enc(x, torch.tensor([x.shape[1]]), ctc=ctc)
    assert olens.tolist() == z[f"{tag}olens"].tolist() and [li for li, _ in inter] == idx
    for li, h in inter:
        e = float((h[0].cpu() - torch.from_numpy(z[f"{tag}inter{li}"])).abs().max())
        print(f"{case} intermediate {li}: max abs err {e:.3e}")
        assert e < TOL
    e = float((out[0].cpu() - torch.from_numpy(z[f"{tag}out"])).abs().max())
    print(f"{case} output: max abs err {e:.3e}")
    assert e < TOL


@pytest.mark.parametrize("case,lens", [("conf64", [203, 71, 150, 9]), ("conf16", [40, 161, 97]), ("tfm64", [150, 63, 9])])
def test_ragged_batch_equals_single_utterances(case, lens):
    z, tag, cfg, idx, w = load_case(case)
    enc, ctc = build(cfg, w, "cuda")
    g = torch.Generator().manual_seed(11)
    x = torch.randn(len(lens), max(lens), 80, generator=g)
    (out, inter), olens, _ = enc(x.cuda(), torch.tensor(lens), ctc=ctc)
    out, inter = out.cpu(), [(li, h.cpu()) for li, h in inter]
    assert bool(torch.isfinite(out).all())
    for i, n in enumerate(lens):
        T = int(olens[i])
        (alone, alone_inter), _, _ = enc(x[i:i + 1, :n].cuda(), torch.tensor([n]), ctc=ctc)
        ref, ref_inter, _ = oracle(cfg, w, idx, x[i, :n])
        e_alone = float((out[i, :T] - alone[0].cpu()).abs().max())
        e_ref = float((out[i, :T].double() - ref).abs().max())
        print(f"{case} utt{i} (T {T}): vs alone {e_alone:.3e}, vs oracle {e_ref:.3e}")
        assert e_alone < 2e-5 and e_ref < TOL
        for (li, h), (_, ha), (_, hr) in zip(inter, alone_inter, ref_inter):
            assert float((h[i, :T] - ha[0].cpu()).abs().max()) < 2e-5 and float((h[i, :T].double() - hr).abs().max()) < TOL


def _check_nbest(res, gold, dn):
    assert len(res) == len(gold) > 0, dn
    for (_, _, _, h), (yseq, score, _) in zip(res, gold):
        assert h.yseq.tolist() == yseq, dn
        assert abs(float(h.score) - score) <= TOL * max(1.0, abs(score)), (dn, float(h.score), score)


def test_speech2text_joint_vs_reference_fixture():
    z, cfg, w = load_model_fixture("interctc_s2t")
    wave = torch.from_numpy(z["wave"])
    s2t = speech2text(cfg, w, beam_size=2, ctc_weight=0.3)
    speech, sl = s2t._to_batch([wave])
    enc, _ = s2t.asr_model.encode(speech, sl)
    assert float((enc[0].cpu() - torch.from_numpy(z["enc"])).abs().max()) < TOL
    assert s2t.asr_model.enc_split(enc) is not None
    assert s2t.ctc_greedy([wave])[0] == z["ctc_greedy"].tolist()
    for dn in DEC_NAMES:
        _check_nbest(speech2text(cfg, w, nbest=10, **decode_params(z, dn))(z["wave"]), decode_results(z, dn), dn)


def test_speech2text_ctc_only_without_decoder_vs_reference_fixture():
    """The LibriSpeech-100 scctc setting: no decoder, ctc_weight 1.0; also decoded in a ragged batch with another utterance."""
    z, cfg, w = load_model_fixture("interctc_ctconly")
    wave = torch.from_numpy(z["wave"])
    assert speech2text(cfg, w, ctc_weight=1.0).ctc_greedy([wave])[0] == z["ctc_greedy"].tolist()
    for dn in ("ctc4", "ctc10"):
        s2t = speech2text(cfg, w, nbest=10, **decode_params(z, dn))
        assert s2t.asr_model.decoder is None
        _check_nbest(s2t(z["wave"]), decode_results(z, dn), dn)
        _check_nbest(s2t.batch_decode([refbuild.waveform(3, 9000), wave])[1], decode_results(z, dn), dn)


def test_bin_asr_inference_from_config_and_checkpoint(tmp_path):
    """bin_asr_inference over a wav.scp with a recipe-style config.yaml and checkpoint of the CTC-only model: the 1- and 2-best token ids and
    scores are those of Speech2Text on the same 16-bit PCM."""
    import wave as wavmod

    from espnet_b200.bin_asr_inference import main, read_sound

    z, cfg, w = load_model_fixture("interctc_ctconly")
    pcm = (np.clip(z["wave"], -1, 1) * 32767).astype(np.int16)
    with wavmod.open(str(tmp_path / "a.wav"), "wb") as f:
        f.setnchannels(1); f.setsampwidth(2); f.setframerate(16000); f.writeframes(pcm.tobytes())
    (tmp_path / "wav.scp").write_text(f"a {tmp_path / 'a.wav'}\n")
    (tmp_path / "config.yaml").write_text(yaml.safe_dump(refbuild.model_yaml(cfg)))
    torch.save(w, str(tmp_path / "model.pth"))
    main(["--output_dir", str(tmp_path / "dec"), "--data_path_and_name_and_type", f"{tmp_path / 'wav.scp'},speech,sound",
          "--asr_train_config", str(tmp_path / "config.yaml"), "--asr_model_file", str(tmp_path / "model.pth"), "--beam_size", "4",
          "--ctc_weight", "1.0", "--nbest", "2"])
    ref = speech2text(cfg, w, beam_size=4, ctc_weight=1.0, nbest=2)(read_sound(str(tmp_path / "a.wav")))
    assert len(ref) == 2
    for k in (1, 2):
        tok = (tmp_path / f"dec/{k}best_recog/token_int").read_text().split()
        assert tok[0] == "a" and tok[1:] == [str(t) for t in ref[k - 1][2]]
        score = float((tmp_path / f"dec/{k}best_recog/score").read_text().split()[1])
        assert math.isclose(score, float(ref[k - 1][3].score), rel_tol=1e-5, abs_tol=1e-5)
