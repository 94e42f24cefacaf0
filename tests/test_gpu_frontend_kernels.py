"""The frontend kernels (csrc/frontend.cu) one by one through the C ABI: espb_stft_logmel_f32, espb_frontend_blocks,
espb_utt_mvn_from_partial_f32, espb_utt_mvn_f32 and espb_global_mvn_f32.  The GPU tests carry pytest.mark.gpu one by one; the CPU tests
of this file run anywhere.

Reference, per utterance, float64 numpy: reflect-pad the samples < len by 256 on both sides (torch.stft center=True), take frame t at
t*hop, multiply by the float32 window the kernel receives (win_length taps zero-padded around the centre to 512, built by
DefaultFrontend._constants), rfft, |X|^2, @ melmat (its float32 values), clamp at 1e-10f, ln.  Every sample at or beyond an utterance's
length is NaN, every output starts NaN, and Tf_max is a few blocks larger than needed: padded frames must be exactly +0, and the
elements past the outputs must stay NaN.

Tolerance of the log-mel features, per element, u = 2^-24.
* FFT.  The kernel packs the windowed frame into 256 complex points (one rounding per product x w), runs a 16 x 16 four-step FFT (two
  16-point DFTs of two radix-4 levels each with a twiddle multiplication between them, and the W256 twiddles between the DFTs) and the
  real-FFT split (add, product with a float32 W512 twiddle, add).
  Each add level rounds once, each product with a float32 twiddle carries 2 roundings and the twiddle's own error: 23 roundings on any
  path.  Each level maps the vector by a matrix that is sqrt(r) times unitary, so a level's rounding errors reach X with an L2 norm of
  at most u sqrt(2 * 256) ||w x||_2 (complex components), and one element of X is bounded by the L2 norm of the error vector:
  |dX_k| <= eX = 34 u * 16 ||w x||_2  (23 sqrt(2) < 34; ||w x||_2 the frame's windowed energy, sqrt(256) = 16).
* Power and mel.  dP_k <= 2 |X_k| eX + eX^2 + 3u P_k.  The fmaf chain over a filter's `count` bins adds count u M (positive terms):
  dM = sum_k w_k dP_k + count u M.
* Log.  logf is within 1 ulp (2u |ln M| relative).  Where dM <= M / 2: |got - ln M| <= dM / (M - dM) + 2u (|ln M| + |got|).  Where the
  bound exceeds half the mel power (quiet bands next to a loud tone), the element is compared in the power domain:
  |exp(got) - max(M, 1e-10f)| <= dM + 3u |got| exp(got).  Where M + dM < 1e-10f the element must be ln(1e-10f) within 1 ulp (digital
  silence, filters with no non-zero bin).
* partial[b][blk][m] is the sum of the kernel's own log-mel rows < Tf in frames [32 blk, 32 blk + 32): each half warp sums its 4 frames
  and the block adds at most 8 such sums, so it is within (32 + 8) u sum |x| of the float64 column sum; blocks with no frame < Tf are
  exactly 0.
* UtteranceMVN: the mean adds the nblk block sums in sequence and divides once, y = x - mean rounds once:
  tol = (40 + nblk + 2) u sum_t |x_t| / Tf + u |y|, against float64 mean subtraction of the kernel's own features.
* GlobalMVN is compared bit for bit with the reference's float32 op order (oracle.frontend.global_mvn).
test_tolerances_catch_plausible_bugs checks on the CPU that each plausible bug moves the float64 reference by more than 10x the
tolerance at a tested shape: reflect padding that repeats the edge sample, the symmetric (non-periodic) Hann window, a short window
left-aligned instead of centred, frames one sample late, the Nyquist bin dropped and an MVN mean taken over Tf_max instead of Tf.

Rows t >= len of espb_utt_mvn_f32's input are neither read nor written.  The reference's UtteranceMVN subtracts the mean from the padded
rows of a zero-padded batch too (they become -mean); those rows are outside the per-utterance semantics (DESIGN.md: every utterance
sees its own frames only), and the test pins that they stay as they were.
"""
import numpy as np
import pytest
import torch

gpu = pytest.mark.gpu

U32 = 2.0 ** -24
NAN = float("nan")
NAN_BITS = int(np.float32(NAN).view(np.int32))
FLOOR = float(np.float32(1e-10))
LOG_FLOOR = float(np.float32(np.log(FLOOR)))

_KEEP = []    # device copies made inline in a call's argument list: only a raw pointer reaches the library, so keep the tensors alive


@pytest.fixture(autouse=True)
def _release_inputs():
    yield
    if _KEEP:
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


def _all_nan_bits(t):
    return bool((t.view(torch.int32) == NAN_BITS).all())


def _tables(device, **kw):
    """DefaultFrontend(**kw): the object and the device tables its forward passes to the kernel (sparse mel filters, window, twiddles)."""
    from espnet_b200 import DefaultFrontend

    fe = DefaultFrontend(**kw)
    return fe, fe._constants(torch.device(device))


# ============================================================================================================== signals
def _noise(rng, n):
    return rng.integers(-32768, 32768, n).astype(np.float32)


def _tone(rng, n, k=37):
    return (20000.0 * np.sin(2 * np.pi * k * np.arange(n) / 512)).astype(np.float32)     # on the centre of bin k


def _dc(rng, n):
    return (3000.0 + 0.05 * _noise(rng, n)).astype(np.float32)


def _impulse(rng, n):
    x = np.zeros(n, dtype=np.float32)
    x[n // 3] = 32767.0
    return x


def _silence(rng, n):
    x = _noise(rng, n)
    x[n // 4:n // 4 + 2000] = 0          # several whole frames of digital silence
    return x


# ============================================================================================================== reference
def _frames(x, n, hop, pad_mode="reflect", late=0):
    xs = x[:n].astype(np.float64)
    pad = np.pad(xs, 256 + 1, mode=pad_mode)[1:]            # one sample beyond the reflection, for frames one sample late
    Tf = 1 + n // hop
    return pad[np.arange(Tf)[:, None] * hop + np.arange(512)[None, :] + late]


def _reference(x, n, hop, window, melmat, count, pad_mode="reflect", late=0, drop_nyquist=False):
    """float64 (M, dM): mel power [Tf][n_mels] of the samples x[:n] and its error bound."""
    fr = _frames(x, n, hop, pad_mode, late) * np.asarray(window, dtype=np.float64)
    X = np.fft.rfft(fr, axis=-1)
    if drop_nyquist:
        X[:, 256] = 0
    P = X.real ** 2 + X.imag ** 2
    W = np.asarray(melmat, dtype=np.float64)
    M = P @ W
    eX = 34 * U32 * 16 * np.sqrt((fr ** 2).sum(-1, keepdims=True))
    dP = 2 * np.abs(X) * eX + eX ** 2 + 3 * U32 * P
    return M, dP @ W + np.asarray(count, dtype=np.float64) * U32 * M


def _log_tol(M, dM):
    return dM / np.maximum(M - dM, 1e-300) + 2 * U32 * np.abs(np.log(np.maximum(M, FLOOR)))


def _check_logmel(got, M, dM, what):
    got = got.astype(np.float64)
    floor = M + dM < FLOOR
    logd = ~floor & (dM <= 0.5 * M)
    powd = ~floor & ~logd
    err = np.abs(got[floor] - LOG_FLOOR)
    assert (err <= abs(np.spacing(np.float32(LOG_FLOOR)))).all(),f"{what}: silent element is not ln(1e-10f) (max err {err.max():.3e})"
    ref = np.log(np.maximum(M[logd], FLOOR))
    tol = _log_tol(M[logd], dM[logd]) + 2 * U32 * np.abs(got[logd])
    err = np.abs(got[logd] - ref)
    if err.size:
        assert (err <= tol).all(), f"{what}: max log err {err.max():.3e}, worst err/tol {(err / tol).max():.2f}"
    eg = np.exp(got[powd])
    err = np.abs(eg - np.maximum(M[powd], FLOOR))
    tol = dM[powd] + 3 * U32 * np.abs(got[powd]) * eg
    if err.size:
        assert (err <= tol).all(), f"{what}: power-domain worst err/tol {(err / tol).max():.2f}"
    return int(floor.sum()), int(logd.sum()), int(powd.sum())


# ============================================================================================================== kernel runs
def _stft(c, n_mels, hop, waves, lens, off=0, extra=2, Lmax=None, Tf_max=None):
    """One espb_stft_logmel_f32 call on the batch [B][Lmax] (samples >= len NaN) starting `off` floats into its buffer, Tf_max `extra`
    blocks (+5 frames) beyond the longest utterance's frame count.  Returns out [B][Tf_max][n_mels], partial [B][nblk][n_mels] (numpy)."""
    from espnet_b200 import lib

    B = len(lens)
    Lmax = max(lens) if Lmax is None else Lmax
    buf = np.full(off + B * Lmax, np.nan, dtype=np.float32)
    for b, n in enumerate(lens):
        buf[off + b * Lmax:off + b * Lmax + n] = waves[b][:n]
    if Tf_max is None:
        Tf_max = 1 + max(lens) // hop + (32 * extra + 5 if extra else 0)
    nblk = lib.load().espb_frontend_blocks(Tf_max)
    assert nblk == (Tf_max + 31) // 32
    n_out, n_part = B * Tf_max * n_mels, B * nblk * n_mels
    out = torch.full((n_out + 7,), NAN, device="cuda")
    part = torch.full((n_part + 7,), NAN, device="cuda")
    wave = _dev(buf)
    _call("espb_stft_logmel_f32", _ptr(wave[off:]), _ptr(_dev(np.asarray(lens, dtype=np.int64))), B, Lmax, hop, _ptr(c["window"]),
          _ptr(c["tw"]), _ptr(c["twt"]), _ptr(c["start"]), _ptr(c["count"]), _ptr(c["offset"]), _ptr(c["weight"]), c["nnz"], n_mels,
          _ptr(out), Tf_max, _ptr(part))
    torch.cuda.synchronize()
    assert _all_nan_bits(out[n_out:]) and _all_nan_bits(part[n_part:]), "stft_logmel wrote past its outputs"
    return out[:n_out].view(B, Tf_max, n_mels).cpu().numpy(), part[:n_part].view(B, nblk, n_mels).cpu().numpy()


def _check_stft(c, fe, hop, waves, lens, out, part, what):
    """Every utterance against the float64 reference, padded frames +0, partial sums against the kernel's own rows."""
    window, melmat, count = c["window"].cpu().numpy(), fe.logmel.melmat.numpy(), c["count"].cpu().numpy()
    counts = [0, 0, 0]
    for b, n in enumerate(lens):
        Tf = 1 + n // hop
        M, dM = _reference(waves[b], n, hop, window, melmat, count)
        counts = [a + k for a, k in zip(counts, _check_logmel(out[b, :Tf], M, dM, f"{what} b{b} len {n}"))]
        assert not out[b, Tf:].view(np.int32).any(), f"{what} b{b}: padded frames are not +0"
        x = out[b].astype(np.float64)
        for blk in range(part.shape[1]):
            rows = x[32 * blk:min(Tf, 32 * blk + 32)]
            if rows.shape[0] == 0:
                assert not part[b, blk].view(np.int32).any(), f"{what} b{b}: partial of block {blk} (no frame < Tf) is not +0"
                continue
            err = np.abs(part[b, blk] - rows.sum(0))
            assert (err <= 40 * U32 * np.abs(rows).sum(0)).all(), f"{what} b{b} block {blk}: partial sum off by {err.max():.3e}"
    print(f"{what}: elements at the floor / log domain / power domain: {counts}")


def _case(hop, lens, signal=_noise, seed=0, off=1, **kw):
    fe, c = _tables("cuda", hop_length=hop, **kw)
    rng = np.random.default_rng(seed)
    waves = [signal(rng, n) for n in lens]
    out, part = _stft(c, fe.n_mels, hop, waves, lens, off=off)
    _check_stft(c, fe, hop, waves, lens, out, part, f"hop {hop} {kw}")
    return fe, c, waves, out, part


# ============================================================================================================== espb_stft_logmel_f32
SHORT = [257, 258, 384, 511, 512, 513]                                       # 257: the shortest accepted (reflect padding needs > 256)
TF_EDGES = [128 * 62, 128 * 62 + 77, 128 * 63, 128 * 63 + 77, 128 * 64, 128 * 64 + 77]   # Tf = 63, 64, 65; multiples of the hop and not


@gpu
@pytest.mark.parametrize("lens", [SHORT, TF_EDGES], ids=["short", "tf_edges"])
def test_stft_logmel_lengths(lens):
    _case(128, lens, seed=len(lens) + lens[0])


def _hop_lens(hop):
    """Frame counts 32 k - 1, 32 k and 32 k + 1, at a multiple of the hop and not (every length > 256)."""
    base = [hop * 31, hop * 32 + hop // 2 + 1, hop * 30 + 1]
    return [n if n > 256 else 257 + 31 * i for i, n in enumerate(base)]


@gpu
@pytest.mark.parametrize("hop", [1, 75, 100, 128, 160, 256, 400, 512, 640, 1024])
def test_stft_logmel_hops(hop):
    """Odd hops take the scalar frame load; hops above 512 skip samples; 1024 is the largest accepted (about 150 KB of shared memory)."""
    _case(hop, _hop_lens(hop), seed=hop)


@gpu
@pytest.mark.parametrize("win_length", [512, 400, 320, 1])
@pytest.mark.parametrize("window", ["hann", "hamming", None])
def test_stft_logmel_windows(window, win_length):
    _case(160, [16000, 9001, 12345], seed=win_length, window=window, win_length=win_length)


@gpu
@pytest.mark.parametrize("kw", [dict(n_mels=1), dict(n_mels=23), dict(n_mels=80), dict(n_mels=96), dict(n_mels=97), dict(n_mels=128),
                                dict(n_mels=128, fmax=2000), dict(fs=8000, n_mels=80), dict(n_mels=80, fmax=8600)],
                         ids=["1", "23", "80", "96", "97", "128", "128_fmax2000", "fs8000", "80_fmax8600"])
def test_stft_logmel_mel_banks(kw):
    """128 mels up to 2 kHz: filters with no non-zero bin give ln(1e-10f); fmax 8600 Hz puts a non-zero weight on the Nyquist bin."""
    fe, c, *_ = _case(128, [8000, 4097, 6001], seed=kw["n_mels"], **kw)
    if kw.get("fmax") == 2000:
        assert int((c["count"] == 0).sum()) > 0
    if kw.get("fmax") == 8600:
        assert float(fe.logmel.melmat[256].max()) > 0


@gpu
@pytest.mark.parametrize("signal", [_noise, _tone, _dc, _impulse, _silence], ids=lambda f: f.__name__[1:])
@pytest.mark.parametrize("hop", [128, 160])
def test_stft_logmel_signals(signal, hop):
    """Noise at int16 scale, a tone on a bin centre, a DC offset, an impulse, digital silence over whole frames."""
    _case(hop, [16000, 7777, 12001], signal=signal, seed=hop)


@gpu
def test_stft_logmel_90s():
    """90 s at hop 160 (9001 frames) next to a shorter utterance."""
    _case(160, [90 * 16000, 90 * 16000 - 12345], seed=90)


@gpu
@pytest.mark.parametrize("hop", [128, 160, 75])
def test_stft_logmel_batch_independence(hop):
    """A ragged batch of 5 with an odd Lmax, one float past alignment: each utterance's rows and partials are bit for bit those of the
    utterance alone (Lmax = len, aligned, so the interior blocks take the 16-byte loads)."""
    lens = [9001, 257, 4096 + 3, 6400, 8191]
    fe, c, waves, out, part = _case(hop, lens, seed=5, off=1)
    for b, n in enumerate(lens):
        Tf = 1 + n // hop
        o1, p1 = _stft(c, fe.n_mels, hop, [waves[b]], [n], off=0, extra=0)
        assert np.array_equal(o1[0, :Tf].view(np.int32), out[b, :Tf].view(np.int32)), f"b{b}: rows differ alone and in the batch"
        assert np.array_equal(p1[0].view(np.int32), part[b, :p1.shape[1]].view(np.int32)), f"b{b}: partials differ"


@gpu
@pytest.mark.parametrize("bad,match", [(dict(hop=1025), "bad shape"), (dict(hop=0), "bad shape"), (dict(n_mels=129), "bad shape"),
                                       (dict(nnz=4097), "bad shape"), (dict(B=0), "bad shape")])
def test_stft_logmel_refusals(bad, match):
    """Refused before any launch: the outputs stay NaN."""
    fe, c = _tables("cuda", n_mels=128)
    a = dict(hop=128, n_mels=128, nnz=c["nnz"], B=1)
    a.update(bad)
    wave = _dev(np.zeros(4000, dtype=np.float32))
    out = torch.full((2 * 32 * 129,), NAN, device="cuda")
    part = torch.full((2 * 129,), NAN, device="cuda")
    with pytest.raises(RuntimeError, match=match):
        _call("espb_stft_logmel_f32", _ptr(wave), _ptr(_dev(np.array([4000], dtype=np.int64))), a["B"], 4000, a["hop"], _ptr(c["window"]),
              _ptr(c["tw"]), _ptr(c["twt"]), _ptr(c["start"]), _ptr(c["count"]), _ptr(c["offset"]), _ptr(c["weight"]), a["nnz"], a["n_mels"],
              _ptr(out), 32, _ptr(part))
    torch.cuda.synchronize()
    assert _all_nan_bits(out) and _all_nan_bits(part)


# ============================================================================================================== UtteranceMVN
def _mvn_check(got, x, n, nblk, what):
    xd = x[:n].astype(np.float64)
    y = xd - xd.mean(0)
    tol = (40 + nblk + 2) * U32 * np.abs(xd).sum(0) / n + U32 * np.abs(y)
    err = np.abs(got[:n] - y)
    assert (err <= tol).all(), f"{what}: max err {err.max():.3e}, worst err/tol {(err / tol).max():.2f}"


@gpu
@pytest.mark.parametrize("hop,n_mels,lens", [(400, 80, [300, 1000]), (128, 128, TF_EDGES), (160, 80, [160 * 62, 160 * 63 + 7, 160 * 64 + 159]),
                                             (160, 128, [257, 16000])])
def test_utt_mvn_from_partial_vs_fp64(hop, n_mels, lens):
    """After the frontend, from its partial sums: Tf = 1 (hop 400, 300 samples), Tf = 32 k +- 1, n_mels 128, hops other than 128."""
    fe, c = _tables("cuda", hop_length=hop, n_mels=n_mels)
    rng = np.random.default_rng(hop + n_mels)
    waves = [_noise(rng, n) for n in lens]
    out, part = _stft(c, n_mels, hop, waves, lens, off=1)
    B, Tf_max, _ = out.shape
    feats = _dev(out)
    _call("espb_utt_mvn_from_partial_f32", _ptr(feats), _ptr(_dev(np.asarray(lens, dtype=np.int64))), B, Tf_max, n_mels, hop,
          _ptr(_dev(part)))
    torch.cuda.synchronize()
    got = feats.cpu().numpy()
    for b, n in enumerate(lens):
        Tf = 1 + n // hop
        _mvn_check(got[b].astype(np.float64), out[b], Tf, part.shape[1], f"hop {hop} b{b} Tf {Tf}")
        assert not got[b, Tf:].view(np.int32).any(), "padded frames must stay +0"


@gpu
@pytest.mark.parametrize("n_mels", [80, 128])
def test_utt_mvn_standalone_vs_fp64(n_mels):
    """feat_lens 1, 31, 32, 33 and Tf_max; rows >= len are NaN and are neither read nor written (they stay NaN: the reference would make
    them -mean, see the module docstring)."""
    lens, Tf_max = [1, 31, 32, 33, 70], 70
    rng = np.random.default_rng(n_mels)
    x = (3 * rng.standard_normal((len(lens), Tf_max, n_mels)) - 12).astype(np.float32)
    for b, n in enumerate(lens):
        x[b, n:] = np.nan
    feats = _dev(x)
    nblk = (Tf_max + 31) // 32
    ws = torch.full((len(lens) * nblk * n_mels + 5,), NAN, device="cuda")
    _call("espb_utt_mvn_f32", _ptr(feats), _ptr(_dev(np.asarray(lens, dtype=np.int64))), len(lens), Tf_max, n_mels, _ptr(ws))
    torch.cuda.synchronize()
    got = feats.cpu().numpy()
    assert _all_nan_bits(ws[len(lens) * nblk * n_mels:])
    for b, n in enumerate(lens):
        _mvn_check(got[b].astype(np.float64), x[b], n, nblk, f"len {n}")
        assert (got[b, n:].view(np.int32) == NAN_BITS).all(), f"len {n}: rows >= len were written"


@gpu
def test_utt_mvn_refuses_n_mels():
    feats = torch.full((2 * 40 * 129,), NAN, device="cuda")
    lens = _dev(np.array([40, 40], dtype=np.int64))
    ws = torch.zeros(2 * 2 * 129, device="cuda")
    with pytest.raises(RuntimeError, match="n_mels > 128"):
        _call("espb_utt_mvn_f32", _ptr(feats), _ptr(lens), 2, 40, 129, _ptr(ws))
    with pytest.raises(RuntimeError, match="n_mels > 128"):
        _call("espb_utt_mvn_from_partial_f32", _ptr(feats), _ptr(lens), 2, 40, 129, 128, _ptr(ws))
    torch.cuda.synchronize()
    assert _all_nan_bits(feats)


# ============================================================================================================== GlobalMVN
@gpu
@pytest.mark.parametrize("norm_vars", [True, False])
@pytest.mark.parametrize("norm_means", [True, False])
def test_global_mvn_bit_exact(norm_means, norm_vars):
    """D = 83, Tmax * D = 24900 > one grid-stride pass (64 x 256 threads); padded frames (NaN on input) become 0."""
    from oracle import frontend as OF

    B, Tmax, D, lens = 3, 300, 83, [300, 1, 157]
    rng = np.random.default_rng(83)
    x = (4 * rng.standard_normal((B, Tmax, D)) + 2).astype(np.float32)
    mean = torch.from_numpy(rng.standard_normal(D) * 3)
    std = torch.from_numpy(np.exp(rng.standard_normal(D)))
    ref = OF.global_mvn(torch.from_numpy(x), torch.tensor(lens), mean, std, norm_means, norm_vars).numpy()
    for b, n in enumerate(lens):
        x[b, n:] = np.nan
    feats = _dev(x)
    _call("espb_global_mvn_f32", _ptr(feats), _ptr(_dev(np.asarray(lens, dtype=np.int64))), B, Tmax, D, _ptr(_dev(mean.float().numpy())),
          _ptr(_dev(std.float().numpy())), int(norm_means), int(norm_vars))
    torch.cuda.synchronize()
    got = feats.cpu().numpy()
    assert np.array_equal(got.view(np.int32), ref.view(np.int32))
    for b, n in enumerate(lens):
        assert (got[b, n:] == 0).all()


# ============================================================================================================== CPU checks
@pytest.mark.parametrize("kw", [dict(n_mels=1), dict(n_mels=80), dict(n_mels=97), dict(n_mels=128), dict(n_mels=128, fmax=2000),
                                dict(fs=8000, n_mels=80), dict(n_mels=80, fmax=8600)])
def test_sparse_mel_tables_rebuild_melmat(kw):
    """start / count / offset / weight of DefaultFrontend._constants give back melmat bit for bit, and count spans the non-zero bins."""
    fe, c = _tables("cpu", **kw)
    mm = fe.logmel.melmat.numpy()
    rebuilt = np.zeros_like(mm)
    start, count, offset, weight = (c[k].numpy() for k in ("start", "count", "offset", "weight"))
    assert c["nnz"] == int(count.sum()) <= 4096
    for m in range(mm.shape[1]):
        rebuilt[start[m]:start[m] + count[m], m] = weight[offset[m]:offset[m] + count[m]]
        nz = np.nonzero(mm[:, m])[0]
        assert count[m] == (nz[-1] + 1 - nz[0] if nz.size else 0)
    # the Slaney construction leaves some -0 weights (0 * a negative ramp); like every zero they stay out of the sparse form
    assert np.array_equal(rebuilt.view(np.int32), (mm + np.float32(0)).view(np.int32))


def test_tolerances_catch_plausible_bugs():
    """On the CPU, from the float64 reference above: each plausible bug named in the module docstring moves the reference by more than
    10x the tolerance the GPU tests use, at a tested shape (int16-scale noise; hop 128 or 160; 80 mels, fmax 8600 for the Nyquist bin)."""
    rng = np.random.default_rng(0)
    fe, c = _tables("cpu", hop_length=160, win_length=400, n_mels=80, fmax=8600)
    window, melmat, count = c["window"].numpy(), fe.logmel.melmat.numpy(), c["count"].numpy()
    n, hop = 9001, 160
    x = _noise(rng, n)
    M, dM = _reference(x, n, hop, window, melmat, count)
    ok = dM <= 0.5 * M
    assert ok.mean() > 0.99
    tol = _log_tol(M, dM)
    ref = np.log(np.maximum(M, FLOOR))

    def over(Mb):
        return float((np.abs(np.log(np.maximum(Mb, FLOOR)) - ref) / tol)[ok].max())

    assert over(_reference(x, n, hop, window, melmat, count, pad_mode="symmetric")[0]) > 10      # reflect padding repeats the edge sample
    assert over(_reference(x, n, hop, window, melmat, count, late=1)[0]) > 10                    # frames one sample late
    assert over(_reference(x, n, hop, window, melmat, count, drop_nyquist=True)[0]) > 10         # the Nyquist bin dropped
    left = np.zeros(512, dtype=np.float32)
    left[:400] = torch.hann_window(400).numpy()
    assert over(_reference(x, n, hop, left, melmat, count)[0]) > 10                              # a short window left-aligned
    fe2, c2 = _tables("cpu", hop_length=128, n_mels=80)
    w2, mm2, cnt2 = c2["window"].numpy(), fe2.logmel.melmat.numpy(), c2["count"].numpy()
    M, dM = _reference(x, n, 128, w2, mm2, cnt2)
    ok, tol, ref = dM <= 0.5 * M, _log_tol(M, dM), np.log(np.maximum(M, FLOOR))
    sym = torch.hann_window(512, periodic=False).numpy()                                          # the symmetric Hann window
    assert float((np.abs(np.log(np.maximum(_reference(x, n, 128, sym, mm2, cnt2)[0], FLOOR)) - ref) / tol)[ok].max()) > 10
    # MVN over Tf_max instead of Tf, at the standalone test's shape (len 33 of Tf_max 70, log-mel-like values)
    feats = (3 * rng.standard_normal((33, 80)) - 12).astype(np.float64)
    y = feats - feats.mean(0)
    tol = (40 + 3 + 2) * U32 * np.abs(feats).sum(0) / 33 + U32 * np.abs(y)
    assert float((np.abs(feats - feats.sum(0) / 70 - y) / tol).max()) > 10
