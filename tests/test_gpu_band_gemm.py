"""The rel-pos band kernel (EspbGemmDesc::band_t > 0) against the generic wgmma GEMM of the same operands: every in-band element
C[i][n], band_t-1-i <= n <= 2*band_t-2-i, n < N, must be bit-identical (same MMA sequence per element)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _split(x):
    from espnet_b200 import ops

    return ops.split_from(x)


def _compare(mode, K, M, N, band_t, Bn, H, Rp, seed):
    """(utterance, head) slices as in the encoder: A rows [Bn*M][H*K] (head h at columns h*K), B [N][L*H*K] shared across utterances
    (layer 1 of L = 2), C [Bn][H][M][Rp]."""
    from espnet_b200 import ops

    torch.manual_seed(seed)
    L, D = 2, H * K
    a = _split(torch.randn(Bn * M, D, device="cuda"))
    b = _split(torch.randn(N, L * D, device="cuda"))

    def run(bt):
        c = torch.full((Bn, H, M, Rp), float("nan"), device="cuda")
        used_tc = ops.gemm(M, N, K, a, Bn * M * D, D, b, N * L * D, L * D, c, Rp, nbx=H, nby=Bn, sa=(K, M * D), sb=(K, 0),
                           sc=(M * Rp, H * M * Rp), b_off=D, band_t=bt, force=mode)
        assert used_tc
        torch.cuda.synchronize()
        return c

    ref, got = run(0), run(band_t)
    i = torch.arange(M, device="cuda")[:, None]
    n = torch.arange(Rp, device="cuda")[None, :]
    band = (n >= band_t - 1 - i) & (n <= 2 * band_t - 2 - i) & (n < N)
    assert band.any()
    r, g = ref[:, :, band], got[:, :, band]
    assert torch.isfinite(r).all()
    mismatch = (r.view(torch.int32) != g.view(torch.int32)).sum().item()
    assert mismatch == 0, f"{mismatch} of {r.numel()} in-band elements differ (max abs diff {(r - g).abs().max().item():.3e})"


@pytest.mark.parametrize("mode", ["tc", "tc2"])
@pytest.mark.parametrize("K", [16, 32, 64, 128])
@pytest.mark.parametrize("T", [50, 128, 300])
@pytest.mark.parametrize("pitch", ["aligned", "odd"])
def test_band_kernel_bit_identical(mode, K, T, pitch):
    R = 2 * T - 1
    Rp = (R + 31) // 32 * 32 if pitch == "aligned" else R + 2   # odd pitch: the band kernel stores scalars
    _compare(mode, K, T, R, T, 2, 3, Rp, seed=T * 131 + K)


@pytest.mark.parametrize("mode", ["tc", "tc2"])
@pytest.mark.parametrize("K", [64, 96, 128])
def test_band_kernel_more_units_than_sms(mode, K):
    """64 (utterance, head) slices x 3 row blocks = 192 units: CTAs take several units each, so the A buffers are reused across units
    (two buffers at K = 64, one at K = 96 and 128; 128-column tiles up to K = 96, 64-column tiles at K = 128)."""
    T = 300
    R = 2 * T - 1
    _compare(mode, K, T, R, T, 8, 8, (R + 31) // 32 * 32, seed=K)


@pytest.mark.parametrize("mode", ["tc", "tc2"])
@pytest.mark.parametrize("K", [64, 128])
@pytest.mark.parametrize("shape", ["rows_past_band", "few_columns"])
def test_band_kernel_skips_empty_units(mode, K, shape):
    """Descriptors whose row blocks partly have no in-band column, interleaved with blocks that have some, over 64 slices (more units
    than SMs): a CTA skips units between the ones it computes."""
    if shape == "rows_past_band":   # band_t 100, M 512: row blocks 2 and 3 (rows >= 2*band_t-1) reach no column
        M, N, band_t = 512, 199, 100
    else:                            # band_t 300, N 100 < band_t - 128: row block 0 reaches no column < N
        M, N, band_t = 300, 100, 300
    _compare(mode, K, M, N, band_t, 8, 8, (N + 31) // 32 * 32, seed=M + N + K)


def test_band_fallback_beyond_k128():
    """K > 128 is not served by the band kernel: the generic kernel computes the whole product, so the band is still right."""
    _compare("tc2", 160, 130, 259, 130, 2, 2, 288, seed=7)
