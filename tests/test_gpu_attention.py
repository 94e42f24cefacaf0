"""-m gpu: the fused wgmma self-attention kernel (csrc/attention.cu, espb_flash_attn_f32) against an fp64 restatement of
RelPositionMultiHeadedAttention / MultiHeadedAttention (attention.py:416-459, 391-414, 121-151) on seeded inputs: single and multiple key
tiles, ragged batches (masked keys, query blocks that are all padding, a 1-frame utterance), T = 937 (the benchmarked length), with and
without the rel-pos term.  Tolerance: 2e-5 absolute on O(1) context vectors (3xTF32 products, fp32 accumulation)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

CASES = [(1, 1, 37, [37]), (2, 2, 100, [100, 64]), (2, 2, 300, [300, 129]), (3, 2, 520, [520, 256, 1]), (1, 8, 937, [937]), (2, 3, 700, [699, 513])]


def _inputs(B, H, T, seed):
    from espnet_b200 import ops
    from espnet_b200.lib import call, ptr

    D, dk = H * 64, 64
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B * T, D, generator=g)
    kv = torch.randn(B * T, 3 * D, generator=g)
    Tp, Rp = (T + 31) // 32 * 32, (2 * T - 1 + 31) // 32 * 32
    bd = 2.0 * torch.randn(B, H, T, Rp, generator=g)
    return D, dk, Tp, Rp, q.cuda(), kv.cuda(), bd.cuda()


def _reference(q, kv, bd, lens, B, H, T, D):
    dk = 64
    qd = q.double().view(B, T, H, dk).permute(0, 2, 1, 3)
    kd = kv[:, D:2 * D].double().view(B, T, H, dk).permute(0, 2, 1, 3)
    vd = kv[:, 2 * D:].double().view(B, T, H, dk).permute(0, 2, 1, 3)
    s = qd @ kd.transpose(-1, -2)
    if bd is not None:
        i = torch.arange(T, device=q.device).view(T, 1)
        j = torch.arange(T, device=q.device).view(1, T)
        s = s + torch.gather(bd.double()[..., : 2 * T - 1], 3, (T - 1 - i + j).expand(B, H, T, T))
    s = s / math.sqrt(dk)
    mask = torch.arange(T, device=q.device).view(1, 1, 1, T) >= torch.tensor(lens, device=q.device).view(B, 1, 1, 1)
    p = torch.softmax(s.masked_fill(mask, float("-inf")), dim=-1).masked_fill(mask, 0.0)
    return (p @ vd).permute(0, 2, 1, 3).reshape(B * T, D)


@pytest.mark.parametrize("relpos", [True, False])
@pytest.mark.parametrize("B,H,T,lens", CASES)
def test_flash_attention_vs_fp64(B, H, T, lens, relpos):
    from espnet_b200 import ops
    from espnet_b200.lib import call, ptr

    D, dk, Tp, Rp, q, kv, bd = _inputs(B, H, T, seed=B * 1000 + T)
    M = B * T
    lens32 = torch.tensor(lens, dtype=torch.int32, device="cuda")
    q_split, kv_split = ops.split_from(q), ops.split_from(kv)
    vt = torch.empty(2, B, H, dk, Tp, device="cuda")
    call("espb_v_transpose_f32", ptr(kv_split), M * 3 * D, B, T, D, H, ptr(lens32), ptr(vt), B * H * dk * Tp, Tp)
    out = torch.full((2, M, D), float("nan"), device="cuda")
    ops.flash_attn(q_split, 0, D, kv_split, D, 3 * D, vt, Tp, bd if relpos else None, Rp, lens32, B, H, T, dk, out)
    torch.cuda.synchronize()
    got = (out[0].double() + out[1].double()).view(B, T, D)
    ref = _reference(q, kv, bd if relpos else None, lens, B, H, T, D).view(B, T, D)
    assert bool(torch.isfinite(out).all()), "padding rows must hold finite values"
    for b, n in enumerate(lens):
        e = (got[b, :n] - ref[b, :n]).abs().max().item()
        print(f"B{B} H{H} T{T} len{n} relpos={relpos}: max abs err {e:.3e}")
        assert e < 2e-5
    # hi plane is a tf32 value, lo plane the exact remainder of the fp32 result
    assert int((out[0].view(torch.int32) & 0x1FFF).abs().max()) == 0
