"""BranchformerEncoder with the reference's constructor / state_dict surface, executed by the espnet_b200 CUDA kernels.

Reference: espnet2/asr/encoder/branchformer_encoder.py:49-293 (BranchformerEncoderLayer), 296-576 (BranchformerEncoder) and
espnet2/asr/layers/cgmlp.py:15-124.  A layer runs an attention branch -- the Conformer's rel-pos "latest" self-attention of layers.py -- and
a cgMLP branch -- the E-Branchformer's, shared in layers.py -- on the same input, merges them, adds the result to the residual and applies
norm_final.  The merge methods:

  concat       linear_out and channel_proj2 write the split (tf32 hi/lo) operand of merge_proj directly, into columns [0, D) and [D, 2D) of
               one [2][M][2D] buffer -- the torch.cat of the reference; merge_proj adds the residual in its epilogue.
  learned_ave  both branches write plain fp32 into one [M, 2D] buffer; espb_branch_pool_f32 computes each utterance's two merge weights on
               the device (attention pooling over its own frames, then a 2-way softmax), espb_branch_merge_f32 writes w1*x1 + w2*x2 as the
               split operand of merge_proj (Linear(D, D)).
  fixed_ave    the same merge kernel with the constant weights 1 - cgmlp_weight and cgmlp_weight.

A layer with one branch (use_attn / use_cgmlp False, or fixed_ave with cgmlp_weight 0 or 1) computes x + merge_proj(branch); with the
Identity merge_proj the branch's last GEMM adds the residual itself.  The torch.nn layers are parameter containers only (reference
checkpoints load by name); forward never calls them.
"""
import math
from typing import List, Optional, Tuple, Union

import torch

from . import ops
from .layers import LN_EPS, EncoderBase, _CgMLP, _PosBias
from .ops import _count, layernorm, linear

MERGE_METHODS = ("concat", "learned_ave", "fixed_ave")


class _Layer(torch.nn.Module):
    def __init__(self, d, heads, use_attn, use_cgmlp, cgmlp_units, cgmlp_kernel, merge_method, cgmlp_weight):
        super().__init__()
        assert use_attn or use_cgmlp, "At least one branch should be valid"
        # both branches are built before a fixed_ave layer drops one, as in the reference: a seeded default init draws the same weights
        self.attn = _PosBias(heads, d) if use_attn else None
        self.cgmlp = _CgMLP(d, cgmlp_units, cgmlp_kernel) if use_cgmlp else None
        if use_attn:
            self.norm_mha = torch.nn.LayerNorm(d, eps=LN_EPS)
        if use_cgmlp:
            self.norm_mlp = torch.nn.LayerNorm(d, eps=LN_EPS)
        self.norm_final = torch.nn.LayerNorm(d, eps=LN_EPS)
        self.merge_method, self.cgmlp_weight = merge_method, float(cgmlp_weight)
        self.use_two_branches = use_attn and use_cgmlp
        if not self.use_two_branches:
            self.merge_proj = torch.nn.Identity()
        elif merge_method == "concat":
            self.merge_proj = torch.nn.Linear(2 * d, d)
        elif merge_method == "learned_ave":
            self.pooling_proj1 = torch.nn.Linear(d, 1)
            self.pooling_proj2 = torch.nn.Linear(d, 1)
            self.weight_proj1 = torch.nn.Linear(d, 1)
            self.weight_proj2 = torch.nn.Linear(d, 1)
            self.merge_proj = torch.nn.Linear(d, d)
        elif merge_method == "fixed_ave":
            assert 0.0 <= self.cgmlp_weight <= 1.0, "cgmlp weight should be between 0.0 and 1.0"
            if self.cgmlp_weight == 0.0:
                self.use_two_branches, self.cgmlp, self.norm_mlp = False, None, None
            elif self.cgmlp_weight == 1.0:
                self.use_two_branches, self.attn, self.norm_mha = False, None, None
            self.merge_proj = torch.nn.Linear(d, d)
        else:
            raise ValueError(f"unknown merge method: {merge_method}")


def _per_layer(name, v, n):
    v = [float(v)] * n if isinstance(v, (int, float)) else list(v)
    if len(v) != n:
        raise ValueError(f"Length of {name} ({len(v)}) should be equal to num_blocks ({n})")
    return v


class BranchformerEncoder(EncoderBase):
    """Drop-in for espnet2.asr.encoder.branchformer_encoder.BranchformerEncoder (inference, CUDA only)."""

    def __init__(self, input_size: int, output_size: int = 256, use_attn: bool = True, attention_heads: int = 4,
                 attention_layer_type: str = "rel_selfattn", pos_enc_layer_type: str = "rel_pos", rel_pos_type: str = "latest",
                 use_cgmlp: bool = True, cgmlp_linear_units: int = 2048, cgmlp_conv_kernel: int = 31, use_linear_after_conv: bool = False,
                 gate_activation: str = "identity", merge_method: str = "concat", cgmlp_weight: Union[float, List[float]] = 0.5,
                 attn_branch_drop_rate: Union[float, List[float]] = 0.0, num_blocks: int = 12, dropout_rate: float = 0.1,
                 positional_dropout_rate: float = 0.1, attention_dropout_rate: float = 0.0, input_layer: Optional[str] = "conv2d",
                 zero_triu: bool = False, padding_idx: int = -1, stochastic_depth_rate: Union[float, List[float]] = 0.0,
                 qk_norm: bool = False, use_flash_attn: bool = True):
        unsupported = []
        if input_layer != "conv2d": unsupported.append(f"input_layer={input_layer}")
        if rel_pos_type != "latest" or pos_enc_layer_type != "rel_pos" or attention_layer_type != "rel_selfattn":
            unsupported.append("rel_pos_type/pos_enc_layer_type/attention_layer_type other than latest/rel_pos/rel_selfattn")
        if use_linear_after_conv or gate_activation != "identity": unsupported.append("use_linear_after_conv / non-identity gate_activation")
        if cgmlp_conv_kernel < 1 or cgmlp_conv_kernel % 2 == 0 or cgmlp_conv_kernel > 127:
            unsupported.append(f"cgmlp_conv_kernel={cgmlp_conv_kernel} (odd, <= 127)")
        if cgmlp_linear_units % 2 or cgmlp_linear_units // 2 > 2048: unsupported.append(f"cgmlp_linear_units={cgmlp_linear_units} (even, <= 4096)")
        if zero_triu or qk_norm: unsupported.append("zero_triu/qk_norm")
        if unsupported:
            raise NotImplementedError("espnet_b200 BranchformerEncoder does not support: " + ", ".join(unsupported))
        if output_size % 32:
            raise NotImplementedError("espnet_b200 BranchformerEncoder: output_size must be a multiple of 32")
        assert output_size % attention_heads == 0
        _per_layer("stochastic_depth_rate", stochastic_depth_rate, num_blocks)   # training only; checked as the reference does
        cgmlp_weight = _per_layer("cgmlp_weight", cgmlp_weight, num_blocks)
        _per_layer("attn_branch_drop_rate", attn_branch_drop_rate, num_blocks)
        super().__init__(input_size, output_size, (
            _Layer(output_size, attention_heads, use_attn, use_cgmlp, cgmlp_linear_units, cgmlp_conv_kernel, merge_method, cgmlp_weight[i])
            for i in range(num_blocks)))
        self.heads, self.num_blocks = attention_heads, num_blocks
        self.cgmlp_units, self.cgmlp_kernel = cgmlp_linear_units, cgmlp_conv_kernel

    def _pack(self):
        pk = self._pack_io()
        f32, ln = self._f32, self._pack_ln
        layers, attns = [], []
        for lyr in self.encoders:
            d = dict(norm_final=ln(lyr.norm_final))
            if lyr.attn is not None:
                d["norm_mha"], d["ai"] = ln(lyr.norm_mha), len(attns)   # ai: row block of this layer's linear_pos in pos_w_all
                d.update(self._pack_mha(lyr.attn))
                attns.append(lyr.attn)
            if lyr.cgmlp is not None:
                d["norm_mlp"] = ln(lyr.norm_mlp)
                d.update(self._pack_cgmlp(lyr.cgmlp))
            if lyr.use_two_branches:
                d["merge"] = lyr.merge_method
                if lyr.merge_method == "learned_ave":
                    d["pool_w"] = torch.cat([f32(lyr.pooling_proj1.weight), f32(lyr.pooling_proj2.weight)], 0).contiguous()
                    d["pool_b"] = torch.cat([f32(lyr.pooling_proj1.bias), f32(lyr.pooling_proj2.bias)], 0).contiguous()
                    d["wt_w"] = torch.cat([f32(lyr.weight_proj1.weight), f32(lyr.weight_proj2.weight)], 0).contiguous()
                    d["wt_b"] = torch.cat([f32(lyr.weight_proj1.bias), f32(lyr.weight_proj2.bias)], 0).contiguous()
                elif lyr.merge_method == "fixed_ave":
                    # (1.0 - w) * x1 + w * x2 with Python floats: each weight is rounded once to fp32 when it meets the fp32 tensor
                    d["fixed"] = (1.0 - lyr.cgmlp_weight, lyr.cgmlp_weight)
            if isinstance(lyr.merge_proj, torch.nn.Linear):
                d["mp_w"], d["mp_b"] = ops.split_from(f32(lyr.merge_proj.weight)), f32(lyr.merge_proj.bias)
            layers.append(d)
        pk["layers"] = layers
        pk["pos_w_all"] = self._pack_pos(attns) if attns else None
        self._packed = pk
        return pk

    # ---------------------------------------------------------------- forward
    @torch.no_grad()
    def forward(self, xs_pad: torch.Tensor, ilens: torch.Tensor, prev_states: torch.Tensor = None
                ) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor]]:
        """xs_pad (B, T_f, idim) float32 CUDA (normalised log-mel), ilens (B,) -> (B, T, D), olens, None.

        Ragged batches follow per-utterance (batch-1) semantics of the reference: every utterance sees only its own frames (own attention
        keys, own conv boundaries in the CSGU, own frames in the learned_ave pooling); rows t >= olens[b] of the output are 0."""
        pk = self._packed or self._pack()
        xs_pad, T, olens, lens32 = self._lengths(xs_pad, ilens)   # check_short_utt: branchformer_encoder.py:550-564
        B, D = xs_pad.shape[0], self._output_size
        M = B * T
        x = self._buf("x", (M, D))
        self._subsample(xs_pad, x, math.sqrt(D))
        if self.trace is not None:
            self.trace.append(x.view(B, T, D).clone())
        p_all = self._pos(T) if pk["pos_w_all"] is not None else None

        xn, qkv, ctx = self._buf("xn", (2, M, D)), self._buf("qkv", (2, M, 3 * D)), self._buf("ctx", (2, M, D))
        for w in pk["layers"]:
            merge, two = w.get("merge"), "merge" in w
            if merge == "concat":
                dst = self._buf("mcat", (2, M, 2 * D))   # [x_att | x_cgmlp] split: merge_proj's operand
                ld, split = 2 * D, True
            elif two:
                dst = self._buf("cat", (M, 2 * D))       # [x_att | x_cgmlp] plain: read by the pool / merge kernels
                ld, split = 2 * D, False
            elif "mp_w" in w:
                dst = self._buf("xb", (2, M, D))         # the one branch, split: merge_proj's operand
                ld, split = D, True
            else:
                dst, ld, split = x, D, False             # Identity merge_proj: the branch adds itself to x
            res = x if dst is x else None
            # branch 1: rel-pos MHSA (branchformer_encoder.py:181-192, attention.py:416-459) -> dst[:, :D]
            if "norm_mha" in w:
                layernorm(x, *w["norm_mha"], LN_EPS, out_split=xn)
                linear(xn, w["qkv_w"], qkv, bias=w["qkv_b"], split_out=True)
                self._relpos_attn(qkv, w, w["ai"], p_all, ctx, B, T, lens32)
                ops.gemm(M, D, D, ctx, M * D, D, w["out_w"], D * D, D, dst, ld, c_plane=M * ld if split else 0, split_out=split,
                         bias=w["out_b"], R=res, ldr=D if res is not None else 0)
            # branch 2: cgMLP (branchformer_encoder.py:195-204, cgmlp.py:110-124) -> dst[:, D:] (dst[:, :D] with one branch)
            if "norm_mlp" in w:
                self._cgmlp(x, xn, w, B, T, lens32, dst, ld, c_off=D if two else 0, split_out=split, residual=res)
            # merge (branchformer_encoder.py:207-286): x += merge_proj(...)
            if merge in ("learned_ave", "fixed_ave"):
                mw = None
                if merge == "learned_ave":
                    mw = self._buf("merge_w", (B, 2))
                    part = self._buf("pool_part", (B * 2 * ((T + 31) // 32) * (D + 2),))
                    ops.call("espb_branch_pool_f32", ops.ptr(dst), ops.ptr(dst[:, D:]), 2 * D, B, T, D, ops.ptr(lens32), ops.ptr(w["pool_w"]),
                             ops.ptr(w["pool_b"]), ops.ptr(w["wt_w"]), ops.ptr(w["wt_b"]), ops.ptr(part), ops.ptr(mw))
                    _count(2)
                w1, w2 = w.get("fixed", (0.0, 0.0))
                xb = self._buf("xb", (2, M, D))
                ops.call("espb_branch_merge_f32", ops.ptr(dst), ops.ptr(dst[:, D:]), 2 * D, M, D, T, ops.ptr(mw), w1, w2, ops.ptr(xb), M * D)
                _count()
                dst = xb
            if "mp_w" in w:
                linear(dst, w["mp_w"], x, bias=w["mp_b"], residual=x)
            layernorm(x, *w["norm_final"], LN_EPS, out_plain=x)
            if self.trace is not None:
                self.trace.append(x.view(B, T, D).clone())
        out, out_split = self._output(x, B, T)
        ops.call("espb_zero_pad_rows_f32", ops.ptr(out), B, T, D, ops.ptr(lens32), 0, 1)
        ops.call("espb_zero_pad_rows_f32", ops.ptr(out_split), B, T, D, ops.ptr(lens32), M * D, 2)
        _count(2)
        return out, olens, None
