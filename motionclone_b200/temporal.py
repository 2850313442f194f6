"""Motion module (AnimateDiff temporal transformer) on this package's CUDA kernels.

Mirrors the reference interface of motionclone/models/motion_module.py — VanillaTemporalModule (:51),
TemporalTransformer3DModel (:88), TemporalTransformerBlock (:164), PositionalEncoding (:228), VersatileAttention (:250)
— with identical constructor arguments, attribute names and state-dict keys, so AnimateDiff motion-module checkpoints
load unchanged. What differs is underneath:

* activations stay token-major `[(b f), h*w, C]` (== NHWC); the reference's `(b f) d c <-> (b d) f c` rearranges
  (:279, :343) and head splits (attention.py:367-379) are expressed as strides of the kernel's [B, F, P, C] view and
  never materialised;
* to_q/to_k/to_v run as one GEMM over a cached concatenated weight; q, k, v are column slices of its output;
* softmax(QK^T)V, the probabilities, top-1 and gathered probabilities come from ONE fused kernel
  (csrc/temporal_attn.cu) instead of baddbmm/softmax/bmm + a second softmax pass + topk/gather.
"""
from __future__ import annotations

import math
from typing import Optional

import torch
import torch.nn.functional as F
from torch import nn

from . import ops
from .spatial import (CrossAttention, FeedForward, GroupNormNHWC, LayerNorm, fold_residual_biases,
                      linear_into_residual)


def zero_module(module: nn.Module) -> nn.Module:
    for p in module.parameters():
        p.detach().zero_()
    return module


class MotionRecordProcessor:
    """Processor protocol of the reference (utils/xformer_attention.py:17-42): `record_qkv(attn, hidden_states, query,
    key, value, attention_mask)` is called by VersatileAttention.forward before the attention core and keeps q, k.

    Extension used by the fused path: `mode` tells the kernel which per-row by-products to emit from the same tile
      None      - attention output only (q, k are still recorded)
      "probs"   - full probabilities [b*d, heads, f, f]            (get_temp_attn_prob, motionclone_functions.py:260)
      "top1"    - top-1 value / uint8 index per row                 (motionclone_functions.py:79)
      "gather"  - probabilities gathered at `ref_idx`               (motionclone_functions.py:91-92)
    Results land in .probs / .top1 / .gathered (graph-carrying when autograd is on).
    """

    def __init__(self, attention_op=None):
        self.attention_op = attention_op
        self.mode: Optional[str] = None
        self.ref_idx: Optional[torch.Tensor] = None
        self.clear()

    def clear(self):
        self._q = self._k = None  # [b, f, d, C] views (kernel layout)
        self.probs = self.top1 = self.gathered = None
        self.heads = self.scale = None

    def record_qkv(self, attn, hidden_states, query, key, value, attention_mask):
        self._q, self._k = query, key
        self.heads, self.scale = attn.heads, attn.scale

    __call__ = record_qkv

    def record_attn_mask(self, attn, hidden_states, query, key, value, attention_mask):
        self.attn = attn
        self.attention_mask = attention_mask

    # the reference's readers expect `[(b d), f, C]` (motionclone_functions.py:267, :275): materialise lazily
    @staticmethod
    def _bd_f_c(t):
        if t is None:
            return None
        b, f, d, c = t.shape
        return t.permute(0, 2, 1, 3).reshape(b * d, f, c)

    @property
    def query(self):
        return self._bd_f_c(self._q)

    @property
    def key(self):
        return self._bd_f_c(self._k)


class PositionalEncoding(nn.Module):
    """motion_module.py:228-247 (sinusoidal, built in fp32, non-persistent buffer `pe` [1, max_len, d_model])."""

    def __init__(self, d_model, dropout=0.0, max_len=24):
        super().__init__()
        self.dropout = nn.Dropout(p=dropout)
        pos = torch.arange(max_len).unsqueeze(1)
        freq = torch.exp(torch.arange(0, d_model, 2) * (-math.log(10000.0) / d_model))
        pe = torch.zeros(1, max_len, d_model)
        pe[0, :, 0::2] = torch.sin(pos * freq)
        pe[0, :, 1::2] = torch.cos(pos * freq)
        self.register_buffer("pe", pe, persistent=False)

    def forward(self, x):  # x: [(b d), f, c] — reference calling convention
        return self.dropout(x + self.pe[:, : x.size(1)])


class VersatileAttention(CrossAttention):
    """Temporal self-attention over the frame axis (motion_module.py:250-345)."""

    def __init__(self, attention_mode=None, cross_frame_attention_mode=None, temporal_position_encoding=False,
                 temporal_position_encoding_max_len=24, *args, **kwargs):
        super().__init__(*args, **kwargs)
        assert attention_mode == "Temporal"
        self.attention_mode = attention_mode
        self.is_cross_attention = kwargs["cross_attention_dim"] is not None
        self.pos_encoder = PositionalEncoding(kwargs["query_dim"], dropout=0.0,
                                              max_len=temporal_position_encoding_max_len) \
            if (temporal_position_encoding and attention_mode == "Temporal") else None

    def extra_repr(self):
        return f"(Module Info) Attention_Mode: {self.attention_mode}, Is_Cross_Attention: {self.is_cross_attention}"

    def forward(self, hidden_states, encoder_hidden_states=None, attention_mask=None, video_length=None,
                pe_applied: bool = False, residual=None):
        if self.attention_mode != "Temporal" or encoder_hidden_states is not None or self.added_kv_proj_dim is not None:
            raise NotImplementedError  # as motion_module.py:286, :298 (cross-frame text attention is never configured)
        if attention_mask is not None or self.group_norm is not None:
            raise NotImplementedError("attention_mask / group_norm are dead in every shipped config (SURVEY appendix)")
        bf, d, c = hidden_states.shape
        f = int(video_length)
        b = bf // f
        x = hidden_states.view(b, f, d, c)
        if self.pos_encoder is not None and not pe_applied:  # :281-282 — PE indexed by the frame axis
            x = x + self.pos_encoder.pe[0, :f].to(x.dtype).view(1, f, 1, c)
        qkv = F.linear(x, self.fused_qkv_weight())  # to_q / to_k / to_v (bias-free, :293-302) as one GEMM
        q, k, v = qkv[..., :c], qkv[..., c:2 * c], qkv[..., 2 * c:]

        proc = self.processor
        mode = None
        if proc is not None:
            proc.record_qkv(self, x, q, k, v, attention_mask)  # :305-306
            mode = proc.mode
        gather_idx = proc.ref_idx if mode == "gather" else None
        if torch.is_grad_enabled() and qkv.requires_grad:
            o, probs, gathered = ops.TemporalAttention.apply(qkv, self.heads, self.scale, mode == "probs", gather_idx)
            top1 = None
            if mode == "top1":
                top1 = ops.top1_rows(ops.TemporalProbs.apply(q, k, self.heads, self.scale).detach())
        else:
            o, probs, top1, gathered = ops.temporal_attention_forward(
                q, k, v, self.heads, self.scale, want_probs=(mode == "probs"), want_top1=(mode == "top1"),
                gather_idx=gather_idx)
        if proc is not None:
            proc.probs = probs if mode == "probs" else None
            proc.top1 = top1
            proc.gathered = gathered if mode == "gather" else None

        if residual is not None:  # residual + to_out(o) without its bias, as one GEMM (spatial.fold_residual_biases)
            return linear_into_residual(o.view(bf, d, c), self.to_out[0], residual)
        o = self.to_out[1](self.to_out[0](o))  # :337-340
        return o.view(bf, d, c)


class TemporalTransformerBlock(nn.Module):
    """motion_module.py:164-225."""

    def __init__(self, dim, num_attention_heads, attention_head_dim, attention_block_types=("Temporal_Self", "Temporal_Self"),
                 dropout=0.0, norm_num_groups=32, cross_attention_dim=768, activation_fn="geglu", attention_bias=False,
                 upcast_attention=False, cross_frame_attention_mode=None, temporal_position_encoding=False,
                 temporal_position_encoding_max_len=24):
        super().__init__()
        blocks, norms = [], []
        for block_name in attention_block_types:
            blocks.append(VersatileAttention(
                attention_mode=block_name.split("_")[0],
                cross_attention_dim=cross_attention_dim if block_name.endswith("_Cross") else None,
                query_dim=dim, heads=num_attention_heads, dim_head=attention_head_dim, dropout=dropout,
                bias=attention_bias, upcast_attention=upcast_attention,
                cross_frame_attention_mode=cross_frame_attention_mode,
                temporal_position_encoding=temporal_position_encoding,
                temporal_position_encoding_max_len=temporal_position_encoding_max_len))
            norms.append(LayerNorm(dim))
        self.attention_blocks = nn.ModuleList(blocks)
        self.norms = nn.ModuleList(norms)
        self.ff = FeedForward(dim, dropout=dropout, activation_fn=activation_fn)
        self.ff_norm = LayerNorm(dim)

    def residual_biases(self):
        """Output biases of the residual branches in order (motion_module.py:213-225)."""
        return [a.to_out[0].bias for a in self.attention_blocks] + [self.ff.net[2].bias]

    def forward(self, hidden_states, encoder_hidden_states=None, attention_mask=None, video_length=None, folded=None):
        """`folded`: pre-bias list of spatial.fold_residual_biases (the stream arrives shifted by the block's output biases
        and every residual add is the beta = 1 epilogue of its GEMM); the TRUE block output is returned."""
        d = hidden_states.shape[1]
        for i, (attn, norm) in enumerate(zip(self.attention_blocks, self.norms)):
            # LayerNorm (:215) and the positional-encoding add (:281-282) in one pass over the tokens
            pe = attn.pos_encoder.pe[0, :video_length].to(hidden_states.dtype) if attn.pos_encoder is not None else None
            ctx = encoder_hidden_states if attn.is_cross_attention else None
            if folded is not None:
                hidden_states = attn(norm(hidden_states, post_add=pe, rows_per_frame=d, pre_bias=folded[i]),
                                     encoder_hidden_states=ctx, video_length=video_length, pe_applied=True,
                                     residual=hidden_states)
            else:
                hidden_states = attn(norm(hidden_states, post_add=pe, rows_per_frame=d), encoder_hidden_states=ctx,
                                     video_length=video_length, pe_applied=True) + hidden_states
        if folded is not None:
            return self.ff(self.ff_norm(hidden_states, pre_bias=folded[-1]), residual=hidden_states)
        return self.ff(self.ff_norm(hidden_states)) + hidden_states


class TemporalTransformer3DModel(nn.Module):
    """motion_module.py:88-161. Accepts the reference's 5-D `[b, c, f, h, w]` or this package's internal frame-major
    NHWC 4-D `[(b f), c, h, w]` (channels_last) together with `video_length`."""

    def __init__(self, in_channels, num_attention_heads, attention_head_dim, num_layers,
                 attention_block_types=("Temporal_Self", "Temporal_Self"), dropout=0.0, norm_num_groups=32,
                 cross_attention_dim=768, activation_fn="geglu", attention_bias=False, upcast_attention=False,
                 cross_frame_attention_mode=None, temporal_position_encoding=False,
                 temporal_position_encoding_max_len=24):
        super().__init__()
        inner_dim = num_attention_heads * attention_head_dim
        self.norm = GroupNormNHWC(num_groups=norm_num_groups, num_channels=in_channels, eps=1e-6, affine=True)
        self.proj_in = nn.Linear(in_channels, inner_dim)
        self.transformer_blocks = nn.ModuleList([
            TemporalTransformerBlock(dim=inner_dim, num_attention_heads=num_attention_heads,
                                     attention_head_dim=attention_head_dim, attention_block_types=attention_block_types,
                                     dropout=dropout, norm_num_groups=norm_num_groups,
                                     cross_attention_dim=cross_attention_dim, activation_fn=activation_fn,
                                     attention_bias=attention_bias, upcast_attention=upcast_attention,
                                     cross_frame_attention_mode=cross_frame_attention_mode,
                                     temporal_position_encoding=temporal_position_encoding,
                                     temporal_position_encoding_max_len=temporal_position_encoding_max_len)
            for _ in range(num_layers)])
        self.proj_out = nn.Linear(inner_dim, in_channels)

    def _folded(self):
        bs = [self.proj_in.bias] + [b for b in self.transformer_blocks[0].residual_biases() if b is not None]
        key = tuple((b.data_ptr(), b._version, b.dtype, b.device) for b in bs)
        if getattr(self, "_fold_cache", None) is None or self._fold_cache[0] != key:
            with torch.no_grad():
                shift, pre = fold_residual_biases([b.detach() for b in self.transformer_blocks[0].residual_biases()])
                self._fold_cache = (key, ((self.proj_in.bias.detach() + shift).contiguous(), pre))
        return self._fold_cache[1]

    def forward(self, hidden_states, encoder_hidden_states=None, attention_mask=None, video_length=None):
        five_d = hidden_states.dim() == 5
        if five_d:
            b, c, f, h, w = hidden_states.shape
            video_length = f
            hidden_states = hidden_states.permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w)
        assert hidden_states.dim() == 4 and video_length is not None
        n, c, h, w = hidden_states.shape
        residual = hidden_states.permute(0, 2, 3, 1).reshape(n, h * w, c)  # token view (zero-copy when channels_last)
        t = self.norm(hidden_states)
        t = t.permute(0, 2, 3, 1).reshape(n, h * w, c)  # a view when the activation is channels_last
        if len(self.transformer_blocks) == 1 and self.proj_in.bias is not None:
            shift, pre = self._folded()
            t = F.linear(t, self.proj_in.weight, shift)
            t = self.transformer_blocks[0](t, encoder_hidden_states=encoder_hidden_states, video_length=video_length,
                                           folded=pre)
        else:
            t = self.proj_in(t)
            for block in self.transformer_blocks:
                t = block(t, encoder_hidden_states=encoder_hidden_states, video_length=video_length)
        t = self.proj_out(t) + residual
        out = t.reshape(n, h, w, c).permute(0, 3, 1, 2)
        if five_d:
            out = out.reshape(b, f, c, h, w).permute(0, 2, 1, 3, 4)
        return out


class VanillaTemporalModule(nn.Module):
    """motion_module.py:51-85."""

    def __init__(self, in_channels, num_attention_heads=8, num_transformer_block=2,
                 attention_block_types=("Temporal_Self", "Temporal_Self"), cross_frame_attention_mode=None,
                 temporal_position_encoding=False, temporal_position_encoding_max_len=32, temporal_attention_dim_div=1,
                 zero_initialize=True):
        super().__init__()
        self.temporal_transformer = TemporalTransformer3DModel(
            in_channels=in_channels, num_attention_heads=num_attention_heads,
            attention_head_dim=in_channels // num_attention_heads // temporal_attention_dim_div,
            num_layers=num_transformer_block, attention_block_types=attention_block_types,
            cross_frame_attention_mode=cross_frame_attention_mode,
            temporal_position_encoding=temporal_position_encoding,
            temporal_position_encoding_max_len=temporal_position_encoding_max_len)
        if zero_initialize:
            self.temporal_transformer.proj_out = zero_module(self.temporal_transformer.proj_out)

    def forward(self, input_tensor, temb, encoder_hidden_states, attention_mask=None, anchor_frame_idx=None,
                video_length=None):
        return self.temporal_transformer(input_tensor, encoder_hidden_states, attention_mask,
                                         video_length=video_length)


def get_motion_module(in_channels, motion_module_type: str, motion_module_kwargs: dict):
    if motion_module_type == "Vanilla":
        return VanillaTemporalModule(in_channels=in_channels, **motion_module_kwargs)
    raise ValueError
