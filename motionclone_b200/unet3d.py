"""AnimateDiff UNet3D, frame-major NHWC.

Topology, constructor arguments and state-dict keys follow the reference (motionclone/models/unet.py:42-249,
unet_blocks.py, resnet.py) so SD1.5 + AnimateDiff checkpoints map one to one. The forward is the MotionClone one
(utils/motionclone_functions.py:478-662): autograd only up to the last guidance block, `only_motion_feature` early
exit, ControlNet residual inputs.

Layout: between blocks the activation is ONE 4-D tensor `[(b f), C, h, w]` in torch.channels_last, i.e.
physically `[(b f), h, w, C]`. Consequences:
  * the reference's "b c f h w <-> (b f) c h w" rearranges around every conv / norm (resnet.py:14-16, 24-26) vanish;
  * cuDNN runs NHWC tensor-core convolutions with no layout transposes;
  * the transformers' token view `[(b f), h*w, C]` is zero-copy (attention.py:109, :127; motion_module.py:147, :156).
Convolutions, GroupNorm/LayerNorm and the linear layers stay on cuDNN / cuBLAS / ATen (SURVEY.md §2b K11-K13);
the hand-written kernels are in the attention and update path (temporal.py, ops.py).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional, Sequence, Tuple, Union

import torch
import torch.nn.functional as F
from torch import nn

from . import ops
from .spatial import FramePooledGroupNormNHWC, GroupNormNHWC, Transformer3DModel
from .temporal import get_motion_module

CL = torch.channels_last


# ----------------------------------------------------------------------------------------------------------------
# resnet.py equivalents
# ----------------------------------------------------------------------------------------------------------------
def _fold5(x):
    b, c, f, h, w = x.shape
    return x.permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w), (b, f)


def _unfold5(y, bf):
    b, f = bf
    return y.reshape(b, f, *y.shape[1:]).permute(0, 2, 1, 3, 4)


class InflatedConv3d(nn.Conv2d):
    """resnet.py:10-18 — a per-frame 2-D conv. 4-D inputs are the internal fast path; 5-D follows the reference."""

    def forward(self, x):
        if x.dim() == 4:
            return super().forward(x)
        x4, bf = _fold5(x)
        return _unfold5(super().forward(x4), bf)


class InflatedGroupNorm(GroupNormNHWC):
    """resnet.py:21-29; 4-D channels_last inputs take the NHWC kernel (optionally with the SiLU that follows)."""

    def forward(self, x, silu: bool = False, chan_bias=None):
        if x.dim() == 4:
            return super().forward(x, silu, chan_bias)
        x4, bf = _fold5(x)
        return _unfold5(super().forward(x4, silu, chan_bias), bf)


class FramePooledGroupNorm(FramePooledGroupNormNHWC):
    """torch.nn.GroupNorm on the 5-D tensor (resnet.py:143-146, 162-165, unet.py:244-247 with
    use_inflated_groupnorm=False): statistics pooled over the f frames of each batch element. 4-D channels_last
    `[(b f), C, h, w]` inputs take the NHWC kernel with the caller's frame count."""

    def forward(self, x, silu: bool = False, chan_bias=None, frames=None):
        if x.dim() == 4:
            return super().forward(x, silu, chan_bias, frames)
        x4, bf = _fold5(x)
        return _unfold5(super().forward(x4, silu, chan_bias, bf[1]), bf)


class Upsample3D(nn.Module):
    """resnet.py:32-80 (nearest 2x in h, w then conv)."""

    def __init__(self, channels, use_conv=False, use_conv_transpose=False, out_channels=None, name="conv"):
        super().__init__()
        if use_conv_transpose or not use_conv:
            raise NotImplementedError
        self.channels, self.out_channels = channels, out_channels or channels
        self.use_conv, self.use_conv_transpose, self.name = use_conv, use_conv_transpose, name
        self.conv = InflatedConv3d(self.channels, self.out_channels, 3, padding=1)

    def forward(self, x, output_size=None):
        assert x.shape[1] == self.channels and x.dim() == 4
        if output_size is None:
            x = F.interpolate(x, scale_factor=2.0, mode="nearest")
        else:
            x = F.interpolate(x, size=output_size[-2:], mode="nearest")
        return self.conv(x)


class Downsample3D(nn.Module):
    """resnet.py:83-106 (stride-2 conv)."""

    def __init__(self, channels, use_conv=False, out_channels=None, padding=1, name="conv"):
        super().__init__()
        if not use_conv or padding == 0:
            raise NotImplementedError
        self.channels, self.out_channels = channels, out_channels or channels
        self.use_conv, self.padding, self.name = use_conv, padding, name
        self.conv = InflatedConv3d(self.channels, self.out_channels, 3, stride=2, padding=padding)

    def forward(self, x):
        assert x.shape[1] == self.channels
        return self.conv(x)


class ResnetBlock3D(nn.Module):
    """resnet.py:109-213 / utils/conv_layer.py:3-50 (numerically identical; the latter also stashes
    `record_hidden_state`, kept here for the blocks prep_unet_conv touches)."""

    def __init__(self, *, in_channels, out_channels=None, conv_shortcut=False, dropout=0.0, temb_channels=512,
                 groups=32, groups_out=None, pre_norm=True, eps=1e-6, non_linearity="swish",
                 time_embedding_norm="default", output_scale_factor=1.0, use_in_shortcut=None,
                 use_inflated_groupnorm=False):
        super().__init__()
        if time_embedding_norm != "default" or non_linearity not in ("swish", "silu"):
            raise NotImplementedError("scale_shift / mish are never configured by the reference")
        out_channels = in_channels if out_channels is None else out_channels
        self.in_channels, self.out_channels = in_channels, out_channels
        self.time_embedding_norm, self.output_scale_factor = time_embedding_norm, output_scale_factor
        groups_out = groups if groups_out is None else groups_out
        self.use_inflated_groupnorm = use_inflated_groupnorm
        norm = InflatedGroupNorm if use_inflated_groupnorm else FramePooledGroupNorm
        self.norm1 = norm(num_groups=groups, num_channels=in_channels, eps=eps, affine=True)
        self.conv1 = InflatedConv3d(in_channels, out_channels, kernel_size=3, stride=1, padding=1)
        self.time_emb_proj = nn.Linear(temb_channels, out_channels) if temb_channels is not None else None
        self.norm2 = norm(num_groups=groups_out, num_channels=out_channels, eps=eps, affine=True)
        self.dropout = nn.Dropout(dropout)
        self.conv2 = InflatedConv3d(out_channels, out_channels, kernel_size=3, stride=1, padding=1)
        self.nonlinearity = F.silu
        self.use_in_shortcut = self.in_channels != self.out_channels if use_in_shortcut is None else use_in_shortcut
        self.conv_shortcut = InflatedConv3d(in_channels, out_channels, kernel_size=1, stride=1, padding=0) \
            if self.use_in_shortcut else None
        self.record_hidden_state = None
        self.keep_hidden_state = False  # set by prep_unet_conv (utils/conv_layer.py:64-69)

    def _fused_ok(self, x) -> bool:
        ps = (self.conv1.bias, self.conv2.bias, self.conv_shortcut.bias if self.conv_shortcut is not None else None)
        return (x.is_cuda and x.dtype == torch.float16 and x.is_contiguous(memory_format=CL)
                and self.out_channels % 8 == 0 and self.output_scale_factor == 1.0 and self.time_emb_proj is not None
                and not any(p is not None and p.requires_grad for p in ps))

    def forward(self, x, temb_act):
        """x `[(b f), C, h, w]`; temb_act `[b, temb_channels]` = SiLU(time embedding) (resnet.py:192 applies the SiLU
        in every block; it is hoisted). The projection runs once per batch element and is broadcast over frames.
        Frame-pooled norms take f = (b f) / b frames per batch element."""
        fk = {} if self.use_inflated_groupnorm else {"frames": x.shape[0] // temb_act.shape[0]}
        if self._fused_ok(x):
            # conv biases never get their own elementwise pass: conv1's joins the time embedding inside norm2's
            # channel bias, conv2's (+ the shortcut conv's) joins the residual add (one launch: csrc/elementwise.cu)
            h = F.conv2d(self.norm1(x, silu=True, **fk), self.conv1.weight, None, 1, 1)
            t = self.time_emb_proj(temb_act) + self.conv1.bias
            h = F.conv2d(self.dropout(self.norm2(h, silu=True, chan_bias=t, **fk)), self.conv2.weight, None, 1, 1)
            if self.keep_hidden_state:
                self.record_hidden_state = h
            bias = self.conv2.bias
            if self.conv_shortcut is not None:
                x = F.conv2d(x, self.conv_shortcut.weight, None)
                bias = bias + self.conv_shortcut.bias
            if torch.is_grad_enabled() and (h.requires_grad or x.requires_grad):
                return ops.BiasResidualAddFn.apply(h, x, bias)
            return ops.bias_residual_add(h, x, bias)
        h = self.conv1(self.norm1(x, silu=True, **fk))
        t = self.time_emb_proj(temb_act) if self.time_emb_proj is not None else None
        # `hidden_states + temb` (resnet.py:194-195) is folded into norm2 (broadcast over frames and pixels)
        h = self.conv2(self.dropout(self.norm2(h, silu=True, chan_bias=t, **fk)))
        if self.keep_hidden_state:
            self.record_hidden_state = h
        if self.conv_shortcut is not None:
            x = self.conv_shortcut(x)
        out = x + h
        return out if self.output_scale_factor == 1.0 else out / self.output_scale_factor


# ----------------------------------------------------------------------------------------------------------------
# unet_blocks.py equivalents
# ----------------------------------------------------------------------------------------------------------------
class _BlockBase(nn.Module):
    gradient_checkpointing = False

    @staticmethod
    def _resnet(cin, cout, temb, eps, groups, inflated_gn, scale=1.0):
        return ResnetBlock3D(in_channels=cin, out_channels=cout, temb_channels=temb, eps=eps, groups=groups,
                             output_scale_factor=scale, use_inflated_groupnorm=inflated_gn)

    @staticmethod
    def _attn(heads, cout, cross_dim, groups, **kw):
        return Transformer3DModel(heads, cout // heads, in_channels=cout, num_layers=1, cross_attention_dim=cross_dim,
                                  norm_num_groups=groups, unet_use_cross_frame_attention=False,
                                  unet_use_temporal_attention=False, **kw)

    @staticmethod
    def _mm(cout, use, mtype, mkw):
        return get_motion_module(in_channels=cout, motion_module_type=mtype, motion_module_kwargs=mkw) if use else None


class CrossAttnDownBlock3D(_BlockBase):
    """unet_blocks.py:281-421."""
    has_cross_attention = True

    def __init__(self, in_channels, out_channels, temb_channels, num_layers=1, resnet_eps=1e-6, resnet_groups=32,
                 attn_num_head_channels=1, cross_attention_dim=1280, downsample_padding=1, add_downsample=True,
                 use_motion_module=None, motion_module_type=None, motion_module_kwargs=None,
                 use_inflated_groupnorm=False, **unused):
        super().__init__()
        self.attn_num_head_channels = attn_num_head_channels
        self.resnets = nn.ModuleList([self._resnet(in_channels if i == 0 else out_channels, out_channels, temb_channels,
                                                   resnet_eps, resnet_groups, use_inflated_groupnorm)
                                      for i in range(num_layers)])
        self.attentions = nn.ModuleList([self._attn(attn_num_head_channels, out_channels, cross_attention_dim,
                                                    resnet_groups) for _ in range(num_layers)])
        self.motion_modules = nn.ModuleList([self._mm(out_channels, use_motion_module, motion_module_type,
                                                      motion_module_kwargs) for _ in range(num_layers)])
        self.downsamplers = nn.ModuleList([Downsample3D(out_channels, use_conv=True, out_channels=out_channels,
                                                        padding=downsample_padding, name="op")]) \
            if add_downsample else None

    def forward(self, x, temb, encoder_hidden_states, video_length):
        outs = ()
        for resnet, attn, mm in zip(self.resnets, self.attentions, self.motion_modules):
            x = resnet(x, temb)
            x = attn(x, encoder_hidden_states=encoder_hidden_states, video_length=video_length).sample
            if mm is not None:
                x = mm(x, None, encoder_hidden_states, video_length=video_length)
            outs += (x,)
        if self.downsamplers is not None:
            for d in self.downsamplers:
                x = d(x)
            outs += (x,)
        return x, outs


class DownBlock3D(_BlockBase):
    """unet_blocks.py:424-521."""
    has_cross_attention = False

    def __init__(self, in_channels, out_channels, temb_channels, num_layers=1, resnet_eps=1e-6, resnet_groups=32,
                 add_downsample=True, downsample_padding=1, use_motion_module=None, motion_module_type=None,
                 motion_module_kwargs=None, use_inflated_groupnorm=False, **unused):
        super().__init__()
        self.resnets = nn.ModuleList([self._resnet(in_channels if i == 0 else out_channels, out_channels, temb_channels,
                                                   resnet_eps, resnet_groups, use_inflated_groupnorm)
                                      for i in range(num_layers)])
        self.motion_modules = nn.ModuleList([self._mm(out_channels, use_motion_module, motion_module_type,
                                                      motion_module_kwargs) for _ in range(num_layers)])
        self.downsamplers = nn.ModuleList([Downsample3D(out_channels, use_conv=True, out_channels=out_channels,
                                                        padding=downsample_padding, name="op")]) \
            if add_downsample else None

    def forward(self, x, temb, encoder_hidden_states, video_length):
        outs = ()
        for resnet, mm in zip(self.resnets, self.motion_modules):
            x = resnet(x, temb)
            if mm is not None:
                x = mm(x, None, encoder_hidden_states, video_length=video_length)
            outs += (x,)
        if self.downsamplers is not None:
            for d in self.downsamplers:
                x = d(x)
            outs += (x,)
        return x, outs


class UNetMidBlock3DCrossAttn(_BlockBase):
    """unet_blocks.py:171-278."""
    has_cross_attention = True

    def __init__(self, in_channels, temb_channels, num_layers=1, resnet_eps=1e-6, resnet_groups=32,
                 attn_num_head_channels=1, output_scale_factor=1.0, cross_attention_dim=1280, use_motion_module=None,
                 motion_module_type=None, motion_module_kwargs=None, use_inflated_groupnorm=False, **unused):
        super().__init__()
        self.attn_num_head_channels = attn_num_head_channels
        resnet_groups = resnet_groups if resnet_groups is not None else min(in_channels // 4, 32)
        self.resnets = nn.ModuleList([self._resnet(in_channels, in_channels, temb_channels, resnet_eps, resnet_groups,
                                                   use_inflated_groupnorm, output_scale_factor)
                                      for _ in range(num_layers + 1)])
        self.attentions = nn.ModuleList([self._attn(attn_num_head_channels, in_channels, cross_attention_dim,
                                                    resnet_groups) for _ in range(num_layers)])
        self.motion_modules = nn.ModuleList([self._mm(in_channels, use_motion_module, motion_module_type,
                                                      motion_module_kwargs) for _ in range(num_layers)])

    def forward(self, x, temb, encoder_hidden_states, video_length):
        x = self.resnets[0](x, temb)
        for attn, resnet, mm in zip(self.attentions, self.resnets[1:], self.motion_modules):
            x = attn(x, encoder_hidden_states=encoder_hidden_states, video_length=video_length).sample
            if mm is not None:
                x = mm(x, None, encoder_hidden_states, video_length=video_length)
            x = resnet(x, temb)
        return x


class CrossAttnUpBlock3D(_BlockBase):
    """unet_blocks.py:524-667."""
    has_cross_attention = True

    def __init__(self, in_channels, out_channels, prev_output_channel, temb_channels, num_layers=1, resnet_eps=1e-6,
                 resnet_groups=32, attn_num_head_channels=1, cross_attention_dim=1280, add_upsample=True,
                 use_motion_module=None, motion_module_type=None, motion_module_kwargs=None,
                 use_inflated_groupnorm=False, **unused):
        super().__init__()
        self.attn_num_head_channels = attn_num_head_channels
        resnets = []
        for i in range(num_layers):
            skip = in_channels if i == num_layers - 1 else out_channels
            cin = prev_output_channel if i == 0 else out_channels
            resnets.append(self._resnet(cin + skip, out_channels, temb_channels, resnet_eps, resnet_groups,
                                        use_inflated_groupnorm))
        self.resnets = nn.ModuleList(resnets)
        self.attentions = nn.ModuleList([self._attn(attn_num_head_channels, out_channels, cross_attention_dim,
                                                    resnet_groups) for _ in range(num_layers)])
        self.motion_modules = nn.ModuleList([self._mm(out_channels, use_motion_module, motion_module_type,
                                                      motion_module_kwargs) for _ in range(num_layers)])
        self.upsamplers = nn.ModuleList([Upsample3D(out_channels, use_conv=True, out_channels=out_channels)]) \
            if add_upsample else None

    def forward(self, x, res_hidden_states_tuple, temb, encoder_hidden_states, video_length, upsample_size=None):
        for resnet, attn, mm in zip(self.resnets, self.attentions, self.motion_modules):
            x = torch.cat([x, res_hidden_states_tuple[-1]], dim=1)
            res_hidden_states_tuple = res_hidden_states_tuple[:-1]
            x = resnet(x, temb)
            x = attn(x, encoder_hidden_states=encoder_hidden_states, video_length=video_length).sample
            if mm is not None:
                x = mm(x, None, encoder_hidden_states, video_length=video_length)
        if self.upsamplers is not None:
            for u in self.upsamplers:
                x = u(x, upsample_size)
        return x


class UpBlock3D(_BlockBase):
    """unet_blocks.py:670-760."""
    has_cross_attention = False

    def __init__(self, in_channels, prev_output_channel, out_channels, temb_channels, num_layers=1, resnet_eps=1e-6,
                 resnet_groups=32, add_upsample=True, use_motion_module=None, motion_module_type=None,
                 motion_module_kwargs=None, use_inflated_groupnorm=False, **unused):
        super().__init__()
        resnets = []
        for i in range(num_layers):
            skip = in_channels if i == num_layers - 1 else out_channels
            cin = prev_output_channel if i == 0 else out_channels
            resnets.append(self._resnet(cin + skip, out_channels, temb_channels, resnet_eps, resnet_groups,
                                        use_inflated_groupnorm))
        self.resnets = nn.ModuleList(resnets)
        self.motion_modules = nn.ModuleList([self._mm(out_channels, use_motion_module, motion_module_type,
                                                      motion_module_kwargs) for _ in range(num_layers)])
        self.upsamplers = nn.ModuleList([Upsample3D(out_channels, use_conv=True, out_channels=out_channels)]) \
            if add_upsample else None

    def forward(self, x, res_hidden_states_tuple, temb, encoder_hidden_states, video_length, upsample_size=None):
        for resnet, mm in zip(self.resnets, self.motion_modules):
            x = torch.cat([x, res_hidden_states_tuple[-1]], dim=1)
            res_hidden_states_tuple = res_hidden_states_tuple[:-1]
            x = resnet(x, temb)
            if mm is not None:
                x = mm(x, None, encoder_hidden_states, video_length=video_length)
        if self.upsamplers is not None:
            for u in self.upsamplers:
                x = u(x, upsample_size)
        return x


_DOWN = {"CrossAttnDownBlock3D": CrossAttnDownBlock3D, "DownBlock3D": DownBlock3D}
_UP = {"CrossAttnUpBlock3D": CrossAttnUpBlock3D, "UpBlock3D": UpBlock3D}


def get_down_block(down_block_type, **kw):
    """unet_blocks.py:12-89."""
    t = down_block_type[7:] if down_block_type.startswith("UNetRes") else down_block_type
    if t not in _DOWN:
        raise ValueError(f"{t} does not exist.")
    if t == "CrossAttnDownBlock3D" and kw.get("cross_attention_dim") is None:
        raise ValueError("cross_attention_dim must be specified for CrossAttnDownBlock3D")
    return _DOWN[t](**kw)


def get_up_block(up_block_type, **kw):
    """unet_blocks.py:92-168."""
    t = up_block_type[7:] if up_block_type.startswith("UNetRes") else up_block_type
    if t not in _UP:
        raise ValueError(f"{t} does not exist.")
    if t == "CrossAttnUpBlock3D" and kw.get("cross_attention_dim") is None:
        raise ValueError("cross_attention_dim must be specified for CrossAttnUpBlock3D")
    return _UP[t](**kw)


# ----------------------------------------------------------------------------------------------------------------
# time embedding (diffusers 0.16 Timesteps / TimestepEmbedding, used at unet.py:101-104)
# ----------------------------------------------------------------------------------------------------------------
class Timesteps(nn.Module):
    def __init__(self, num_channels: int, flip_sin_to_cos: bool, downscale_freq_shift: float):
        super().__init__()
        self.num_channels, self.flip_sin_to_cos, self.downscale_freq_shift = num_channels, flip_sin_to_cos, downscale_freq_shift

    def forward(self, timesteps):
        half = self.num_channels // 2
        exponent = -math.log(10000) * torch.arange(half, dtype=torch.float32, device=timesteps.device)
        emb = timesteps[:, None].float() * torch.exp(exponent / (half - self.downscale_freq_shift))[None, :]
        sin, cos = torch.sin(emb), torch.cos(emb)
        return torch.cat([cos, sin], dim=-1) if self.flip_sin_to_cos else torch.cat([sin, cos], dim=-1)


class TimestepEmbedding(nn.Module):
    def __init__(self, in_channels: int, time_embed_dim: int):
        super().__init__()
        self.linear_1 = nn.Linear(in_channels, time_embed_dim)
        self.act = nn.SiLU()
        self.linear_2 = nn.Linear(time_embed_dim, time_embed_dim)

    def forward(self, sample):
        return self.linear_2(self.act(self.linear_1(sample)))


@dataclass
class UNet3DConditionOutput:
    sample: torch.Tensor


class _Config(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)


class UNet3DConditionModel(nn.Module):
    """unet.py:38-249 (constructor / topology) with the MotionClone forward (motionclone_functions.py:478-662)."""

    _supports_gradient_checkpointing = False

    def __init__(self, sample_size: Optional[int] = None, in_channels: int = 4, out_channels: int = 4,
                 center_input_sample: bool = False, flip_sin_to_cos: bool = True, freq_shift: int = 0,
                 down_block_types: Tuple[str, ...] = ("CrossAttnDownBlock3D", "CrossAttnDownBlock3D",
                                                      "CrossAttnDownBlock3D", "DownBlock3D"),
                 mid_block_type: str = "UNetMidBlock3DCrossAttn",
                 up_block_types: Tuple[str, ...] = ("UpBlock3D", "CrossAttnUpBlock3D", "CrossAttnUpBlock3D",
                                                    "CrossAttnUpBlock3D"),
                 only_cross_attention: Union[bool, Tuple[bool, ...]] = False,
                 block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280), layers_per_block: int = 2,
                 downsample_padding: int = 1, mid_block_scale_factor: float = 1, act_fn: str = "silu",
                 norm_num_groups: int = 32, norm_eps: float = 1e-5, cross_attention_dim: int = 1280,
                 attention_head_dim: Union[int, Tuple[int, ...]] = 8, dual_cross_attention: bool = False,
                 use_linear_projection: bool = False, class_embed_type: Optional[str] = None,
                 num_class_embeds: Optional[int] = None, upcast_attention: bool = False,
                 resnet_time_scale_shift: str = "default", use_inflated_groupnorm=False, use_motion_module=False,
                 motion_module_resolutions=(1, 2, 4, 8), motion_module_mid_block=False,
                 motion_module_decoder_only=False, motion_module_type=None, motion_module_kwargs=None,
                 unet_use_cross_frame_attention=False, unet_use_temporal_attention=False):
        super().__init__()
        cfg = {k: v for k, v in locals().items() if k not in ("self", "__class__")}
        self.config = _Config(cfg)
        if class_embed_type is not None or num_class_embeds is not None or dual_cross_attention or upcast_attention \
                or use_linear_projection or unet_use_cross_frame_attention or unet_use_temporal_attention \
                or center_input_sample or only_cross_attention not in (False, (False,) * 4, [False] * 4):
            raise NotImplementedError("configuration outside the reference's live path (SURVEY.md appendix A)")
        motion_module_kwargs = dict(motion_module_kwargs or {})
        self.sample_size = sample_size
        self.input_config = None  # set by the driver (t2v_video_sample.py:69)
        ch = block_out_channels
        time_embed_dim = ch[0] * 4
        self.conv_in = InflatedConv3d(in_channels, ch[0], kernel_size=3, padding=(1, 1))
        self.time_proj = Timesteps(ch[0], flip_sin_to_cos, freq_shift)
        self.time_embedding = TimestepEmbedding(ch[0], time_embed_dim)
        self.class_embedding = None
        if isinstance(attention_head_dim, int):
            attention_head_dim = (attention_head_dim,) * len(down_block_types)

        # registered before the mid block, as in unet.py:116-118 (`self.mid_block = None` registers nothing): module
        # order down, up, mid is the key order of a motion representation that guides the mid block's motion module
        self.down_blocks = nn.ModuleList()
        self.up_blocks = nn.ModuleList()
        out_c = ch[0]
        for i, btype in enumerate(down_block_types):
            res = 2 ** i
            in_c, out_c = out_c, ch[i]
            self.down_blocks.append(get_down_block(
                btype, num_layers=layers_per_block, in_channels=in_c, out_channels=out_c, temb_channels=time_embed_dim,
                add_downsample=i != len(ch) - 1, resnet_eps=norm_eps, resnet_groups=norm_num_groups,
                cross_attention_dim=cross_attention_dim, attn_num_head_channels=attention_head_dim[i],
                downsample_padding=downsample_padding,
                use_motion_module=use_motion_module and (res in motion_module_resolutions) and not motion_module_decoder_only,
                motion_module_type=motion_module_type, motion_module_kwargs=motion_module_kwargs,
                use_inflated_groupnorm=use_inflated_groupnorm))

        if mid_block_type != "UNetMidBlock3DCrossAttn":
            raise ValueError(f"unknown mid_block_type : {mid_block_type}")
        self.mid_block = UNetMidBlock3DCrossAttn(
            in_channels=ch[-1], temb_channels=time_embed_dim, resnet_eps=norm_eps, resnet_groups=norm_num_groups,
            output_scale_factor=mid_block_scale_factor, cross_attention_dim=cross_attention_dim,
            attn_num_head_channels=attention_head_dim[-1],
            use_motion_module=use_motion_module and motion_module_mid_block, motion_module_type=motion_module_type,
            motion_module_kwargs=motion_module_kwargs, use_inflated_groupnorm=use_inflated_groupnorm)

        self.num_upsamplers = 0
        rch = list(reversed(ch))
        rheads = list(reversed(attention_head_dim))
        out_c = rch[0]
        for i, btype in enumerate(up_block_types):
            res = 2 ** (3 - i)
            final = i == len(ch) - 1
            prev_c, out_c = out_c, rch[i]
            in_c = rch[min(i + 1, len(ch) - 1)]
            self.num_upsamplers += 0 if final else 1
            self.up_blocks.append(get_up_block(
                btype, num_layers=layers_per_block + 1, in_channels=in_c, out_channels=out_c,
                prev_output_channel=prev_c, temb_channels=time_embed_dim, add_upsample=not final,
                resnet_eps=norm_eps, resnet_groups=norm_num_groups, cross_attention_dim=cross_attention_dim,
                attn_num_head_channels=rheads[i],
                use_motion_module=use_motion_module and (res in motion_module_resolutions),
                motion_module_type=motion_module_type, motion_module_kwargs=motion_module_kwargs,
                use_inflated_groupnorm=use_inflated_groupnorm))

        # resnet norms and the output norm only: the transformer and motion-module norms stay per frame in both modes
        norm_out = InflatedGroupNorm if use_inflated_groupnorm else FramePooledGroupNorm
        self.conv_norm_out = norm_out(num_channels=ch[0], num_groups=norm_num_groups, eps=norm_eps)
        self.conv_act = nn.SiLU()
        self.conv_out = InflatedConv3d(ch[0], out_channels, kernel_size=3, padding=1)

    # ---- plumbing the reference gets from diffusers' ModelMixin ----
    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @property
    def device(self):
        return next(self.parameters()).device

    def enable_xformers_memory_efficient_attention(self, *a, **k):
        return self  # fused attention cores are always on (t2v_video_sample.py:39-40 keeps working)

    def set_attention_slice(self, slice_size):
        return None  # unet.py:251-314: never called by the reference; the fused cores do not materialise scores

    def to_channels_last(self):
        return self.to(memory_format=CL)

    # ---- forward ----
    def _guidance_cut(self) -> int:
        """Index of the last up block that runs under grad (and, in extraction, at all): the integer suffix of the last
        `motion_guidance_blocks` entry (motionclone_functions.py:602). An entry without one ('mid_block', 'up_blocks')
        raises the ValueError of int(), as in the reference."""
        cfg = self.input_config
        blocks = getattr(cfg, "motion_guidance_blocks", None) if cfg is not None else None
        if blocks is None and isinstance(cfg, dict):
            blocks = cfg.get("motion_guidance_blocks")
        if blocks is None:
            return len(self.up_blocks) - 1
        return int(blocks[-1].split(".")[-1])  # motionclone_functions.py:602

    def forward(self, sample: torch.Tensor, timestep: Union[torch.Tensor, float, int],
                encoder_hidden_states: torch.Tensor, class_labels: Optional[torch.Tensor] = None,
                attention_mask: Optional[torch.Tensor] = None,
                down_block_additional_residuals: Optional[Sequence[torch.Tensor]] = None,
                mid_block_additional_residual: Optional[torch.Tensor] = None, return_dict: bool = True,
                only_motion_feature: bool = False):
        """Signature of unet_customized_forward (motionclone_functions.py:478-492). sample `[b, 4, f, h, w]`,
        encoder_hidden_states `[b, 77, c]`; returns `.sample [b, 4, f, h, w]`."""
        if attention_mask is not None or class_labels is not None:
            raise NotImplementedError("attention_mask / class_labels are never passed on the live path")
        cut = self._guidance_cut()  # before any launch: a bad block list fails here, not after the down blocks ran
        b, cin, f, hh, ww = sample.shape
        up_factor = 2 ** self.num_upsamplers
        forward_upsample_size = any(s % up_factor != 0 for s in (hh, ww))  # :516-518

        timesteps = timestep
        if not torch.is_tensor(timesteps):
            dt = torch.float64 if isinstance(timestep, float) else torch.int64
            timesteps = torch.tensor([timesteps], dtype=dt, device=sample.device)
        elif timesteps.dim() == 0:
            timesteps = timesteps[None].to(sample.device)
        timesteps = timesteps.expand(b)
        emb = self.time_embedding(self.time_proj(timesteps).to(dtype=self.dtype))  # :545-551
        temb = F.silu(emb)  # every resnet applies SiLU before its own projection (resnet.py:192): hoisted

        x = sample.permute(0, 2, 1, 3, 4).reshape(b * f, cin, hh, ww).contiguous(memory_format=CL)
        x = self.conv_in(x)
        skips = (x,)
        for blk in self.down_blocks:
            x, outs = blk(x, temb, encoder_hidden_states, f)
            skips += outs

        def as4d(r):  # ControlNet residuals arrive 5-D [b,c,f,h,w] or 4-D broadcast over frames (:585-587)
            if r.dim() == 5:
                return r.permute(0, 2, 1, 3, 4).reshape(b * f, r.shape[1], r.shape[3], r.shape[4])
            return r.repeat_interleave(f, dim=0)

        if down_block_additional_residuals is not None:
            skips = tuple(s + as4d(r) for s, r in zip(skips, down_block_additional_residuals))
        x = self.mid_block(x, temb, encoder_hidden_states, f)
        if mid_block_additional_residual is not None:
            x = x + as4d(mid_block_additional_residual)

        for i, blk in enumerate(self.up_blocks):
            if i > cut and only_motion_feature:
                return 0  # :627-628
            n = len(blk.resnets)
            res, skips = skips[-n:], skips[:-n]
            size = skips[-1].shape[2:] if (i != len(self.up_blocks) - 1 and forward_upsample_size) else None
            if i <= cut:
                x = blk(x, res, temb, encoder_hidden_states, f, upsample_size=size)
            else:
                with torch.no_grad():  # :629
                    x = blk(x, res, temb, encoder_hidden_states, f, upsample_size=size)

        fk = {} if self.config.use_inflated_groupnorm else {"frames": f}
        x = self.conv_out(self.conv_norm_out(x, silu=True, **fk))  # conv_act (SiLU) fused into the norm
        out = x.reshape(b, f, x.shape[1], hh, ww).permute(0, 2, 1, 3, 4)
        return UNet3DConditionOutput(sample=out) if return_dict else (out,)
