"""SparseCtrl (sparse ControlNet for AnimateDiff) on the same NHWC blocks and kernels as the UNet.

Interface, constructor arguments and state-dict keys follow motionclone/models/sparse_controlnet.py:
SparseControlNetConditioningEmbedding (:49-82), SparseControlNetModel (:85-587; from_unet :317-370, forward :450-587).
The half-UNet reuses unet3d's down / mid blocks (motion modules with ONE temporal attention each,
configs/sparsectrl/*.yaml:14), so temporal attention runs on csrc/temporal_attn.cu and the norms / GEGLU on
csrc/norm_act.cu. It is only ever called under no_grad (utils/motionclone_functions.py:177, :25).

Differences underneath: activations are frame-major NHWC; with `set_noisy_sample_input_to_zero` the input is the
conv_in bias broadcast (:516-518) — no convolution runs; the step-invariant condition embedding (:525 recomputes it every
step) is cached per condition tensor.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple, Union

import torch
import torch.nn.functional as F
from torch import nn

from .unet3d import (CL, InflatedConv3d, TimestepEmbedding, Timesteps, UNetMidBlock3DCrossAttn, _Config,
                     get_down_block)


def zero_module(module: nn.Module) -> nn.Module:
    for p in module.parameters():
        nn.init.zeros_(p)
    return module


class SparseControlNetConditioningEmbedding(nn.Module):
    """sparse_controlnet.py:49-82: conv_in -> SiLU -> (conv, SiLU, stride-2 conv, SiLU) x 3 -> zero-init conv_out."""

    def __init__(self, conditioning_embedding_channels: int, conditioning_channels: int = 3,
                 block_out_channels: Tuple[int, ...] = (16, 32, 96, 256)):
        super().__init__()
        self.conv_in = InflatedConv3d(conditioning_channels, block_out_channels[0], kernel_size=3, padding=1)
        self.blocks = nn.ModuleList([])
        for i in range(len(block_out_channels) - 1):
            cin, cout = block_out_channels[i], block_out_channels[i + 1]
            self.blocks.append(InflatedConv3d(cin, cin, kernel_size=3, padding=1))
            self.blocks.append(InflatedConv3d(cin, cout, kernel_size=3, padding=1, stride=2))
        self.conv_out = zero_module(InflatedConv3d(block_out_channels[-1], conditioning_embedding_channels,
                                                   kernel_size=3, padding=1))

    def forward(self, conditioning):  # 4-D [(f), c, H, W] (internal) or the reference's 5-D
        e = F.silu(self.conv_in(conditioning))
        for block in self.blocks:
            e = F.silu(block(e))
        return self.conv_out(e)


class SparseControlNetOutput:
    def __init__(self, down_block_res_samples, mid_block_res_sample):
        self.down_block_res_samples, self.mid_block_res_sample = down_block_res_samples, mid_block_res_sample


class SparseControlNetModel(nn.Module):
    _supports_gradient_checkpointing = False

    def __init__(self, in_channels: int = 4, conditioning_channels: int = 3, flip_sin_to_cos: bool = True,
                 freq_shift: int = 0,
                 down_block_types: Tuple[str, ...] = ("CrossAttnDownBlock3D", "CrossAttnDownBlock3D",
                                                      "CrossAttnDownBlock3D", "DownBlock3D"),
                 only_cross_attention: Union[bool, Tuple[bool, ...]] = False,
                 block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280), layers_per_block: int = 2,
                 downsample_padding: int = 1, mid_block_scale_factor: float = 1, act_fn: str = "silu",
                 norm_num_groups: Optional[int] = 32, norm_eps: float = 1e-5, cross_attention_dim: int = 1280,
                 attention_head_dim: Union[int, Tuple[int, ...]] = 8,
                 num_attention_heads: Optional[Union[int, Tuple[int, ...]]] = None, use_linear_projection: bool = False,
                 class_embed_type: Optional[str] = None, num_class_embeds: Optional[int] = None,
                 upcast_attention: bool = False, resnet_time_scale_shift: str = "default",
                 projection_class_embeddings_input_dim: Optional[int] = None,
                 controlnet_conditioning_channel_order: str = "rgb",
                 conditioning_embedding_out_channels: Optional[Tuple[int, ...]] = (16, 32, 96, 256),
                 global_pool_conditions: bool = False, use_motion_module=True, motion_module_resolutions=(1, 2, 4, 8),
                 motion_module_mid_block=False, motion_module_type="Vanilla", motion_module_kwargs=None,
                 concate_conditioning_mask: bool = True, use_simplified_condition_embedding: bool = False,
                 set_noisy_sample_input_to_zero: bool = False):
        super().__init__()
        self.config = _Config({k: v for k, v in locals().items() if k not in ("self", "__class__")})
        if class_embed_type is not None or num_class_embeds is not None or use_linear_projection or upcast_attention \
                or global_pool_conditions or only_cross_attention not in (False, (False,) * 4, [False] * 4):
            raise NotImplementedError("configuration outside the reference's live SparseCtrl path")
        if motion_module_kwargs is None:
            motion_module_kwargs = dict(num_attention_heads=8, num_transformer_block=1,
                                        attention_block_types=["Temporal_Self"], temporal_position_encoding=True,
                                        temporal_position_encoding_max_len=32, temporal_attention_dim_div=1)
        motion_module_kwargs = {k: v for k, v in dict(motion_module_kwargs).items() if k != "causal_temporal_attention"}
        num_attention_heads = num_attention_heads or attention_head_dim
        if len(block_out_channels) != len(down_block_types):
            raise ValueError(f"Must provide the same number of `block_out_channels` as `down_block_types`. "
                             f"`block_out_channels`: {block_out_channels}. `down_block_types`: {down_block_types}.")
        self.set_noisy_sample_input_to_zero = set_noisy_sample_input_to_zero
        ch = block_out_channels
        self.conv_in = InflatedConv3d(in_channels, ch[0], kernel_size=3, padding=1)
        if concate_conditioning_mask:
            conditioning_channels = conditioning_channels + 1
        self.concate_conditioning_mask = concate_conditioning_mask
        if use_simplified_condition_embedding:
            self.controlnet_cond_embedding = zero_module(InflatedConv3d(conditioning_channels, ch[0], kernel_size=3,
                                                                        padding=1)).to(torch.float16)
        else:
            self.controlnet_cond_embedding = SparseControlNetConditioningEmbedding(
                conditioning_embedding_channels=ch[0], block_out_channels=conditioning_embedding_out_channels,
                conditioning_channels=conditioning_channels).to(torch.float16)
        self.use_simplified_condition_embedding = use_simplified_condition_embedding
        time_embed_dim = ch[0] * 4
        self.time_proj = Timesteps(ch[0], flip_sin_to_cos, freq_shift)
        self.time_embedding = TimestepEmbedding(ch[0], time_embed_dim)
        self.class_embedding = None
        if isinstance(attention_head_dim, int):
            attention_head_dim = (attention_head_dim,) * len(down_block_types)
        if isinstance(num_attention_heads, int):
            num_attention_heads = (num_attention_heads,) * len(down_block_types)

        self.down_blocks = nn.ModuleList([])
        self.controlnet_down_blocks = nn.ModuleList([zero_module(InflatedConv3d(ch[0], ch[0], kernel_size=1))])
        out_c = ch[0]
        for i, btype in enumerate(down_block_types):
            res = 2 ** i
            in_c, out_c = out_c, ch[i]
            final = i == len(ch) - 1
            self.down_blocks.append(get_down_block(
                btype, num_layers=layers_per_block, in_channels=in_c, out_channels=out_c, temb_channels=time_embed_dim,
                add_downsample=not final, resnet_eps=norm_eps, resnet_groups=norm_num_groups,
                cross_attention_dim=cross_attention_dim,
                attn_num_head_channels=attention_head_dim[i] if attention_head_dim[i] is not None else out_c,
                downsample_padding=downsample_padding,
                use_motion_module=use_motion_module and (res in motion_module_resolutions),
                motion_module_type=motion_module_type, motion_module_kwargs=motion_module_kwargs,
                use_inflated_groupnorm=True))  # per-frame norms whatever the UNet uses (sparse_controlnet.py:272)
            for _ in range(layers_per_block + (0 if final else 1)):
                self.controlnet_down_blocks.append(zero_module(InflatedConv3d(out_c, out_c, kernel_size=1)))
        self.controlnet_mid_block = zero_module(InflatedConv3d(ch[-1], ch[-1], kernel_size=1))
        self.mid_block = UNetMidBlock3DCrossAttn(
            in_channels=ch[-1], temb_channels=time_embed_dim, resnet_eps=norm_eps, resnet_groups=norm_num_groups,
            output_scale_factor=mid_block_scale_factor, cross_attention_dim=cross_attention_dim,
            attn_num_head_channels=num_attention_heads[-1],
            use_motion_module=use_motion_module and motion_module_mid_block, motion_module_type=motion_module_type,
            motion_module_kwargs=motion_module_kwargs, use_inflated_groupnorm=True)  # sparse_controlnet.py:310
        self._cond_cache = None

    @property
    def dtype(self):
        return self.conv_in.weight.dtype

    @property
    def device(self):
        return self.conv_in.weight.device

    @staticmethod
    def image_layer_filter(state_dict):
        """sparse_controlnet.py:372-ff: drop the motion-module entries when copying image layers from the UNet."""
        return {k: v for k, v in state_dict.items() if "motion_modules." not in k}

    @classmethod
    def from_unet(cls, unet, controlnet_conditioning_channel_order: str = "rgb",
                  conditioning_embedding_out_channels: Optional[Tuple[int, ...]] = (16, 32, 96, 256),
                  load_weights_from_unet: bool = True, controlnet_additional_kwargs: Optional[dict] = None):
        """sparse_controlnet.py:317-370."""
        c = unet.config
        controlnet = cls(in_channels=c.in_channels, flip_sin_to_cos=c.flip_sin_to_cos, freq_shift=c.freq_shift,
                         down_block_types=c.down_block_types, only_cross_attention=c.only_cross_attention,
                         block_out_channels=c.block_out_channels, layers_per_block=c.layers_per_block,
                         downsample_padding=c.downsample_padding, mid_block_scale_factor=c.mid_block_scale_factor,
                         act_fn=c.act_fn, norm_num_groups=c.norm_num_groups, norm_eps=c.norm_eps,
                         cross_attention_dim=c.cross_attention_dim, attention_head_dim=c.attention_head_dim,
                         num_attention_heads=c.get("num_attention_heads"),
                         use_linear_projection=c.use_linear_projection, class_embed_type=c.class_embed_type,
                         num_class_embeds=c.num_class_embeds, upcast_attention=c.upcast_attention,
                         resnet_time_scale_shift=c.resnet_time_scale_shift,
                         projection_class_embeddings_input_dim=c.get("projection_class_embeddings_input_dim"),
                         controlnet_conditioning_channel_order=controlnet_conditioning_channel_order,
                         conditioning_embedding_out_channels=conditioning_embedding_out_channels,
                         **dict(controlnet_additional_kwargs or {}))
        if load_weights_from_unet:
            for name in ("conv_in", "time_embedding", "down_blocks", "mid_block"):
                missing, unexpected = getattr(controlnet, name).load_state_dict(
                    cls.image_layer_filter(getattr(unet, name).state_dict()), strict=False)
                assert len(unexpected) == 0
        return controlnet

    def _condition_embedding(self, controlnet_cond, conditioning_mask):
        """[1, c, f, H, W] (+ mask) -> 4-D NHWC fp16 embedding [(f), C0, h, w]; cached: it does not change between steps."""
        # identity-keyed: the cache holds the tensors, so their storage cannot be recycled under the same address
        key = (controlnet_cond, conditioning_mask, controlnet_cond._version,
               None if conditioning_mask is None else conditioning_mask._version)
        c = self._cond_cache
        if c is not None and c[0][0] is controlnet_cond and c[0][1] is conditioning_mask and c[0][2:] == key[2:]:
            return c[1]
        cond = controlnet_cond
        if self.concate_conditioning_mask:
            cond = torch.cat([controlnet_cond, conditioning_mask], dim=1)
        cond = cond.to(torch.float16)  # sparse_controlnet.py:523 (hard-coded)
        b, c, f, hh, ww = cond.shape
        x = cond.permute(0, 2, 1, 3, 4).reshape(b * f, c, hh, ww).contiguous(memory_format=CL)
        e = self.controlnet_cond_embedding(x)
        self._cond_cache = (key, e)
        return e

    @torch.no_grad()
    def forward(self, sample, timestep, encoder_hidden_states, controlnet_cond, conditioning_mask=None,
                conditioning_scale: float = 1.0, class_labels=None, attention_mask=None, cross_attention_kwargs=None,
                guess_mode: bool = False, return_dict: bool = True):
        """sparse_controlnet.py:450-587. sample `[b, 4, f, h, w]`; returns 12 down residuals + 1 mid residual, each a
        5-D `[b, c, f, h, w]` view of an NHWC tensor (zero-copy into unet3d's forward)."""
        if attention_mask is not None or class_labels is not None or guess_mode:
            raise NotImplementedError("attention_mask / class_labels / guess_mode are never used by the reference")
        b, _, f, hh, ww = sample.shape
        timesteps = timestep
        if not torch.is_tensor(timesteps):
            dt = torch.float64 if isinstance(timestep, float) else torch.int64
            timesteps = torch.tensor([timesteps], dtype=dt, device=sample.device)
        elif timesteps.dim() == 0:
            timesteps = timesteps[None].to(sample.device)
        timesteps = timesteps.repeat(b // timesteps.shape[0]).expand(b)
        text = encoder_hidden_states.repeat(b // encoder_hidden_states.shape[0], 1, 1)
        emb = self.time_embedding(self.time_proj(timesteps).to(dtype=self.dtype))
        temb = F.silu(emb)
        if self.set_noisy_sample_input_to_zero:  # :516-518: conv_in(0) == bias, no convolution needed
            x = self.conv_in.bias.view(1, -1, 1, 1).expand(b * f, -1, hh, ww)
        else:
            x = self.conv_in(sample.permute(0, 2, 1, 3, 4).reshape(b * f, -1, hh, ww).contiguous(memory_format=CL))
        e = self._condition_embedding(controlnet_cond, conditioning_mask)  # [(f), C0, h, w], batch 1
        x = (x.reshape(b, f, -1, hh, ww) + e.to(x.dtype).reshape(1, f, -1, hh, ww)).reshape(b * f, -1, hh, ww)
        x = x.contiguous(memory_format=CL)

        skips = (x,)
        for blk in self.down_blocks:
            x, outs = blk(x, temb, text, f)
            skips += outs
        x = self.mid_block(x, temb, text, f)

        def out5(t):
            return t.reshape(b, f, t.shape[1], t.shape[2], t.shape[3]).permute(0, 2, 1, 3, 4)

        down = [out5(conv(s) * conditioning_scale) for s, conv in zip(skips, self.controlnet_down_blocks)]
        mid = out5(self.controlnet_mid_block(x) * conditioning_scale)
        if not return_dict:
            return (down, mid)
        return SparseControlNetOutput(down_block_res_samples=down, mid_block_res_sample=mid)
