"""Synthetic (seeded) UNet configs, weights and inputs shared by bench.py, the tests and the golden generator.

There is no network on the build/GPU boxes, so no SD1.5 / AnimateDiff checkpoint exists; BASELINE.json asks for
"random-init SD1.5 + v3_sd15_mm". Weights are drawn per parameter NAME from a counter-based numpy Philox stream so
the reference model (run once in the build container, oracle/gen_golden.py) and this package's model (state-dict keys
identical to the reference: motionclone/models/unet.py:42-249) get bit-identical fp32 values on any machine.

The reference zero-initialises every motion module `proj_out` (motion_module.py:77-78); with random weights that
would make the temporal path a no-op on the output, so it is drawn like any other projection (SURVEY.md appendix).
"""
from __future__ import annotations

import zlib
from typing import Dict, Mapping, Sequence

import numpy as np
import torch

# SD1.5 unet/config.json values read at unet.py:483-487 (not vendored by the reference; listed in SURVEY.md §8c)
UNET_SD15_CONFIG = dict(
    sample_size=64, in_channels=4, out_channels=4, center_input_sample=False, flip_sin_to_cos=True, freq_shift=0,
    down_block_types=("CrossAttnDownBlock3D", "CrossAttnDownBlock3D", "CrossAttnDownBlock3D", "DownBlock3D"),
    mid_block_type="UNetMidBlock3DCrossAttn",
    up_block_types=("UpBlock3D", "CrossAttnUpBlock3D", "CrossAttnUpBlock3D", "CrossAttnUpBlock3D"),
    only_cross_attention=False, block_out_channels=(320, 640, 1280, 1280), layers_per_block=2,
    downsample_padding=1, mid_block_scale_factor=1, act_fn="silu", norm_num_groups=32, norm_eps=1e-5,
    cross_attention_dim=768, attention_head_dim=8, dual_cross_attention=False, use_linear_projection=False,
    class_embed_type=None, num_class_embeds=None, upcast_attention=False, resnet_time_scale_shift="default",
    # configs/model_config/model_config.yaml:1-15 (unet_additional_kwargs)
    use_inflated_groupnorm=True, use_motion_module=True, motion_module_resolutions=(1, 2, 4, 8),
    motion_module_mid_block=False, motion_module_decoder_only=False, motion_module_type="Vanilla",
    motion_module_kwargs=dict(num_attention_heads=8, num_transformer_block=1,
                              attention_block_types=("Temporal_Self", "Temporal_Self"),
                              temporal_position_encoding=True, temporal_attention_dim_div=1, zero_initialize=True),
    unet_use_cross_frame_attention=False, unet_use_temporal_attention=False,
)

# Same topology, narrow channels: the CPU oracle and the reference finish a guided sample in seconds.
UNET_TINY_CONFIG = dict(UNET_SD15_CONFIG, sample_size=16, block_out_channels=(64, 128, 256, 256),
                        cross_attention_dim=96)

# The reference's default GroupNorm mode (unet.py:80, resnet.py:126): resnet and output norms pool their statistics over
# the frames of each batch element (torch.nn.GroupNorm on the 5-D tensor); the state dict is the same.
UNET_SD15_POOLED_GN_CONFIG = dict(UNET_SD15_CONFIG, use_inflated_groupnorm=False)
UNET_TINY_POOLED_GN_CONFIG = dict(UNET_TINY_CONFIG, use_inflated_groupnorm=False)

# configs/model_config/inference-v2.yaml: a motion module in the mid block as well (two more temporal attentions)
UNET_TINY_MIDV2_CONFIG = dict(UNET_TINY_CONFIG, motion_module_mid_block=True)

# configs/model_config/model_config.yaml:17-21
NOISE_SCHEDULER_KWARGS = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="linear", steps_offset=1,
                              clip_sample=False)


def _rng(name: str, seed: int) -> np.random.Generator:
    return np.random.Generator(np.random.Philox(key=[zlib.crc32(name.encode()), seed]))


def synthetic_tensor(name: str, shape: Sequence[int], seed: int) -> torch.Tensor:
    """fp32 tensor for parameter `name`; scale chosen by role so activations stay O(1)-O(10) in fp16."""
    shape = tuple(int(s) for s in shape)
    z = _rng(name, seed).standard_normal(size=shape, dtype=np.float32)
    leaf = name.rsplit(".", 1)[-1]
    if len(shape) >= 2:  # conv / linear weight: fan-in scaling; branch-closing projections at half gain
        fan_in = int(np.prod(shape[1:]))
        closing = any(t in name for t in (".to_out.0.", ".ff.net.2.", ".proj_out.", ".conv2.", ".conv_out."))
        z *= (0.5 if closing else 1.0) / np.sqrt(fan_in)
    elif leaf == "weight":  # norm gain
        z = 1.0 + 0.1 * z
    else:  # bias
        z *= 0.05
    return torch.from_numpy(np.ascontiguousarray(z))


def synthetic_state_dict(shapes: Mapping[str, Sequence[int]], seed: int = 42) -> Dict[str, torch.Tensor]:
    return {k: synthetic_tensor(k, s, seed) for k, s in shapes.items()}


def load_synthetic_weights(module: torch.nn.Module, seed: int = 42) -> None:
    """In-place, parameter by parameter (no second full copy of a 1.3 B-parameter model in RAM)."""
    with torch.no_grad():
        for k, p in module.state_dict().items():
            p.copy_(synthetic_tensor(k, p.shape, seed).to(dtype=p.dtype, device=p.device))


def synthetic_normal(tag: str, shape: Sequence[int], seed: int) -> torch.Tensor:
    shape = tuple(int(s) for s in shape)
    return torch.from_numpy(_rng("input:" + tag, seed).standard_normal(size=shape, dtype=np.float32))


# configs/sparsectrl/latent_condition.yaml / image_condition.yaml (controlnet_additional_kwargs)
_SPARSECTRL_COMMON = dict(set_noisy_sample_input_to_zero=True, use_motion_module=True, motion_module_resolutions=[1, 2, 4, 8],
                          motion_module_mid_block=False, motion_module_type="Vanilla",
                          motion_module_kwargs=dict(num_attention_heads=8, num_transformer_block=1,
                                                    attention_block_types=["Temporal_Self"],
                                                    temporal_position_encoding=True,
                                                    temporal_position_encoding_max_len=32, temporal_attention_dim_div=1))
SPARSECTRL_LATENT_KWARGS = dict(_SPARSECTRL_COMMON, use_simplified_condition_embedding=True, conditioning_channels=4)
SPARSECTRL_IMAGE_KWARGS = dict(_SPARSECTRL_COMMON, use_simplified_condition_embedding=False, conditioning_channels=3)


def synthetic_condition(kind: str, n_images: int, height: int, width: int, video_length: int, seed: int):
    """Synthetic SparseCtrl inputs: 'latent' -> condition latents [n, 4, h/8, w/8] ~ N(0,1) (stands in for the VAE encode
    of the condition images); 'image' -> RGB condition images [n, 3, h, w] quantised to uint8 levels in [0, 1] (what
    ToTensor() yields, motionclone_functions.py:112-117) and clip pixels [f, 3, h, w] in [-1, 1]."""
    if kind == "latent":
        return dict(cond_latents=synthetic_normal("cond_latents", (n_images, 4, height // 8, width // 8), seed))
    u8 = np.random.Generator(np.random.Philox(key=[zlib.crc32(b"cond_images"), seed])).integers(
        0, 256, size=(n_images, 3, height, width), dtype=np.uint8)
    pix = np.random.Generator(np.random.Philox(key=[zlib.crc32(b"clip_pixels"), seed])).uniform(
        -1.0, 1.0, size=(video_length, 3, height, width)).astype(np.float32)
    return dict(cond_images_u8=torch.from_numpy(u8), cond_images=torch.from_numpy(u8).float() / 255.0,
                clip_pixels=torch.from_numpy(pix))


def synthetic_inputs(video_length: int, height: int, width: int, cross_attention_dim: int, seed: int = 42):
    """SURVEY.md §8d: latents seed s, reference-clip latent s+1, clip noise s+2, text embeddings s+3."""
    shp = (1, 4, video_length, height // 8, width // 8)
    return dict(
        noisy_latents=synthetic_normal("latents", shp, seed),
        clip_latents=synthetic_normal("clip", shp, seed + 1),
        clip_noise=synthetic_normal("clip_noise", shp, seed + 2),
        text_embeddings=synthetic_normal("text", (2, 77, cross_attention_dim), seed + 3),  # row 0 = uncond
    )
