"""CPU restatement of the mid-block motion module (models/unet_blocks.py:271-278 with motion_module_mid_block=True, the v2
model config configs/model_config/inference-v2.yaml). TEST INFRASTRUCTURE, like oracle/mc_oracle.py, whose down and mid
blocks build no mid-block motion module.

`mid_block_motion_module()` swaps mc_oracle's `_down_and_mid` for the version below while it is active, so every entry
point of mc_oracle (unet_forward, obtain_motion_representation, single_step, sample_loop) runs the v2 topology; guided
blocks are given to them as before (`guidance_blocks`, `motion_guidance_blocks`).
"""
from __future__ import annotations

from contextlib import contextmanager
from typing import Optional

from torch import Tensor

from oracle import mc_oracle as O


def _down_and_mid_v2(sd: O._SD, cfg: dict, x: Tensor, emb: Tensor, text: Tensor, mm_heads: int, pes: dict,
                     record: Optional[dict], guided, prefix: str = ""):
    """mc_oracle._down_and_mid with the mid block of models/unet_blocks.py:271-278:
    resnets.0 -> (attentions.0 -> motion_modules.0 -> resnets.1)."""
    groups, eps = cfg["norm_num_groups"], cfg["norm_eps"]
    heads = cfg["attention_head_dim"]
    chans = cfg["block_out_channels"]
    skips = [x]
    for i, btype in enumerate(cfg["down_block_types"]):
        blk = sd.sub(f"down_blocks.{i}")
        for j in range(cfg["layers_per_block"]):
            x = O._resnet(blk.sub(f"resnets.{j}"), x, emb, groups, eps)
            if btype.startswith("CrossAttn"):
                x = O._spatial_transformer(blk.sub(f"attentions.{j}"), x, text, heads, groups)
            mname = f"{prefix}down_blocks.{i}.motion_modules.{j}"
            x = O._motion_module(blk.sub(f"motion_modules.{j}"), x, mm_heads, groups, pes, record, mname, guided(mname))
            skips.append(x)
        if i < len(chans) - 1:
            x = O._conv(blk, "downsamplers.0.conv", x, stride=2, padding=1)
            skips.append(x)
    mid = sd.sub("mid_block")
    x = O._resnet(mid.sub("resnets.0"), x, emb, groups, eps)
    x = O._spatial_transformer(mid.sub("attentions.0"), x, text, heads, groups)
    mname = f"{prefix}mid_block.motion_modules.0"
    x = O._motion_module(mid.sub("motion_modules.0"), x, mm_heads, groups, pes, record, mname, guided(mname))
    x = O._resnet(mid.sub("resnets.1"), x, emb, groups, eps)
    return x, skips


@contextmanager
def mid_block_motion_module():
    """mc_oracle with the v2 mid block while the context is active."""
    plain = O._down_and_mid
    O._down_and_mid = _down_and_mid_v2
    try:
        yield
    finally:
        O._down_and_mid = plain
