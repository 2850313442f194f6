"""Multi-GPU plumbing: independent samples shard across ranks; ONE broadcast of the packed motion representation.

The reference is single-process / single-GPU (SURVEY.md §2a). Samples (JSONL lines, t2v_video_sample.py:75-105) are
independent, so the path shards with no data-path collective; the only shared state is the reference clip's motion
representation (6 x (fp16 values + uint8 indices), 590 KB at 16x512x512 for the shipped `up_blocks.1`), which rank 0
extracts once and broadcasts as a single contiguous byte buffer (NCCL on GPUs, gloo in the CPU tests). Guided modules
at other or mixed UNet levels have sizes of their own: `representation_manifest_for` derives them from the UNet."""
from __future__ import annotations

import os
from typing import Dict, List, Sequence, Tuple

import torch
import torch.distributed as dist


def init_from_env(backend: str | None = None) -> Tuple[int, int, int]:
    """(rank, world, local_rank) from torchrun's environment; initialises the process group when world > 1."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group(backend=backend or ("nccl" if torch.cuda.is_available() else "gloo"),
                                rank=rank, world_size=world)
    return rank, world, local


def shard_samples(n_samples: int, rank: int, world: int) -> List[int]:
    """Round-robin: rank r takes samples r, r+W, ... (SURVEY.md §8e)."""
    return list(range(rank, n_samples, world))


def pack_representation(rep: Dict[str, Sequence[torch.Tensor]]) -> Tuple[torch.Tensor, list]:
    """-> (uint8 buffer, manifest [(name, val_shape, idx_shape)]); values fp16, indices uint8, module order kept."""
    chunks, manifest = [], []
    for name, (val, idx) in rep.items():
        v = val.detach().to(torch.float16).contiguous()
        i = idx.detach().to(torch.uint8).contiguous()
        manifest.append((name, tuple(v.shape), tuple(i.shape)))
        chunks += [v.view(torch.uint8).reshape(-1), i.reshape(-1)]
    return torch.cat(chunks), manifest


def unpack_representation(buf: torch.Tensor, manifest: list) -> Dict[str, List[torch.Tensor]]:
    out, off = {}, 0
    for name, vshape, ishape in manifest:
        nv = 2 * int(torch.Size(vshape).numel())
        ni = int(torch.Size(ishape).numel())
        val = buf[off:off + nv].clone().view(torch.float16).reshape(vshape)
        off += nv
        idx = buf[off:off + ni].clone().reshape(ishape)
        off += ni
        out[name] = [val, idx]
    return out


def representation_manifest(module_names: Sequence[str], positions: int, heads: int, frames: int) -> list:
    """The layout of the packed motion representation is a pure function of the configuration: for every guided module
    (utils/motionclone_functions.py:264-266) top-1 values fp16 and indices uint8 of shape [positions, heads, frames, 1]
    (:79-81), positions = (h/32) * (w/32) for `up_blocks.1`. Every rank derives it locally, so the broadcast below is the
    ONLY collective of the path."""
    shape = (int(positions), int(heads), int(frames), 1)
    return [(str(n), shape, shape) for n in module_names]


def representation_manifest_for(unet, module_names: Sequence[str], height: int, width: int, frames: int) -> list:
    """The manifest for guided modules at any UNet level (any `motion_guidance_blocks`): module m gets
    [positions_m, heads_m, frames, 1], positions_m the latent positions at m's level. Level 0 is the latent
    (height / 8) x (width / 8); each down block but the last halves it, rounding up (stride-2 conv, padding 1);
    down_blocks.i runs at level i, the mid block at the last level and up_blocks.i at level (levels - 1 - i)."""
    levels = len(unet.down_blocks)
    sizes = [(int(height) // 8, int(width) // 8)]
    for _ in range(levels - 1):
        sizes.append(((sizes[-1][0] + 1) // 2, (sizes[-1][1] + 1) // 2))
    out = []
    for name in module_names:
        parts = str(name).split(".")
        if parts[0] == "down_blocks":
            level = int(parts[1])
        elif parts[0] == "up_blocks":
            level = levels - 1 - int(parts[1])
        elif parts[0] == "mid_block":
            level = levels - 1
        else:
            raise ValueError(f"'{name}' is not a module of the down, mid or up blocks")
        h, w = sizes[level]
        shape = (h * w, int(unet.get_submodule(str(name)).heads), int(frames), 1)
        out.append((str(name), shape, shape))
    return out


def manifest_nbytes(manifest: list) -> int:
    return sum(2 * int(torch.Size(v).numel()) + int(torch.Size(i).numel()) for _, v, i in manifest)


def broadcast_representation(rep, device, manifest: list, src: int = 0):
    """B1 (SURVEY.md §8e): rank `src` passes its representation, the others pass None; everyone gets the dict.
    Exactly one collective: a `broadcast` of the packed byte buffer whose layout `manifest` every rank already knows."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return rep
    if dist.get_rank() == src:
        buf, have = pack_representation(rep)
        if [tuple(m) for m in have] != [tuple(m) for m in manifest]:
            raise ValueError("motion representation does not match the manifest derived from the configuration")
        buf = buf.to(device)
    else:
        buf = torch.empty(manifest_nbytes(manifest), dtype=torch.uint8, device=device)
    dist.broadcast(buf, src=src)
    return unpack_representation(buf, manifest)
