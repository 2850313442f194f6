"""motionclone_b200 — H100-native (sm_90a) implementation of MotionClone's guided video-diffusion denoising loop,
behind the reference's own Python surface (VersatileAttention / CrossAttention / the nine bound functions).
See DESIGN.md; the C ABI underneath is include/motionclone_b200.h."""
from . import _lib  # noqa: F401

__all__ = ["build_pipeline"]


def build_pipeline(unet_config: dict, infer_config: dict, device="cuda", dtype=None, weight_seed: int = 42,
                   state_dict=None, controlnet_kwargs=None, controlnet_state_dict=None, use_cuda_graphs: bool = True,
                   scheduler_kwargs=None):
    """UNet3D (synthetic or given weights) + DDIMScheduler + AnimationPipeline with the nine functions bound
    (what t2v_video_sample.py:36-73 does). `controlnet_kwargs` (configs/sparsectrl/*.yaml controlnet_additional_kwargs)
    adds a SparseCtrl built with from_unet as i2v_video_sample.py:41-59 does (synthetic weights: seed + 1).
    `use_cuda_graphs`: the no-grad UNet forwards of the sampling loop (the plain step's b=2 forward, the guided step's
    unconditional forward) are captured once per shape and replayed (guidance._GraphedUNetForward).
    `scheduler_kwargs` are the inference YAML's noise_scheduler_kwargs (DDIMScheduler arguments such as prediction_type,
    clip_sample, clip_sample_range), laid over the shipped ones (synthetic.NOISE_SCHEDULER_KWARGS)."""
    import torch

    from .guidance import bind_motionclone
    from .pipeline import AnimationPipeline, DDIMScheduler
    from .synthetic import NOISE_SCHEDULER_KWARGS, load_synthetic_weights
    from .unet3d import UNet3DConditionModel, _Config

    dtype = dtype or torch.float16
    unet = UNet3DConditionModel(**unet_config)
    if state_dict is not None:
        unet.load_state_dict(state_dict, strict=False)  # pos_encoder.pe is non-persistent (util.py:137)
    else:
        load_synthetic_weights(unet, weight_seed)
    controlnet = None
    if controlnet_kwargs is not None:
        from .controlnet import SparseControlNetModel
        unet.config["num_attention_heads"] = 8  # i2v_video_sample.py:47-48
        unet.config["projection_class_embeddings_input_dim"] = None
        controlnet = SparseControlNetModel.from_unet(unet, controlnet_additional_kwargs=dict(controlnet_kwargs))
        if controlnet_state_dict is not None:
            controlnet.load_state_dict({k: v for k, v in controlnet_state_dict.items() if "pos_encoder.pe" not in k})
        else:
            load_synthetic_weights(controlnet, weight_seed + 1)
        controlnet = controlnet.to(device=device, dtype=dtype).to(memory_format=torch.channels_last).eval()
    unet = unet.to(device=device, dtype=dtype).to(memory_format=torch.channels_last).eval()
    pipe = AnimationPipeline(unet=unet, scheduler=DDIMScheduler(**dict(NOISE_SCHEDULER_KWARGS, **(scheduler_kwargs or {}))),
                             controlnet=controlnet)
    pipe.use_cuda_graphs = bool(use_cuda_graphs)
    return bind_motionclone(pipe, _Config(dict(infer_config)))
