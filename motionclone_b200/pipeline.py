"""Pipeline shell and scheduler state for the guided denoising loop.

`AnimationPipeline` mirrors what the nine MotionClone functions touch on the reference's pipeline object
(motionclone/pipelines/pipeline_animation.py:46-324): `unet`, `scheduler`, `vae`, `text_encoder`, `tokenizer`,
`controlnet`, `device`, `_execution_device`, `vae_scale_factor`, `_encode_prompt`, `prepare_latents` (:297-324),
`prepare_extra_step_kwargs` (:265-280), `decode_latents` (:249-263), `progress_bar`. CLIP and the VAE are outside
the hot path (SURVEY.md §2 #9): they are optional collaborators; synthetic runs pass embeddings / latents directly.

`DDIMScheduler` carries the diffusers-0.16 DDIMScheduler state the bound functions read (betas, alphas_cumprod on
the host in fp32, final_alpha_cumprod, init_noise_sigma, config); the step itself is
guidance.schedule_customized_step (reference: motionclone_functions.py:285).
"""
from __future__ import annotations

import inspect
from contextlib import contextmanager
from typing import Optional

import torch

from .unet3d import _Config


class DDIMScheduler:
    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", trained_betas=None, clip_sample: bool = True,
                 set_alpha_to_one: bool = True, steps_offset: int = 0, prediction_type: str = "epsilon",
                 thresholding: bool = False, dynamic_thresholding_ratio: float = 0.995, clip_sample_range: float = 1.0,
                 sample_max_value: float = 1.0):
        self.config = _Config({k: v for k, v in locals().items() if k != "self"})
        if trained_betas is not None:
            self.betas = torch.tensor(trained_betas, dtype=torch.float32)
        elif beta_schedule == "linear":
            self.betas = torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
        elif beta_schedule == "scaled_linear":
            self.betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps,
                                        dtype=torch.float32) ** 2
        else:
            raise NotImplementedError(f"{beta_schedule} does is not implemented for {self.__class__}")
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)  # fp32, host
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.init_noise_sigma = 1.0
        self.num_inference_steps = None
        self.timesteps = torch.arange(num_train_timesteps - 1, -1, -1, dtype=torch.int64)
        self.timesteps_host = self.timesteps.numpy()
        self.variance_type = None

    def scale_model_input(self, sample, timestep=None):
        return sample

    def _get_variance(self, timestep, prev_timestep):
        a_t = self.alphas_cumprod[timestep]
        a_p = self.alphas_cumprod[prev_timestep] if prev_timestep >= 0 else self.final_alpha_cumprod
        return ((1 - a_p) / (1 - a_t)) * (1 - a_t / a_p)

    def step(self, model_output, timestep, sample, eta: float = 0.0, use_clipped_model_output: bool = False,
             generator=None, variance_noise=None, return_dict: bool = True):
        raise NotImplementedError("MotionClone binds customized_step (motionclone_functions.py:285) instead")


class _Bar:
    def update(self, *a):
        pass


class AnimationPipeline:
    def __init__(self, vae=None, text_encoder=None, tokenizer=None, unet=None, scheduler=None, controlnet=None):
        self.vae, self.text_encoder, self.tokenizer = vae, text_encoder, tokenizer
        self.unet, self.scheduler, self.controlnet = unet, scheduler, controlnet
        self.vae_scale_factor = 8 if vae is None else 2 ** (len(vae.config.block_out_channels) - 1)
        self.prompt_embeds: Optional[torch.Tensor] = None  # [2B, 77, c]: [uncond_1..B, cond_1..B] (synthetic runs)
        self.motion_representation_path = None
        self.motion_representation_dict = None
        self.input_config = None

    def to(self, device=None, dtype=None):
        self.unet.to(device=device, dtype=dtype)
        return self

    @property
    def device(self) -> torch.device:
        return self.unet.device

    @property
    def _execution_device(self) -> torch.device:
        return self.device

    @contextmanager
    def progress_bar(self, total=None):
        yield _Bar()

    def invalidate_cuda_graphs(self):
        """Drop the captured UNet forwards (call after replacing or editing weights; see guidance._GraphedUNetForward)."""
        self.__dict__.pop("_unet_graphs", None)

    def set_prompt_embeds(self, embeds: torch.Tensor):
        """[2B, 77, cross_attention_dim] = [uncond_1..B, cond_1..B] for a batch of B samples (the order diffusers'
        _encode_prompt returns, :139 of the functions file); B = 1 is [uncond, cond]. Motion extraction
        (obtain_motion_representation) uses row 0."""
        self.prompt_embeds = embeds
        return self

    def _encode_prompt(self, prompt, device, num_videos_per_prompt, do_classifier_free_guidance, negative_prompt):
        if self.prompt_embeds is not None:
            return self.prompt_embeds.to(device=device, dtype=self.unet.dtype)
        raise NotImplementedError("CLIP text encoding is outside the hot path: call set_prompt_embeds([uncond, cond])")

    def _encode_uncond(self):
        if self.prompt_embeds is not None:
            return self.prompt_embeds[[0]].to(device=self.device, dtype=self.unet.dtype)
        raise NotImplementedError("CLIP text encoding is outside the hot path: call set_prompt_embeds([uncond, cond])")

    def prepare_extra_step_kwargs(self, generator, eta):
        """pipeline_animation.py:265-280."""
        params = set(inspect.signature(self.scheduler.step).parameters.keys())
        kw = {}
        if "eta" in params:
            kw["eta"] = eta
        if "generator" in params:
            kw["generator"] = generator
        return kw

    def prepare_latents(self, batch_size, num_channels_latents, video_length, height, width, dtype, device, generator,
                        latents=None):
        """pipeline_animation.py:297-324."""
        shape = (batch_size, num_channels_latents, video_length, height // self.vae_scale_factor,
                 width // self.vae_scale_factor)
        if isinstance(generator, list) and len(generator) != batch_size:
            raise ValueError(f"You have passed a list of generators of length {len(generator)}, but requested an "
                             f"effective batch size of {batch_size}. Make sure the batch size matches the length of "
                             "the generators.")
        if latents is None:
            if isinstance(generator, list):
                latents = torch.cat([torch.randn(shape, generator=g, device=device, dtype=dtype) for g in generator], 0)
            else:
                latents = torch.randn(shape, generator=generator, device=device, dtype=dtype)
        else:
            if tuple(latents.shape) != shape:
                raise ValueError(f"Unexpected latents shape, got {latents.shape}, expected {shape}")
            latents = latents.to(device=device, dtype=dtype, non_blocking=True)
        return latents * self.scheduler.init_noise_sigma

    @torch.no_grad()
    def decode_latents(self, latents):
        """pipeline_animation.py:249-263 (needs a VAE; excluded from the measured loop)."""
        if self.vae is None:
            raise NotImplementedError("VAE decode is outside the hot path: use sample_video(return_latents=True)")
        f = latents.shape[2]
        z = (1 / 0.18215 * latents).permute(0, 2, 1, 3, 4).flatten(0, 1)
        video = torch.cat([self.vae.decode(z[i:i + 1]).sample for i in range(z.shape[0])])
        video = video.reshape(-1, f, *video.shape[1:]).permute(0, 2, 1, 3, 4)
        return (video / 2 + 0.5).clamp(0, 1).cpu().float().numpy()
