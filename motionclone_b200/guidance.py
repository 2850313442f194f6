"""The nine MotionClone functions, H100-native (sm_90a), with the reference's names and signatures.

The reference keeps its algorithm in nine free functions (motionclone/utils/motionclone_functions.py) that the entry
scripts bind onto the pipeline / scheduler / unet instances with `fn.__get__(obj)` (t2v_video_sample.py:57-65). The
same nine names live here and bind the same way (`bind_motionclone` does the t2v_video_sample.py:57-73 wiring):

    add_noise                      :19    obtain_motion_representation :25    compute_temp_loss   :85
    sample_video                   :102   single_step_video            :173   get_temp_attn_prob  :260
    schedule_customized_step       :285   schedule_set_timesteps       :413   unet_customized_forward :478

What changes underneath (DESIGN.md §4 T1/T2 and §5):
  * one fused temporal-attention kernel emits the attention output AND the top-1 pair (extraction) or the
    probabilities gathered at the reference indices (guided steps): no second softmax pass, no [N,8,L,L] tensor,
    no topk / gather launches; the loss and its closed-form gradient are two small launches;
  * CFG combine + score-guided DDIM update is one launch; alpha-bar values are indexed on the HOST by step index, so
    the per-step device sync of `alphas_cumprod[timestep]` (:332) is gone;
  * the motion representation is moved to the device once per sample, not once per step (:91, :94).
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Union

import numpy as np
import torch

from . import _lib, ops
from .temporal import MotionRecordProcessor, VersatileAttention
from .unet3d import UNet3DConditionModel, UNet3DConditionOutput  # noqa: F401  (re-export, as the reference does)


def classify_blocks(block_list: Sequence[str], name: str) -> bool:
    """utils/util.py:434-440 (substring match)."""
    return any(block in name for block in block_list)


def _cfg_get(cfg, key, default=None):
    if isinstance(cfg, dict):
        return cfg.get(key, default)
    return getattr(cfg, key, default)


def prep_unet_attention(unet, motion_gudiance_blocks):
    """utils/xformer_attention.py:45-52: install a recording processor on the guided VersatileAttention modules."""
    for name, module in unet.named_modules():
        if "VersatileAttention" in type(module).__name__ and classify_blocks(motion_gudiance_blocks, name):
            module.set_processor(MotionRecordProcessor())
    return unet


def prep_unet_conv(unet):
    """utils/conv_layer.py:64-69: the reference swaps in a numerically identical forward that also stashes
    `record_hidden_state` (never read on the live path). Here it only raises the stash flag."""
    for blk in unet.up_blocks:
        for resnet in blk.resnets:
            resnet.keep_hidden_state = True
    return unet


def guided_modules(self) -> Dict[str, VersatileAttention]:
    """Name -> module in `named_modules()` order: the key order of the motion representation (:264-266)."""
    blocks = _cfg_get(self.input_config, "motion_guidance_blocks")
    return {name: m for name, m in self.unet.named_modules()
            if "VersatileAttention" in type(m).__name__ and classify_blocks(blocks, name)}


def _set_processor_mode(self, mode: Optional[str], ref_idx: Optional[Dict[str, torch.Tensor]] = None):
    for name, m in guided_modules(self).items():
        if m.processor is None:
            m.set_processor(MotionRecordProcessor())
        m.processor.clear()
        m.processor.mode = mode
        m.processor.ref_idx = None if ref_idx is None else ref_idx[name]


def _controlnet_residuals(self, latents, step_t, text, images):
    """SparseCtrl call of :46-72 / :176-197: zero-filled condition + mask with the conditioned frames set, then the
    controlnet under no_grad. The assembled condition is cached (it does not change between steps); so is its embedding
    inside the controlnet."""
    cfg = self.input_config
    idx = list(_cfg_get(cfg, "image_index"))
    # identity-keyed (the cache keeps `images` alive, so its storage cannot be recycled under the same address)
    key = (images, images._version, latents.shape[2], tuple(idx), latents.dtype)
    cache = getattr(self, "_cn_cond_cache", None)
    if cache is None or cache[0][0] is not images or cache[0][1:] != key[1:]:
        shp = list(images.shape)
        shp[2] = latents.shape[2]
        cond = torch.zeros(shp, device=latents.device, dtype=latents.dtype)
        mask = torch.zeros([shp[0], 1] + shp[2:], device=latents.device, dtype=latents.dtype)
        cond[:, :, idx] = images.to(device=latents.device, dtype=latents.dtype)
        mask[:, :, idx] = 1
        self._cn_cond_cache = cache = (key, cond, mask)
    with torch.no_grad():
        return self.controlnet(latents, step_t, encoder_hidden_states=text, controlnet_cond=cache[1],
                               conditioning_mask=cache[2], conditioning_scale=_cfg_get(cfg, "controlnet_scale"),
                               guess_mode=False, return_dict=False)


# ----------------------------------------------------------------------------------------------------------------
# 1. add_noise
# ----------------------------------------------------------------------------------------------------------------
def add_noise(self, timestep, x_0, noise_pred):
    """:19-23."""
    alpha_prod_t = self.scheduler.alphas_cumprod[int(timestep)]
    return ops.add_noise(x_0, noise_pred, alpha_prod_t)


# ----------------------------------------------------------------------------------------------------------------
# 2. obtain_motion_representation
# ----------------------------------------------------------------------------------------------------------------
@torch.no_grad()
def obtain_motion_representation(self, generator=None, motion_representation_path: str = None, duration=None,
                                 use_controlnet=False):
    """:25-82. The VAE-encoded clip is taken from `input_config.video_latents` [1,4,f,h,w] when given (synthetic
    latents, BASELINE.json configs); decoding a video file + VAE + CLIP are outside the path (SURVEY.md §2 #9, #12)
    and require `self.vae` / `self.text_encoder` objects supplied by the caller."""
    cfg = self.input_config
    video_latents = _cfg_get(cfg, "video_latents")
    if video_latents is None:
        raise NotImplementedError("video decode + VAE encode are outside the hot path: pass input_config.video_latents")
    video_latents = video_latents.to(device=self.device, dtype=self.unet.dtype)
    uncond = _cfg_get(cfg, "uncond_embeddings")
    if uncond is None:
        uncond = self._encode_uncond()
    step_t = int(_cfg_get(cfg, "add_noise_step"))
    noise = _cfg_get(cfg, "video_noise")
    if noise is None:
        noise = torch.randn(video_latents.shape, generator=generator, device=video_latents.device,
                            dtype=video_latents.dtype)
    noisy_latents = self.add_noise(step_t, video_latents, noise.to(video_latents))
    down_res = mid_res = None
    if use_controlnet:  # :46-72 — the condition is taken from the CLIP itself at `image_index`
        idx = list(_cfg_get(cfg, "image_index"))
        if self.controlnet.use_simplified_condition_embedding:
            images = video_latents[:, :, idx]
        else:
            pixels = _cfg_get(cfg, "video_pixels")  # [f, 3, H, W] in [-1, 1] == video_preprocess output (:29)
            if pixels is None:
                raise NotImplementedError("video decode is outside the hot path: pass input_config.video_pixels")
            pixels = pixels.to(device=self.device, dtype=self.unet.dtype)
            images = ((pixels.unsqueeze(0).permute(0, 2, 1, 3, 4) + 1) / 2)[:, :, idx]
        down_res, mid_res = _controlnet_residuals(self, noisy_latents, step_t, uncond.to(noisy_latents), images)

    _set_processor_mode(self, "top1")
    self.unet(noisy_latents, step_t, encoder_hidden_states=uncond.to(noisy_latents), return_dict=False,
              only_motion_feature=True, down_block_additional_residuals=down_res,
              mid_block_additional_residual=mid_res)
    motion_representation = {}
    for name, m in guided_modules(self).items():
        val, idx = m.processor.top1  # fused top-1 epilogue == topk(k=1) + uint8 cast of :79
        motion_representation[name] = [val, idx]
    _set_processor_mode(self, None)
    if motion_representation_path is not None:
        torch.save(motion_representation, motion_representation_path)  # same on-disk format as :81
    self.motion_representation_path = motion_representation_path
    self.motion_representation_dict = motion_representation
    self._repr_source = motion_representation_path
    self._repr_on_device = None
    return motion_representation


# ----------------------------------------------------------------------------------------------------------------
# 3. compute_temp_loss / 6. get_temp_attn_prob
# ----------------------------------------------------------------------------------------------------------------
def _device_representation(self, device):
    cache = getattr(self, "_repr_on_device", None)
    if cache is None or cache[0] is not self.motion_representation_dict or cache[1] != device:
        rep = {k: (v[0].to(device=device, dtype=torch.float16).contiguous(),
                   v[1].to(device=device, dtype=torch.uint8).contiguous())
               for k, v in self.motion_representation_dict.items()}
        for k, (val, idx) in rep.items():  # a stale / foreign .pt must fail here, as torch.gather would (:91-92)
            frames = val.shape[-2]
            if val.shape != idx.shape or val.dim() != 4 or val.shape[-1] != 1:
                raise ValueError(f"motion representation '{k}': expected value / index tensors of shape [N, heads, L, 1], "
                                 f"got {tuple(val.shape)} / {tuple(idx.shape)}")
            if int(idx.max()) >= frames:
                raise ValueError(f"motion representation '{k}': index {int(idx.max())} >= video_length {frames}")
        self._repr_on_device = (self.motion_representation_dict, device, rep)
        cache = self._repr_on_device
    return cache[2]


def compute_temp_loss(self, temp_attn_prob_control_dict):
    """:85-100. Values of the dict are either full probabilities `[b*d, heads, f, f]` (the reference's contract) or
    the already-gathered probabilities `[b*d, heads, f, 1]` produced by the fused forward."""
    names = list(temp_attn_prob_control_dict.keys())
    rep = _device_representation(self, next(iter(temp_attn_prob_control_dict.values())).device)
    cur, ref = [], []
    for name in names:
        p = temp_attn_prob_control_dict[name]
        val_ref, idx_ref = rep[name]
        if p.shape[-1] != 1:
            p = torch.gather(p, index=idx_ref.to(torch.int64), dim=-1)  # :92 (API-compat path; differentiable)
        cur.append(p)
        ref.append(val_ref)
    return ops.motion_loss(cur, ref)


def get_temp_attn_prob(self, index_select=None):
    """:260-283. Full probabilities of the guided modules, graph-carrying when the recorded q, k are."""
    if index_select is not None:
        raise NotImplementedError("index_select is dead in every shipped config (SURVEY.md appendix A)")
    out = {}
    for name, m in guided_modules(self).items():
        proc = m.processor
        if proc.probs is not None:
            out[name] = proc.probs  # emitted by the forward tile (mode "probs")
        else:
            out[name] = ops.TemporalProbs.apply(proc._q, proc._k, m.heads, m.scale) \
                if torch.is_grad_enabled() and proc._q.requires_grad else \
                ops.temporal_attention_forward(proc._q, proc._k, None, m.heads, m.scale, want_o=False,
                                               want_probs=True)[1]
    return out


# ----------------------------------------------------------------------------------------------------------------
# 4. sample_video / 5. single_step_video
# ----------------------------------------------------------------------------------------------------------------
def sample_video(self, eta: float = 0.0, generator=None, noisy_latents: Optional[torch.Tensor] = None,
                 add_controlnet: bool = False, return_latents: bool = False):
    """:102-171. `return_latents=True` skips the VAE decode (off the measured path, SURVEY.md §8d) and returns the
    final latents `[1, 4, f, h/8, w/8]`."""
    cfg = self.input_config
    self.add_controlnet = add_controlnet
    if add_controlnet:  # :111-128 — image files + VAE encode are off the path: the caller passes their result
        images = _cfg_get(cfg, "controlnet_images")
        if images is None:
            raise NotImplementedError("image loading + VAE encode are outside the hot path: pass "
                                      "input_config.controlnet_images [1, c, n_images, h, w] (latents x 0.18215 for the "
                                      "simplified embedding, RGB in [0, 1] otherwise)")
        self.controlnet_images = images.to(device=self.device, dtype=self.unet.dtype)
    batch_size = 1
    device = self._execution_device
    self.text_embeddings = self._encode_prompt(_cfg_get(cfg, "new_prompt"), device, 1, True,
                                               _cfg_get(cfg, "negative_prompt"))
    noisy_latents = self.prepare_latents(batch_size, self.unet.config.in_channels, _cfg_get(cfg, "video_length"),
                                         _cfg_get(cfg, "height"), _cfg_get(cfg, "width"), self.text_embeddings.dtype,
                                         device, generator, noisy_latents)
    path = getattr(self, "motion_representation_path", None)
    if path is not None and getattr(self, "_repr_source", None) != path:
        self.motion_representation_dict = torch.load(path)  # :154
        self._repr_source = path
    elif getattr(self, "motion_representation_dict", None) is None:
        raise ValueError("no motion representation: run obtain_motion_representation or set motion_representation_path")
    self.motion_scale = _cfg_get(cfg, "motion_guidance_weight")
    extra_step_kwargs = self.prepare_extra_step_kwargs(generator, eta)
    with self.progress_bar(total=_cfg_get(cfg, "inference_steps")) as bar:
        for step_index, step_t in enumerate(self.scheduler.timesteps_host):
            noisy_latents = self.single_step_video(noisy_latents, step_index, int(step_t), extra_step_kwargs)
            bar.update()
    if return_latents:
        return noisy_latents
    return self.decode_latents(noisy_latents)


class _GraphedUNetForward:
    """CUDA-graph replay of one no-grad `unet(sample, t, text)` shape (round-2 loop engineering, SURVEY.md §8f-2): the
    b=2 forward of a plain step is ~1 700 kernel launches whose inter-launch gaps are ~8 % of its device time; replayed
    as ONE graph launch they disappear. Inputs live in static buffers (the timestep is a 0-dim device tensor, so the
    sinusoidal embedding is computed inside the graph); the TMA tensor maps and kernel arguments recorded at capture keep
    pointing at the graph's own (address-stable) pool. Weights must not be replaced after capture
    (`pipeline.invalidate_cuda_graphs()` drops the captures)."""

    def __init__(self, unet, sample, step_t, text):
        dev = sample.device
        self.sample = sample.clone()
        self.step_t = step_t.detach().to(dev).clone()
        self.text = text.clone()
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side), torch.no_grad():
            for _ in range(2):  # warm-up on the capture stream: lazy initialisations (workspaces, caches) happen here
                unet(self.sample, self.step_t, encoder_hidden_states=self.text)
        torch.cuda.current_stream(dev).wait_stream(side)
        self.graph = torch.cuda.CUDAGraph()
        n0 = _lib.launch_count()
        with torch.cuda.graph(self.graph), torch.no_grad():
            self.out = unet(self.sample, self.step_t, encoder_hidden_states=self.text).sample
        self.n_kernels = _lib.launch_count() - n0  # this library's kernels inside the graph (counted again per replay)

    def __call__(self, sample, step_t, text):
        self.sample.copy_(sample)
        self.step_t.copy_(step_t)
        if text.data_ptr() != self.text.data_ptr():
            self.text.copy_(text)
        self.graph.replay()
        _lib.add_launch_count(self.n_kernels)
        return self.out


def _unet_nograd(self, sample, step_t, text, step_index):
    """No-grad UNet forward without SparseCtrl residuals: replayed from a CUDA graph when the pipeline allows it (the
    timestep then comes from the scheduler's DEVICE copy of the schedule: no host value is baked into the graph)."""
    if not getattr(self, "use_cuda_graphs", False) or not sample.is_cuda:
        return self.unet(sample, step_t, encoder_hidden_states=text).sample
    step_t = self.scheduler.timesteps[step_index]  # 0-dim int64 device tensor, no sync
    graphs = self.__dict__.setdefault("_unet_graphs", {})
    key = (tuple(sample.shape), sample.dtype, tuple(text.shape))
    g = graphs.get(key)
    if g is None:
        g = graphs[key] = _GraphedUNetForward(self.unet, sample, step_t, text)
    return g(sample, step_t, text)


def single_step_video(self, noisy_latents, step_index, step_t, extra_step_kwargs):
    """:173-257."""
    cfg = self.input_config
    down = mid = None
    if getattr(self, "add_controlnet", False):  # :176-197: SparseCtrl at b=2 ([uncond, cond]) under no_grad
        down, mid = _controlnet_residuals(self, noisy_latents.expand(2, -1, -1, -1, -1), step_t, self.text_embeddings,
                                          self.controlnet_images)
    guidance_steps = _cfg_get(cfg, "guidance_steps")
    cfg_scale = _cfg_get(cfg, "cfg_scale")
    if step_index < guidance_steps:
        rep = _device_representation(self, noisy_latents.device)
        control_latents = noisy_latents.clone().detach()
        control_latents.requires_grad = True
        with torch.no_grad():
            _set_processor_mode(self, None)
            if down is None:
                eps_u = _unet_nograd(self, noisy_latents, step_t, self.text_embeddings[[0]], step_index)
            else:
                eps_u = self.unet(noisy_latents, step_t, encoder_hidden_states=self.text_embeddings[[0]],
                                  down_block_additional_residuals=[r[0:1] for r in down],
                                  mid_block_additional_residual=mid[0:1]).sample
        _set_processor_mode(self, "gather", {k: v[1] for k, v in rep.items()})
        eps_c = self.unet(control_latents, step_t, encoder_hidden_states=self.text_embeddings[[1]],
                          down_block_additional_residuals=None if down is None else [r[1:2] for r in down],
                          mid_block_additional_residual=None if mid is None else mid[1:2]).sample
        gathered = {name: m.processor.gathered for name, m in guided_modules(self).items()}
        loss_motion = self.motion_scale * self.compute_temp_loss(gathered)
        if step_index < _cfg_get(cfg, "warm_up_steps"):  # :228-230
            loss_motion = ((step_index + 1) / _cfg_get(cfg, "warm_up_steps")) * loss_motion
        if step_index > guidance_steps - _cfg_get(cfg, "cool_up_steps"):  # :232-234 (strict '>')
            loss_motion = ((guidance_steps - step_index) / _cfg_get(cfg, "cool_up_steps")) * loss_motion
        gradient = torch.autograd.grad(loss_motion, control_latents, allow_unused=True)[0]
        assert gradient is not None, f"Step {step_index}: grad is None"
        self.last_loss, self.last_gradient = loss_motion.detach(), gradient.detach()
        _set_processor_mode(self, None)
        out = self.scheduler.customized_step_fused(eps_c.detach(), eps_u, cfg_scale, step_index,
                                                   control_latents.detach(), score=gradient.detach(),
                                                   **extra_step_kwargs)
        return out.detach()
    with torch.no_grad():
        _set_processor_mode(self, None)
        if down is None:
            pair = _unet_nograd(self, noisy_latents.expand(2, -1, -1, -1, -1), step_t, self.text_embeddings, step_index)
        else:
            pair = self.unet(noisy_latents.expand(2, -1, -1, -1, -1), step_t, encoder_hidden_states=self.text_embeddings,
                             down_block_additional_residuals=down, mid_block_additional_residual=mid).sample
        out = self.scheduler.customized_step_fused(pair[[1]], pair[[0]], cfg_scale, step_index, noisy_latents,
                                                   score=None, **extra_step_kwargs)
    return out.detach()


# ----------------------------------------------------------------------------------------------------------------
# 7. schedule_customized_step / 8. schedule_set_timesteps
# ----------------------------------------------------------------------------------------------------------------
def _step_alphas(self, step_index):
    """:326-335 with the timestep read from the host copy (no device sync)."""
    ts = self.timesteps_host
    t = int(ts[step_index])
    prev_t = int(ts[step_index + 1]) if step_index + 1 < len(ts) else -1
    a_t = self.alphas_cumprod[t]
    a_prev = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.final_alpha_cumprod
    return a_t, a_prev


def _check_step_args(self, eta, use_clipped_model_output, variance_noise, indices, return_middle):
    if self.num_inference_steps is None:
        raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the "
                         "scheduler")  # :303-306
    pt = self.config.prediction_type
    if pt not in ("epsilon", "sample", "v_prediction"):
        raise ValueError(f"prediction_type given as {pt} must be one of `epsilon`, `sample`, or `v_prediction`")
    if pt != "epsilon" or self.config.thresholding or self.config.clip_sample or eta != 0.0 \
            or use_clipped_model_output or variance_noise is not None or indices is not None or return_middle:
        raise NotImplementedError("only the live configuration is built: epsilon prediction, eta=0, no clip/threshold, "
                                  "no indices/return_middle (SURVEY.md appendix A)")


@torch.no_grad()
def schedule_customized_step(self, model_output, step_index: int, sample, eta: float = 0.0,
                             use_clipped_model_output: bool = False, generator=None, variance_noise=None,
                             return_dict: bool = True, score=None, guidance_scale=1.0, indices=None,
                             return_middle=False):
    """:285-409 (`model_output` is the already CFG-combined epsilon, as the reference calls it at :241/:256)."""
    _check_step_args(self, eta, use_clipped_model_output, variance_noise, indices, return_middle)
    a_t, a_prev = _step_alphas(self, step_index)
    if score is not None:
        assert model_output.shape == score.shape  # :381
    use_score = score is not None and guidance_scale > 0.0
    prev_sample = ops.cfg_ddim_step(model_output, None, sample, score if use_score else None, 0.0, a_t, a_prev,
                                    guidance_scale)
    if not return_dict:
        return (prev_sample,)
    return prev_sample, None, a_prev


@torch.no_grad()
def schedule_customized_step_fused(self, eps_cond, eps_uncond, cfg_scale: float, step_index: int, sample,
                                   score=None, guidance_scale=1.0, eta: float = 0.0, generator=None):
    """CFG combine (:239/:255) + customized_step (:285-409) in ONE launch; returns x_{t-1}."""
    _check_step_args(self, eta, False, None, None, False)
    a_t, a_prev = _step_alphas(self, step_index)
    use_score = score is not None and guidance_scale > 0.0
    return ops.cfg_ddim_step(eps_cond, eps_uncond, sample, score if use_score else None, cfg_scale, a_t, a_prev,
                             guidance_scale)


def schedule_set_timesteps(self, num_inference_steps: int, guidance_steps: int = 0, guiduance_scale: float = 0.0,
                           device: Union[str, torch.device] = None, timestep_spacing_type="uneven"):
    """:413-472 (all four spacings; "uneven" is the live one)."""
    T = self.config.num_train_timesteps
    if num_inference_steps > T:
        raise ValueError(f"`num_inference_steps`: {num_inference_steps} cannot be larger than "
                         f"`self.config.train_timesteps`: {T} as the unet model trained with this scheduler can only "
                         f"handle maximal {T} timesteps.")
    self.num_inference_steps = num_inference_steps
    if timestep_spacing_type == "uneven":
        split = int((1 - guiduance_scale) * T)
        tg = np.linspace(split, T - 1, guidance_steps).round()[::-1].copy().astype(np.int64)
        tv = np.linspace(0, split - 1, num_inference_steps - guidance_steps).round()[::-1].copy().astype(np.int64)
        timesteps = np.concatenate((tg, tv))
    elif timestep_spacing_type == "linspace":
        timesteps = np.linspace(0, T - 1, num_inference_steps).round()[::-1].copy().astype(np.int64)
    elif timestep_spacing_type == "leading":
        ratio = T // num_inference_steps
        timesteps = (np.arange(0, num_inference_steps) * ratio).round()[::-1].copy().astype(np.int64)
        timesteps += self.config.steps_offset
    elif timestep_spacing_type == "trailing":
        ratio = T / num_inference_steps
        timesteps = np.round(np.arange(T, 0, -ratio)).astype(np.int64)
        timesteps -= 1
    else:
        raise ValueError(f"{timestep_spacing_type} is not supported. Please make sure to choose one of 'leading' or "
                         "'trailing'.")
    self.timesteps_host = timesteps                      # host copy: indexed by step_index without a device sync
    self.timesteps = torch.from_numpy(timesteps).to(device)


# ----------------------------------------------------------------------------------------------------------------
# 9. unet_customized_forward
# ----------------------------------------------------------------------------------------------------------------
def unet_customized_forward(self, sample, timestep, encoder_hidden_states, class_labels=None, attention_mask=None,
                            down_block_additional_residuals=None, mid_block_additional_residual=None,
                            return_dict: bool = True, only_motion_feature: bool = False):
    """:478-662 — UNet3DConditionModel.forward in this package already IS the customised forward; this wrapper exists
    so `unet.forward = unet_customized_forward.__get__(unet)` (t2v_video_sample.py:59) keeps working."""
    return UNet3DConditionModel.forward(self, sample, timestep, encoder_hidden_states, class_labels, attention_mask,
                                        down_block_additional_residuals, mid_block_additional_residual, return_dict,
                                        only_motion_feature)


def bind_motionclone(pipeline, config):
    """t2v_video_sample.py:57-73: bind the nine functions, freeze the UNet, install processors, set timesteps."""
    s = pipeline.scheduler
    s.customized_step = schedule_customized_step.__get__(s)
    s.customized_step_fused = schedule_customized_step_fused.__get__(s)
    s.customized_set_timesteps = schedule_set_timesteps.__get__(s)
    pipeline.unet.forward = unet_customized_forward.__get__(pipeline.unet)
    pipeline.sample_video = sample_video.__get__(pipeline)
    pipeline.single_step_video = single_step_video.__get__(pipeline)
    pipeline.get_temp_attn_prob = get_temp_attn_prob.__get__(pipeline)
    pipeline.add_noise = add_noise.__get__(pipeline)
    pipeline.compute_temp_loss = compute_temp_loss.__get__(pipeline)
    pipeline.obtain_motion_representation = obtain_motion_representation.__get__(pipeline)
    for p in pipeline.unet.parameters():
        p.requires_grad = False
    if getattr(pipeline, "controlnet", None) is not None:  # i2v_video_sample.py:96-97
        for p in pipeline.controlnet.parameters():
            p.requires_grad = False
    pipeline.input_config, pipeline.unet.input_config = config, config
    pipeline.unet = prep_unet_attention(pipeline.unet, _cfg_get(config, "motion_guidance_blocks"))
    pipeline.unet = prep_unet_conv(pipeline.unet)
    s.customized_set_timesteps(_cfg_get(config, "inference_steps"), _cfg_get(config, "guidance_steps"),
                               _cfg_get(config, "guidance_scale"), device=pipeline.device,
                               timestep_spacing_type="uneven")
    return pipeline
