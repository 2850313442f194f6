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


def _guidance_layout(self):
    """(cut, guided module names, the guided modules in up blocks after the cut). Down-block and mid-block modules and
    those in up blocks <= cut run under grad in the conditional pass and before extraction's early return
    (motionclone_functions.py:602, :627-629); the others run under no_grad, and extraction never reaches them."""
    cut = self.unet._guidance_cut()
    names = list(guided_modules(self))
    late = [n for n in names if n.startswith("up_blocks.") and int(n.split(".")[1]) > cut]
    return cut, names, late


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
    cut, _, late = _guidance_layout(self)
    if late:
        raise ValueError(f"motion_guidance_blocks: guided module(s) {late} lie in up blocks after the cut up_blocks.{cut} "
                         f"(the suffix of the last entry, {list(_cfg_get(cfg, 'motion_guidance_blocks'))[-1]!r}); "
                         "extraction stops after that block and never runs them. End the list with the highest guided "
                         "up block.")
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
def _check_representation(rep, frames: int, label: str = "motion representation"):
    """Value / index tensors of shape [N, heads, frames, 1] with every index < frames (a stale or foreign .pt must fail
    here, as torch.gather would at :91-92). N is checked per module, so modules of different UNet levels (N = the
    latent positions of the module's level) are accepted side by side."""
    for k, (val, idx) in rep.items():
        if val.shape != idx.shape or val.dim() != 4 or val.shape[-1] != 1:
            raise ValueError(f"{label} '{k}': expected value / index tensors of shape [N, heads, L, 1], "
                             f"got {tuple(val.shape)} / {tuple(idx.shape)}")
        if val.shape[-2] != frames:
            raise ValueError(f"{label} '{k}': {val.shape[-2]} frames, the video has {frames}")
        if int(idx.max()) >= frames:
            raise ValueError(f"{label} '{k}': index {int(idx.max())} >= video_length {frames}")


def _rep_to_device(rep, device):
    out = {k: (v[0].to(device=device, dtype=torch.float16).contiguous(),
               v[1].to(device=device, dtype=torch.uint8).contiguous()) for k, v in rep.items()}
    for k, (val, _) in out.items():
        _check_representation({k: out[k]}, val.shape[-2])
    return out


def _device_representation(self, device):
    cache = getattr(self, "_repr_on_device", None)
    if cache is None or cache[0] is not self.motion_representation_dict or cache[1] != device:
        self._repr_on_device = (self.motion_representation_dict, device,
                                _rep_to_device(self.motion_representation_dict, device))
        cache = self._repr_on_device
    return cache[2]


def _device_batch(self, device, batch: int):
    """Per-sample device copies of the B representations the sampling loop runs with (`_sample_reps`, one dict per
    sample; a shared dict is copied once) and, per guided module, the B index tensors concatenated to [B*d, heads, f, 1]:
    the row order ((b*d + p)*heads + h)*f + frame in which the temporal kernel reads its `gather_idx`. Made once per
    sample_video call, not once per step."""
    reps = getattr(self, "_sample_reps", None) or [self.motion_representation_dict] * batch
    cache = getattr(self, "_batch_on_device", None)
    if (cache is None or cache[1] != device or len(cache[0]) != len(reps)
            or any(a is not b for a, b in zip(cache[0], reps))):
        per_dict = {}
        for r in reps:
            if id(r) not in per_dict:
                per_dict[id(r)] = _device_representation(self, device) if r is self.motion_representation_dict \
                    else _rep_to_device(r, device)
        dev_reps = [per_dict[id(r)] for r in reps]
        cat_idx = {k: (dev_reps[0][k][1] if len(reps) == 1 else torch.cat([d[k][1] for d in dev_reps]))
                   for k in dev_reps[0]}
        self._batch_on_device = cache = (list(reps), device, dev_reps, cat_idx)
    return cache[2], cache[3]


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
def _load_representation(rep):
    return torch.load(rep) if isinstance(rep, str) else rep  # :154 (same on-disk format as :81)


def _batch_size(self, text_embeddings, noisy_latents, generator, motion_representation) -> int:
    """B of a sample_video call, from every input that carries it; any disagreement is a ValueError."""
    if text_embeddings.dim() != 3 or text_embeddings.shape[0] < 2 or text_embeddings.shape[0] % 2:
        raise ValueError(f"prompt embeddings must be [2B, 77, c] = [uncond_1..B, cond_1..B], got "
                         f"{tuple(text_embeddings.shape)}")
    counts = {"prompt embeddings (2B rows)": text_embeddings.shape[0] // 2}
    if noisy_latents is not None:
        if noisy_latents.dim() != 5:
            raise ValueError(f"noisy_latents must be [B, 4, f, h/8, w/8], got {tuple(noisy_latents.shape)}")
        counts["noisy_latents"] = noisy_latents.shape[0]
    if isinstance(generator, (list, tuple)):
        counts["generators"] = len(generator)
    if isinstance(motion_representation, (list, tuple)):
        counts["motion representations"] = len(motion_representation)
    if len(set(counts.values())) != 1:
        raise ValueError("batch size mismatch: " + ", ".join(f"{k} {v}" for k, v in counts.items()))
    return next(iter(counts.values()))


def _resolve_representations(self, motion_representation, batch: int, frames: int):
    """The B representation dicts of a call, checked on the host before anything runs on the device. None: the pipeline's
    own (obtain_motion_representation, motion_representation_path or motion_representation_dict), shared by all samples;
    one dict / path: shared; a list of B dicts / paths: one per sample."""
    if motion_representation is None:
        path = getattr(self, "motion_representation_path", None)
        if path is not None and getattr(self, "_repr_source", None) != path:
            self.motion_representation_dict = torch.load(path)  # :154
            self._repr_source = path
        elif getattr(self, "motion_representation_dict", None) is None:
            raise ValueError("no motion representation: run obtain_motion_representation, set "
                             "motion_representation_path or pass motion_representation")
        reps = [self.motion_representation_dict] * batch
    elif isinstance(motion_representation, (list, tuple)):
        reps = [_load_representation(r) for r in motion_representation]
    else:
        self.motion_representation_dict = _load_representation(motion_representation)
        self.motion_representation_path = self._repr_source = None
        reps = [self.motion_representation_dict] * batch
    names = list(guided_modules(self))
    prev = getattr(self, "_reps_checked", None)  # the same dicts as the last call: checked then (no device reads per call)
    if prev is not None and prev[1] == frames and len(prev[0]) == len(reps) and all(a is b for a, b in zip(prev[0], reps)):
        return reps
    checked = set()
    for i, rep in enumerate(reps):
        if id(rep) in checked:
            continue
        missing = [n for n in names if n not in rep]
        if missing:
            raise ValueError(f"motion representation {i}: no entry for guided module(s) {missing}")
        _check_representation({n: rep[n] for n in names}, frames, f"motion representation {i}")
        checked.add(id(rep))
    self._reps_checked = (list(reps), frames)
    return reps


def sample_video(self, eta: float = 0.0, generator=None, noisy_latents: Optional[torch.Tensor] = None,
                 add_controlnet: bool = False, return_latents: bool = False, motion_representation=None):
    """:102-171, for a batch of B samples sharing f, h, w, the schedule and the guidance settings. B comes from the
    inputs: `noisy_latents` [B, 4, f, h/8, w/8] or a list of B generators, prompt embeddings [2B, 77, c] in the order
    [uncond_1..B, cond_1..B], and `motion_representation`: None (the pipeline's own), one dict or path shared by all
    samples, or a list of B dicts or paths. Sample s gets what a B = 1 call on sample s alone gets, up to the
    batch-size-dependent algorithms of cuBLAS / cuDNN (DESIGN.md §5). `return_latents=True` skips the VAE decode (off
    the measured path, SURVEY.md §8d) and returns the final latents [B, 4, f, h/8, w/8]. After a call, `last_loss` is
    the summed guidance loss of the last guided step and `last_loss_per_sample` [B] its per-sample terms."""
    cfg = self.input_config
    device = self._execution_device
    text_embeddings = self._encode_prompt(_cfg_get(cfg, "new_prompt"), device, 1, True,
                                          _cfg_get(cfg, "negative_prompt"))
    batch_size = _batch_size(self, text_embeddings, noisy_latents, generator, motion_representation)
    frames = _cfg_get(cfg, "video_length")
    if add_controlnet and batch_size > 1:
        raise NotImplementedError(f"SparseCtrl (add_controlnet=True) runs one sample per call; got a batch of "
                                  f"{batch_size}: call sample_video once per sample")
    if 2 * batch_size * frames > 1024:  # the plain step's b = 2B UNet pass: GroupNorm takes at most 1024 frames
        raise ValueError(f"a batch of {batch_size} x {frames} frames exceeds 1024 frames in the b = 2B UNet pass: "
                         f"use at most {1024 // (2 * frames)} samples per call")
    cut, names, late = _guidance_layout(self)
    if _cfg_get(cfg, "guidance_steps") > 0 and len(late) == len(names):
        raise ValueError(f"motion_guidance_blocks {list(_cfg_get(cfg, 'motion_guidance_blocks'))}: no guided module "
                         f"runs under grad (guided: {names}; the cut is up_blocks.{cut}, and later up blocks run under "
                         "no_grad), so the guidance loss has no gradient")
    reps = _resolve_representations(self, motion_representation, batch_size, frames)
    self.add_controlnet = add_controlnet
    if add_controlnet:  # :111-128 — image files + VAE encode are off the path: the caller passes their result
        images = _cfg_get(cfg, "controlnet_images")
        if images is None:
            raise NotImplementedError("image loading + VAE encode are outside the hot path: pass "
                                      "input_config.controlnet_images [1, c, n_images, h, w] (latents x 0.18215 for the "
                                      "simplified embedding, RGB in [0, 1] otherwise)")
        self.controlnet_images = images.to(device=self.device, dtype=self.unet.dtype)
    self.text_embeddings = text_embeddings
    noisy_latents = self.prepare_latents(batch_size, self.unet.config.in_channels, frames,
                                         _cfg_get(cfg, "height"), _cfg_get(cfg, "width"), self.text_embeddings.dtype,
                                         device, generator, noisy_latents)
    self.motion_scale = _cfg_get(cfg, "motion_guidance_weight")
    extra_step_kwargs = self.prepare_extra_step_kwargs(generator, eta)
    self._sample_reps = reps
    try:
        with self.progress_bar(total=_cfg_get(cfg, "inference_steps")) as bar:
            for step_index, step_t in enumerate(self.scheduler.timesteps_host):
                noisy_latents = self.single_step_video(noisy_latents, step_index, int(step_t), extra_step_kwargs)
                bar.update()
    finally:  # a direct single_step_video call guides with motion_representation_dict
        self._sample_reps = None
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


def _unet_nograd(self, sample, step_t, text, step_index, samples: int = 1):
    """No-grad UNet forward of `samples` samples without SparseCtrl residuals: replayed from a CUDA graph when the
    pipeline allows it (the timestep then comes from the scheduler's DEVICE copy of the schedule: no host value is baked
    into the graph). The GroupNorm tiling depends on `samples`, so it is part of the graph key."""
    with ops.batch_samples(samples):
        if not getattr(self, "use_cuda_graphs", False) or not sample.is_cuda:
            return self.unet(sample, step_t, encoder_hidden_states=text).sample
        step_t = self.scheduler.timesteps[step_index]  # 0-dim int64 device tensor, no sync
        graphs = self.__dict__.setdefault("_unet_graphs", {})
        key = (tuple(sample.shape), sample.dtype, tuple(text.shape), samples)
        g = graphs.get(key)
        if g is None:
            g = graphs[key] = _GraphedUNetForward(self.unet, sample, step_t, text)
        return g(sample, step_t, text)


def _step_weight(self, step_index, loss):
    """Warm-up / cool-down ramp of the guidance loss (:228-234; the cool-down test is a strict '>')."""
    cfg = self.input_config
    guidance_steps = _cfg_get(cfg, "guidance_steps")
    if step_index < _cfg_get(cfg, "warm_up_steps"):
        loss = ((step_index + 1) / _cfg_get(cfg, "warm_up_steps")) * loss
    if step_index > guidance_steps - _cfg_get(cfg, "cool_up_steps"):
        loss = ((guidance_steps - step_index) / _cfg_get(cfg, "cool_up_steps")) * loss
    return loss


def single_step_video(self, noisy_latents, step_index, step_t, extra_step_kwargs):
    """:173-257 for a batch of B = noisy_latents.shape[0] samples (text embeddings [uncond_1..B, cond_1..B])."""
    cfg = self.input_config
    B = noisy_latents.shape[0]
    text_u, text_c = self.text_embeddings[:B], self.text_embeddings[B:]
    down = mid = None
    if getattr(self, "add_controlnet", False):  # :176-197: SparseCtrl at b=2 ([uncond, cond]) under no_grad
        down, mid = _controlnet_residuals(self, noisy_latents.expand(2, -1, -1, -1, -1), step_t, self.text_embeddings,
                                          self.controlnet_images)
    guidance_steps = _cfg_get(cfg, "guidance_steps")
    cfg_scale = _cfg_get(cfg, "cfg_scale")
    if step_index < guidance_steps:
        dev_reps, cat_idx = _device_batch(self, noisy_latents.device, B)
        control_latents = noisy_latents.clone().detach()
        control_latents.requires_grad = True
        with torch.no_grad():
            _set_processor_mode(self, None)
            if down is None:
                eps_u = _unet_nograd(self, noisy_latents, step_t, text_u, step_index, samples=B)
            else:
                eps_u = self.unet(noisy_latents, step_t, encoder_hidden_states=text_u,
                                  down_block_additional_residuals=[r[0:1] for r in down],
                                  mid_block_additional_residual=mid[0:1]).sample
        _set_processor_mode(self, "gather", cat_idx)
        with ops.batch_samples(B):
            eps_c = self.unet(control_latents, step_t, encoder_hidden_states=text_c,
                              down_block_additional_residuals=None if down is None else [r[1:2] for r in down],
                              mid_block_additional_residual=None if mid is None else mid[1:2]).sample
        gathered = {name: m.processor.gathered for name, m in guided_modules(self).items()}
        # one loss launch per sample on its own contiguous rows: each sample's value and gradient are those of B = 1
        losses = []
        for s in range(B):
            cur, ref = [], []
            for name, p in gathered.items():
                d = p.shape[0] // B
                cur.append(p[s * d:(s + 1) * d])
                ref.append(dev_reps[s][name][0])
            losses.append(_step_weight(self, step_index, self.motion_scale * ops.motion_loss(cur, ref)))
        loss_motion = losses[0]
        for extra in losses[1:]:
            loss_motion = loss_motion + extra
        gradient = torch.autograd.grad(loss_motion, control_latents, allow_unused=True)[0]
        assert gradient is not None, f"Step {step_index}: grad is None"
        self.last_loss, self.last_gradient = loss_motion.detach(), gradient.detach()
        self.last_loss_per_sample = torch.stack([l.detach() for l in losses])
        _set_processor_mode(self, None)
        out = self.scheduler.customized_step_fused(eps_c.detach(), eps_u, cfg_scale, step_index,
                                                   control_latents.detach(), score=gradient.detach(),
                                                   **extra_step_kwargs)
        return out.detach()
    with torch.no_grad():
        _set_processor_mode(self, None)
        if down is None:  # one b = 2B pass [x_1..B, x_1..B]; each CFG pair counts as one GroupNorm sample
            pair = _unet_nograd(self, noisy_latents.repeat(2, 1, 1, 1, 1), step_t, self.text_embeddings, step_index,
                                samples=B)
        else:
            pair = self.unet(noisy_latents.expand(2, -1, -1, -1, -1), step_t, encoder_hidden_states=self.text_embeddings,
                             down_block_additional_residuals=down, mid_block_additional_residual=mid).sample
        out = self.scheduler.customized_step_fused(pair[B:], pair[:B], cfg_scale, step_index, noisy_latents,
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


def _check_step_args(self, indices, return_middle):
    if self.num_inference_steps is None:
        raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the "
                         "scheduler")  # :303-306
    pt = self.config.prediction_type
    if pt not in ops.PREDICTION_TYPES:  # :348-352
        raise ValueError(f"prediction_type given as {pt} must be one of `epsilon`, `sample`, or `v_prediction`")
    unbuilt = [name for name, on in (("thresholding", self.config.thresholding), ("indices", indices is not None),
                                     ("return_middle", return_middle),
                                     ("learned variance", self.variance_type in ("learned", "learned_range"))) if on]
    if unbuilt:
        raise NotImplementedError(f"customized_step: {', '.join(unbuilt)} not built (dynamic thresholding is a per-sample "
                                  "quantile, a kernel of its own; the others are dead in every shipped config, "
                                  "SURVEY.md appendix A)")


def randn_tensor(shape, generator=None, device=None, dtype=None):
    """diffusers 0.16 utils.randn_tensor: a CPU generator draws on the CPU and the result is moved to `device`, a
    generator of the device draws there; a list of B generators draws one [1, ...] tensor each and concatenates, so
    sample s of a batch gets the noise its own generator gives in a B = 1 call."""
    device = torch.device(device)
    rand_device = device
    batch_size = shape[0]
    if generator is not None:
        gen_type = (generator[0] if isinstance(generator, (list, tuple)) else generator).device.type
        if gen_type != device.type and gen_type == "cpu":
            rand_device = torch.device("cpu")
        elif gen_type != device.type and gen_type == "cuda":
            raise ValueError(f"Cannot generate a {device} tensor from a generator of type {gen_type}.")
    if isinstance(generator, (list, tuple)):
        if len(generator) != batch_size:
            raise ValueError(f"{len(generator)} generators for a batch of {batch_size}")
        one = (1,) + tuple(shape[1:])
        return torch.cat([torch.randn(one, generator=g, device=rand_device, dtype=dtype) for g in generator],
                         dim=0).to(device)
    return torch.randn(tuple(shape), generator=generator, device=rand_device, dtype=dtype).to(device)


def _variance_noise(model_output, eta, generator, variance_noise):
    """:391-401. Nothing is drawn when eta <= 0: the generator's state is untouched."""
    if not eta > 0:
        return None
    if variance_noise is not None and generator is not None:
        raise ValueError("Cannot pass both generator and variance_noise. Please make sure that either `generator` or"
                         " `variance_noise` stays `None`.")
    if variance_noise is None:
        return randn_tensor(model_output.shape, generator=generator, device=model_output.device,
                            dtype=model_output.dtype)
    return variance_noise.to(device=model_output.device, dtype=model_output.dtype)


def _fused_step(self, eps_cond, eps_uncond, cfg_scale, step_index, sample, score, guidance_scale, eta,
                use_clipped_model_output, generator, variance_noise, want_pred_x0):
    """One launch for CFG combine + :339-404. The variant follows from the scheduler's configuration and the step's
    arguments alone; the configuration the guided loop ships with (epsilon, no clip, eta = 0) takes mc_cfg_ddim_step."""
    a_t, a_prev = _step_alphas(self, step_index)
    if score is not None:
        assert eps_cond.shape == score.shape  # :381
    if score is None or not guidance_scale > 0.0:
        score = None
    cfg = self.config
    noise = _variance_noise(eps_cond, eta, generator, variance_noise)
    if cfg.prediction_type == "epsilon" and not cfg.clip_sample and not use_clipped_model_output and eta == 0.0:
        return ops.cfg_ddim_step(eps_cond, eps_uncond, sample, score, cfg_scale, a_t, a_prev, guidance_scale), None, a_prev
    prev_sample, pred_x0 = ops.ddim_step(
        eps_cond, eps_uncond, sample, score, cfg_scale, a_t, a_prev, guidance_scale, prediction_type=cfg.prediction_type,
        clip_sample_range=cfg.clip_sample_range if cfg.clip_sample else None,
        use_clipped_model_output=bool(use_clipped_model_output), eta=eta, noise=noise, want_pred_x0=want_pred_x0)
    return prev_sample, pred_x0, a_prev


@torch.no_grad()
def schedule_customized_step(self, model_output, step_index: int, sample, eta: float = 0.0,
                             use_clipped_model_output: bool = False, generator=None, variance_noise=None,
                             return_dict: bool = True, score=None, guidance_scale=1.0, indices=None,
                             return_middle=False):
    """:285-409 (`model_output` is the already CFG-combined model output, as the reference calls it at :241/:256): every
    `prediction_type`, `clip_sample` / `clip_sample_range`, `use_clipped_model_output`, and eta > 0 with the noise of
    `generator` (one, or a list of B for a batch of B) or `variance_noise`. Returns the reference's tuple
    (prev_sample, pred_original_sample, alpha_prod_t_prev); on the shipped configuration (epsilon prediction, no clip,
    eta = 0, `use_clipped_model_output=False`) pred_original_sample is None, as it is not part of that launch."""
    _check_step_args(self, indices, return_middle)
    out = _fused_step(self, model_output, None, 0.0, step_index, sample, score, guidance_scale, eta,
                      use_clipped_model_output, generator, variance_noise, want_pred_x0=return_dict)
    if not return_dict:
        return (out[0],)
    return out


@torch.no_grad()
def schedule_customized_step_fused(self, eps_cond, eps_uncond, cfg_scale: float, step_index: int, sample,
                                   score=None, guidance_scale=1.0, eta: float = 0.0, generator=None,
                                   variance_noise=None, use_clipped_model_output: bool = False):
    """CFG combine (:239/:255) + customized_step (:285-409) in ONE launch for the whole batch; returns x_{t-1}."""
    _check_step_args(self, None, False)
    return _fused_step(self, eps_cond, eps_uncond, cfg_scale, step_index, sample, score, guidance_scale, eta,
                       use_clipped_model_output, generator, variance_noise, want_pred_x0=False)[0]


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
