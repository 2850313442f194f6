"""CPU restatement of the whole scheduler step, utils/motionclone_functions.py:285-409. TEST INFRASTRUCTURE, like
oracle/mc_oracle.py (whose `ddim_guided_step` is the eta = 0 / epsilon / no-clip path of this one): fp32 on the CPU is
the truth mode, the same code on fp16 CUDA tensors is the reference's eager op sequence on that device.

Pinned against runs of the UNMODIFIED reference with eta > 0, v_prediction and clip_sample
(scripts/gen_golden_scheduler.py -> tests/golden/ref_tiny8_{eta,vpred,clip}.npz) in tests/test_scheduler_cpu.py.
"""
from __future__ import annotations

from contextlib import contextmanager
from typing import List, Optional, Sequence

import torch

from . import mc_oracle as O

Tensor = torch.Tensor


def get_variance(a_t: Tensor, a_prev: Tensor) -> Tensor:
    """diffusers 0.16 DDIMScheduler._get_variance (called at :364) on 0-dim fp32 tensors."""
    beta_prod_t = 1 - a_t
    beta_prod_t_prev = 1 - a_prev
    return (beta_prod_t_prev / beta_prod_t) * (1 - a_t / a_prev)


def ddim_step(model_output: Tensor, sample: Tensor, score: Optional[Tensor], a_t: Tensor, a_prev: Tensor,
              guidance_scale: float = 1.0, *, prediction_type: str = "epsilon", clip_sample_range: Optional[float] = None,
              use_clipped_model_output: bool = False, eta: float = 0.0, variance_noise: Optional[Tensor] = None):
    """:335-404, statement for statement; returns (prev_sample, pred_original_sample). `clip_sample_range=None` is
    `clip_sample: false`. Every op rounds to the tensor dtype, as the eager op sequence does."""
    alpha_prod_t = a_t.to(torch.float32).cpu()
    alpha_prod_t_prev = a_prev.to(torch.float32).cpu()
    beta_prod_t = 1 - alpha_prod_t                                                                       # :335
    if prediction_type == "epsilon":                                                                     # :339-341
        pred_original_sample = (sample - beta_prod_t ** (0.5) * model_output) / alpha_prod_t ** (0.5)
        pred_epsilon = model_output
    elif prediction_type == "sample":                                                                    # :342-344
        pred_original_sample = model_output
        pred_epsilon = (sample - alpha_prod_t ** (0.5) * pred_original_sample) / beta_prod_t ** (0.5)
    elif prediction_type == "v_prediction":                                                              # :345-347
        pred_original_sample = (alpha_prod_t ** 0.5) * sample - (beta_prod_t ** 0.5) * model_output
        pred_epsilon = (alpha_prod_t ** 0.5) * model_output + (beta_prod_t ** 0.5) * sample
    else:
        raise ValueError(prediction_type)
    if clip_sample_range is not None:                                                                    # :357-360
        pred_original_sample = pred_original_sample.clamp(-clip_sample_range, clip_sample_range)
    variance = get_variance(alpha_prod_t, alpha_prod_t_prev)                                             # :364
    std_dev_t = eta * variance ** (0.5)                                                                  # :365
    if use_clipped_model_output:                                                                         # :367-369
        pred_epsilon = (sample - alpha_prod_t ** (0.5) * pred_original_sample) / beta_prod_t ** (0.5)
    if score is not None and guidance_scale > 0.0:                                                       # :375-382
        pred_epsilon = pred_epsilon - guidance_scale * (1 - alpha_prod_t) ** (0.5) * score
    pred_sample_direction = (1 - alpha_prod_t_prev - std_dev_t ** 2) ** (0.5) * pred_epsilon            # :386
    prev_sample = alpha_prod_t_prev ** (0.5) * pred_original_sample + pred_sample_direction              # :389
    if eta > 0:                                                                                          # :391-404
        prev_sample = prev_sample + std_dev_t * variance_noise
    return prev_sample, pred_original_sample


def ddim_step_fp16_sequence(eps_cond: Tensor, eps_uncond: Optional[Tensor], x: Tensor, score: Optional[Tensor],
                            cfg_scale: float, a_t: Tensor, a_prev: Tensor, guidance_scale: float = 1.0, *,
                            prediction_type: str = "epsilon", clip_sample_range: Optional[float] = None,
                            use_clipped_model_output: bool = False, eta: float = 0.0,
                            variance_noise: Optional[Tensor] = None):
    """What the reference's eager CUDA ops compute for fp16 tensors at :239 + :339-404, on fp32 values with an explicit
    fp16 rounding h() after every op (mc_oracle.cfg_ddim_step_fp16_sequence for every branch): 0-dim fp32 CPU operands
    stay fp32, `tensor / cpu_scalar` multiplies by the fp32 reciprocal, clamp compares in fp32 against fp32 limits.
    Returns (prev_sample, pred_original_sample) as fp16."""
    h = lambda t: t.to(torch.float16).to(torch.float32)  # noqa: E731
    a_t = a_t.to(torch.float32).cpu()
    a_prev = a_prev.to(torch.float32).cpu()
    sa, sb = a_t ** 0.5, (1 - a_t) ** 0.5
    inv_sa, inv_sb = 1.0 / sa, 1.0 / sb
    std = eta * get_variance(a_t, a_prev) ** 0.5
    sap, c = a_prev ** 0.5, (1 - a_prev - std ** 2) ** 0.5
    e, xf = eps_cond.float(), x.float()
    if eps_uncond is not None:
        e = h(e + h(cfg_scale * h(e - eps_uncond.float())))
    if prediction_type == "epsilon":
        x0, pe = h(h(xf - h(sb * e)) * inv_sa), e
    elif prediction_type == "sample":
        x0, pe = e, h(h(xf - h(sa * e)) * inv_sb)
    else:
        x0, pe = h(h(sa * xf) - h(sb * e)), h(h(sa * e) + h(sb * xf))
    if clip_sample_range is not None:
        r = torch.tensor(clip_sample_range, dtype=torch.float32)
        x0 = h(torch.clamp(x0, -r, r))
    if use_clipped_model_output:
        pe = h(h(xf - h(sa * x0)) * inv_sb)
    if score is not None and guidance_scale > 0.0:
        pe = h(pe - h((guidance_scale * (1 - a_t) ** 0.5) * score.float()))
    xp = h(h(sap * x0) + h(c * pe))
    if eta > 0:
        xp = h(xp + h(std * variance_noise.float()))
    return xp.to(torch.float16), x0.to(torch.float16)


@contextmanager
def scheduler_step(step_kwargs: dict, eta: float, noises: Optional[Sequence[Tensor]]):
    """While active, mc_oracle's sampling loop takes its scheduler step from `ddim_step` with the given configuration;
    step i of the loop reads `noises[i]` (the variance noise the reference drew at that step)."""
    plain, calls = O.ddim_guided_step, iter(range(10 ** 9))

    def step(eps, x, score, a_t, a_prev, guidance_scale=1.0, reciprocal_div=False):
        i = next(calls)
        nz = None if not eta > 0 else noises[i].to(device=x.device, dtype=x.dtype)
        return ddim_step(eps, x, score, a_t, a_prev, guidance_scale, eta=eta, variance_noise=nz, **step_kwargs)[0]

    O.ddim_guided_step = step
    try:
        yield
    finally:
        O.ddim_guided_step = plain


def step_kwargs_of(scheduler_kwargs: dict) -> dict:
    """DDIMScheduler configuration (noise_scheduler_kwargs) -> the keyword arguments of `ddim_step`."""
    return dict(prediction_type=scheduler_kwargs.get("prediction_type", "epsilon"),
                clip_sample_range=scheduler_kwargs.get("clip_sample_range", 1.0)
                if scheduler_kwargs.get("clip_sample", True) else None)


def sample_loop(sd, cfg, icfg: dict, latents: Tensor, text: Tensor, representation, scheduler_kwargs: dict,
                eta: float = 0.0, noises: Optional[Sequence[Tensor]] = None, **kw) -> List[Tensor]:
    """mc_oracle.sample_loop (:102-171) under a scheduler configuration, eta and per-step variance noise."""
    with scheduler_step(step_kwargs_of(scheduler_kwargs), eta, noises):
        return O.sample_loop(sd, cfg, icfg, latents, text, representation, **kw)
