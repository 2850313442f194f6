"""The whole scheduler step (utils/motionclone_functions.py:285-409: eta > 0, sample / v prediction, x0 clipping,
use_clipped_model_output) without a device: the oracle restatement (oracle/scheduler_oracle.py) against runs of the
UNMODIFIED reference (tests/golden/ref_tiny8_{eta,vpred,clip}.npz, scripts/gen_golden_scheduler.py), the host scalars,
and the argument contract of the bound step. No kernel is launched here."""
import json
import math
import os

import numpy as np
import pytest
import torch

from motionclone_b200 import ops
from motionclone_b200.guidance import (randn_tensor, schedule_customized_step, schedule_customized_step_fused,
                                       schedule_set_timesteps)
from motionclone_b200.pipeline import DDIMScheduler
from motionclone_b200.synthetic import NOISE_SCHEDULER_KWARGS, UNET_TINY_CONFIG, synthetic_inputs, synthetic_state_dict
from oracle import mc_oracle as O
from oracle import scheduler_oracle as S

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
CASES = ["tiny8_eta", "tiny8_vpred", "tiny8_clip"]


def _case(case):
    g = np.load(os.path.join(GOLDEN, f"ref_{case}.npz"))
    meta = json.loads(str(g["meta"]))
    shapes = json.load(open(os.path.join(GOLDEN, "ref_state_dict_shapes_tiny.json")))
    sd = synthetic_state_dict(shapes, meta["weight_seed"])
    icfg = meta["infer"]
    inp = synthetic_inputs(icfg["video_length"], icfg["height"], icfg["width"], UNET_TINY_CONFIG["cross_attention_dim"],
                           meta["input_seed"])
    return g, meta, sd, icfg, inp


def _rel(a, b):
    b = torch.as_tensor(b)
    return (a - b).abs().max().item() / (b.abs().max().item() + 1e-12)


@pytest.mark.parametrize("case", CASES)
def test_oracle_sampling_loop_vs_reference(case):
    g, meta, sd, icfg, inp = _case(case)
    rep = {str(n): [torch.from_numpy(g[f"repr_val_{i}"]), torch.from_numpy(g[f"repr_idx_{i}"])]
           for i, n in enumerate(g["repr_names"])}
    skw = dict(NOISE_SCHEDULER_KWARGS, **meta["scheduler_kwargs"])
    noises = torch.from_numpy(g["variance_noise"]) if meta["eta"] > 0 else None
    assert (noises is not None) == (case == "tiny8_eta")
    ref = g["latents_per_step"]
    if case == "tiny8_clip":
        # clip_sample with range 1 saturates on this random-init UNet and the loop then amplifies a difference several
        # times per step, so the last-bit differences between two CPUs' convolutions would outgrow 1e-5 within four steps:
        # each step starts from the reference's own previous latents instead (step 0, guided, boundary, first plain)
        ts = O.uneven_timesteps(icfg["inference_steps"], icfg["guidance_steps"], icfg["guidance_scale"])
        steps, prev = [], inp["noisy_latents"]
        with S.scheduler_step(S.step_kwargs_of(skw), 0.0, None):
            for i in range(4):
                steps.append(O.single_step(sd, UNET_TINY_CONFIG, icfg, prev, i, ts, O.alphas_cumprod(),
                                           inp["text_embeddings"], rep))
                prev = torch.from_numpy(ref[i])
    else:
        # the eta case runs to the last step (alpha_prev = 1: std_dev_t = 0); v_prediction covers guided, boundary, first plain
        steps = S.sample_loop(sd, UNET_TINY_CONFIG, icfg, inp["noisy_latents"], inp["text_embeddings"], rep, skw,
                              eta=meta["eta"], noises=noises, max_steps=icfg["inference_steps"] if noises is not None else 4)
    rels = [_rel(s, ref[i]) for i, s in enumerate(steps)]
    print(case, "oracle vs reference, per step:", rels, "bitwise:", [torch.equal(s, torch.from_numpy(ref[i]))
                                                                      for i, s in enumerate(steps)])
    # fp32 CPU vs fp32 CPU, op for op: the bar of test_oracle_golden.py (bitwise on the CPU the fixtures were written on; up
    # to 4.4e-6 on another x86 CPU, whose convolutions round differently). The clipped run's latents stay within +-3.4, a
    # third to a thirtieth of the other runs', so the same absolute difference is a larger share of max |x| (1.6e-5 there):
    # 1e-4, the bar test_oracle_golden.py uses for its SparseCtrl cases
    assert max(rels) <= (1e-4 if case == "tiny8_clip" else 1e-5)
    if case == "tiny8_clip":  # every x0 of this run is clipped somewhere: the branch is live
        assert np.abs(ref[-1]).max() < np.abs(np.load(os.path.join(GOLDEN, "ref_tiny8.npz"))["latents_per_step"][-1]).max()


@pytest.mark.parametrize("case", CASES)
def test_oracle_direct_step_vs_reference(case):
    """customized_step(..., use_clipped_model_output=True, eta=0.3, variance_noise=..., score=...) as the reference ran
    it under each case's scheduler configuration."""
    g = np.load(os.path.join(GOLDEN, f"ref_{case}.npz"))
    meta = json.loads(str(g["meta"]))
    d, icfg = meta["direct"], meta["infer"]
    skw = dict(NOISE_SCHEDULER_KWARGS, **meta["scheduler_kwargs"])
    ts = O.uneven_timesteps(icfg["inference_steps"], icfg["guidance_steps"], icfg["guidance_scale"])
    a_t, a_prev = O.ddim_scalars(O.alphas_cumprod(), ts, d["step_index"])
    t = lambda k: torch.from_numpy(g[k])  # noqa: E731
    prev, x0 = S.ddim_step(t("direct_model_output"), t("direct_sample"), t("direct_score"), a_t, a_prev,
                           d["guidance_scale"], eta=d["eta"], variance_noise=t("direct_noise"),
                           use_clipped_model_output=d["use_clipped_model_output"], **S.step_kwargs_of(skw))
    print(case, "direct step bitwise:", torch.equal(prev, t("direct_prev_sample")),
          torch.equal(x0, t("direct_pred_original_sample")))
    assert _rel(prev, t("direct_prev_sample")) <= 1e-5 and _rel(x0, t("direct_pred_original_sample")) <= 1e-5  # as above
    assert float(g["direct_alpha_prod_t_prev"]) == float(a_prev)
    if skw["clip_sample"]:
        assert x0.abs().max().item() == skw["clip_sample_range"]  # the clamp is hit exactly


def _scheduler(steps=10, guided=5, gs=0.3, **kw):
    s = DDIMScheduler(**dict(NOISE_SCHEDULER_KWARGS, **kw))
    s.customized_set_timesteps = schedule_set_timesteps.__get__(s)
    s.customized_step = schedule_customized_step.__get__(s)
    s.customized_step_fused = schedule_customized_step_fused.__get__(s)
    s.customized_set_timesteps(steps, guided, gs, device="cpu")
    return s


def test_host_scalars_closed_form():
    s = _scheduler()
    ts = [int(t) for t in s.timesteps_host]
    assert ts == [999, 924, 850, 775, 700, 699, 524, 350, 175, 0]  # the c1 schedule (BASELINE.json configs[0])
    acp = s.alphas_cumprod.double()
    for i, t in enumerate(ts):
        prev_t = ts[i + 1] if i + 1 < len(ts) else -1
        a_t, a_p = acp[t].item(), (acp[prev_t].item() if prev_t >= 0 else 1.0)
        var = (1 - a_p) / (1 - a_t) * (1 - a_t / a_p)
        got = s._get_variance(t, prev_t)
        assert got.dtype == torch.float32 and abs(got.item() - var) <= 1e-5 * var + 1e-9  # fp32 against float64
        assert torch.equal(got, S.get_variance(s.alphas_cumprod[t], s.alphas_cumprod[prev_t] if prev_t >= 0
                                               else s.final_alpha_cumprod))
        for eta in (0.0, 0.3, 1.0):
            std = ops.ddim_std_dev(s.alphas_cumprod[t], s.alphas_cumprod[prev_t] if prev_t >= 0 else s.final_alpha_cumprod,
                                   eta)
            assert abs(std.item() - eta * math.sqrt(var)) <= 1e-5  # fp32 against float64
            direction = (1 - a_p - (eta ** 2) * var)
            assert direction >= -1e-7  # sigma_t^2 <= 1 - alpha_prev for every eta in [0, 1] (DDIM eq. 16)
            if prev_t < 0:  # last step: alpha_prev = 1, variance 0, so the noise term is 0 whatever eta is
                assert std.item() == 0.0 and got.item() == 0.0


def test_randn_tensor_batch_rule():
    """A list of B generators draws one [1, ...] tensor per sample: sample s gets what its generator gives alone."""
    shape = (3, 4, 2, 8, 8)
    batch = randn_tensor(shape, [torch.Generator().manual_seed(s) for s in (5, 6, 7)], "cpu", torch.float32)
    for i, s in enumerate((5, 6, 7)):
        alone = randn_tensor((1,) + shape[1:], torch.Generator().manual_seed(s), "cpu", torch.float32)
        assert torch.equal(batch[i:i + 1], alone)
    with pytest.raises(ValueError):
        randn_tensor(shape, [torch.Generator().manual_seed(1)] * 2, "cpu", torch.float32)


def test_step_argument_contract():
    x = torch.randn(1, 4, 2, 8, 8).half()
    s = _scheduler()
    g = torch.Generator().manual_seed(3)
    with pytest.raises(ValueError, match="Cannot pass both generator and variance_noise"):
        s.customized_step(x, 0, x, eta=0.5, generator=g, variance_noise=x)
    with pytest.raises(ValueError, match="Cannot pass both generator and variance_noise"):
        s.customized_step_fused(x, x, 7.5, 0, x, eta=0.5, generator=g, variance_noise=x)
    for kw in (dict(indices=[0]), dict(return_middle=True)):
        with pytest.raises(NotImplementedError, match="indices|return_middle"):
            s.customized_step(x, 0, x, score=x, **kw)
    with pytest.raises(NotImplementedError, match="thresholding"):
        _scheduler(thresholding=True).customized_step(x, 0, x)
    learned = _scheduler()
    learned.variance_type = "learned_range"
    with pytest.raises(NotImplementedError, match="learned variance"):
        learned.customized_step(torch.cat([x, x], 1), 0, x)
    with pytest.raises(ValueError, match="prediction_type"):
        _scheduler(prediction_type="bogus").customized_step(x, 0, x)
    unset = DDIMScheduler(**NOISE_SCHEDULER_KWARGS)
    with pytest.raises(ValueError, match="set_timesteps"):
        schedule_customized_step(unset, x, 0, x)
    # eta = 0 draws nothing: the generator's state is untouched (the call then stops at the CPU tensors: no CPU path)
    state = g.get_state()
    for sched in (s, _scheduler(prediction_type="v_prediction", clip_sample=True)):
        with pytest.raises(TypeError):
            sched.customized_step(x, 0, x, eta=0.0, generator=g)
    assert torch.equal(g.get_state(), state)
    # eta > 0 draws exactly one tensor of the model output's shape from it
    with pytest.raises(TypeError):
        s.customized_step(x, 0, x, eta=0.5, generator=g)
    want = torch.Generator().manual_seed(3)
    torch.randn(x.shape, generator=want, dtype=x.dtype)
    assert torch.equal(g.get_state(), want.get_state())


def test_ops_ddim_step_argument_checks():
    x = torch.randn(1, 4, 2, 8, 8).half()
    acp = O.alphas_cumprod()
    with pytest.raises(ValueError, match="prediction_type"):
        ops.ddim_step(x, None, x, None, 0.0, acp[999], acp[900], prediction_type="bogus")
    with pytest.raises(ValueError, match="noise"):  # eta > 0 without noise is an error, not a silent eta = 0
        ops.ddim_step(x, None, x, None, 0.0, acp[999], acp[900], eta=0.5)
    with pytest.raises(ValueError, match="noise"):
        ops.ddim_step(x, None, x, None, 0.0, acp[999], acp[900], eta=0.0, noise=x)
    with pytest.raises(TypeError):  # no CPU path
        ops.ddim_step(x, None, x, None, 0.0, acp[999], acp[900], prediction_type="sample")
