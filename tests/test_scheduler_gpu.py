"""The whole scheduler step on the GPU (utils/motionclone_functions.py:285-409; csrc/elementwise.cu, mc_ddim_step_ex):
every variant of the fused kernel bit for bit against the reference's eager op sequence on the same device and against
the CPU statement of its fp16 roundings (oracle/scheduler_oracle.py), the C-ABI contract, batch invariance of the noise,
and the sampling loop end to end on fixtures written by the unmodified reference
(tests/golden/ref_tiny8_{eta,vpred,clip}.npz)."""
import ctypes
import itertools
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from motionclone_b200 import _lib  # noqa: E402
from motionclone_b200.guidance import (schedule_customized_step, schedule_customized_step_fused,  # noqa: E402
                                       schedule_set_timesteps)
from motionclone_b200.pipeline import DDIMScheduler  # noqa: E402
from motionclone_b200.synthetic import NOISE_SCHEDULER_KWARGS, UNET_TINY_CONFIG, synthetic_inputs  # noqa: E402
from oracle import mc_oracle as O  # noqa: E402
from oracle import scheduler_oracle as S  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
CLIP_RANGE = 1.0
STEPS = (0, 13, 24, 25, 48, 49)  # first, guided, boundary, plain, last (alpha_prev = 1: std_dev_t = 0)


def _ops():
    from motionclone_b200 import ops
    return ops


def _dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def _inputs(shape, dev, seed=1):
    """eps_cond, eps_uncond, x, score, noise in fp16. x mixes O(1) values, latents at the largest magnitude the loop
    reaches (~1e2, DESIGN.md §2) and zeros; eps_cond starts with the clamp bounds and their fp16 neighbours (with the
    `sample` prediction type and no eps_uncond, eps_cond IS x0, so these meet the clamp exactly) and zeros."""
    g = torch.Generator().manual_seed(seed)
    ec, eu, x, sc, nz = (torch.randn(shape, generator=g) for _ in range(5))
    n = x.numel()
    xf = x.view(-1)
    xf[n // 3: 2 * n // 3] *= 100.0
    xf[:: 17] = 0.0
    edge = torch.tensor([CLIP_RANGE, -CLIP_RANGE, 0.0, -0.0], dtype=torch.float16)
    up = (edge[:2].view(torch.int16) + 1).view(torch.float16)    # one fp16 step outside +-range
    down = (edge[:2].view(torch.int16) - 1).view(torch.float16)  # one fp16 step inside
    special = torch.cat([edge, up, down]).float()
    ec.view(-1)[: special.numel()] = special
    return tuple(t.to(dev, torch.float16) for t in (ec, eu, x, sc * 0.05, nz))


def _check_variant(shape, pred, clip, rederive, with_score, eta, with_uncond, steps, dev, cpu_statement=True):
    ops = _ops()
    ec, eu, x, sc, nz = _inputs(shape, dev)
    acp = O.alphas_cumprod()
    timesteps = O.uneven_timesteps(50, 25, 0.3)
    kw = dict(prediction_type=pred, clip_sample_range=CLIP_RANGE if clip else None, use_clipped_model_output=rederive,
              eta=eta)
    what = f"{pred} clip={clip} rederive={rederive} score={with_score} eta={eta} uncond={with_uncond}"
    for step in steps:
        a_t, a_prev = O.ddim_scalars(acp, timesteps, step)
        score = sc if with_score else None
        noise = nz if eta > 0 else None
        got, got_x0 = ops.ddim_step(ec, eu if with_uncond else None, x, score, 7.5, a_t, a_prev, noise=noise,
                                    want_pred_x0=True, **kw)
        only = ops.ddim_step(ec, eu if with_uncond else None, x, score, 7.5, a_t, a_prev, noise=noise, **kw)
        assert only[1] is None and torch.equal(only[0], got), f"{what} step {step}: the x0 store changed x_prev"
        # the reference's statements (:239, :339-404) executed by ATen on the same device
        eps = O.cfg_combine(ec, eu, 7.5) if with_uncond else ec
        want, want_x0 = S.ddim_step(eps, x, score, a_t, a_prev, variance_noise=noise, **kw)
        assert torch.isfinite(want).all()
        assert torch.equal(got, want), f"{what} step {step}: x_prev differs from the eager CUDA op sequence"  # bitwise
        assert torch.equal(got_x0, want_x0), f"{what} step {step}: pred_original_sample differs from eager"  # bitwise
        if cpu_statement:  # and the explicit CPU statement of that rounding sequence
            c = lambda t: None if t is None else t.cpu()  # noqa: E731
            cpu, cpu_x0 = S.ddim_step_fp16_sequence(c(ec), c(eu) if with_uncond else None, c(x), c(score), 7.5, a_t,
                                                    a_prev, variance_noise=c(noise), **kw)
            assert torch.equal(got.cpu(), cpu), f"{what} step {step}: x_prev differs from the CPU statement"  # bitwise
            assert torch.equal(got_x0.cpu(), cpu_x0), f"{what} step {step}: x0 differs from the CPU statement"  # bitwise


@pytest.mark.parametrize("pred", ["epsilon", "sample", "v_prediction"])
@pytest.mark.parametrize("clip", [False, True])
@pytest.mark.parametrize("rederive", [False, True])
def test_ddim_step_variants_bit_exact(pred, clip, rederive):
    """3 prediction types x clip x re-derive, each with / without score, eta in {0, 0.3, 1.0}, with / without
    eps_uncond, at six schedule positions; 1 155 elements (not a multiple of the 8-wide vectors: the tail path runs)."""
    dev = _dev()
    for with_score, eta, with_uncond in itertools.product((False, True), (0.0, 0.3, 1.0), (False, True)):
        _check_variant((1, 3, 5, 7, 11), pred, clip, rederive, with_score, eta, with_uncond, STEPS, dev)


@pytest.mark.parametrize("pred", ["epsilon", "sample", "v_prediction"])
@pytest.mark.parametrize("batch", [1, 4])
def test_ddim_step_full_size_bit_exact(pred, batch):
    """[B, 4, 16, 64, 64] (the 16 x 512 x 512 sample of BASELINE.json configs[1]): everything on, and everything off."""
    dev = _dev()
    _check_variant((batch, 4, 16, 64, 64), pred, True, True, True, 0.3, True, (13, 49), dev)
    _check_variant((batch, 4, 16, 64, 64), pred, False, False, False, 0.0, True, (25,), dev, cpu_statement=False)


@pytest.mark.parametrize("with_score,with_uncond", [(False, True), (True, True), (True, False)])
def test_default_variant_equals_cfg_ddim_step(with_score, with_uncond):
    """epsilon, no clip, no re-derive, no noise through mc_ddim_step_ex is mc_cfg_ddim_step's kernel: bitwise equal."""
    ops, dev = _ops(), _dev()
    acp, timesteps = O.alphas_cumprod(), O.uneven_timesteps(50, 25, 0.3)
    for shape in ((1, 4, 16, 64, 64), (1, 3, 5, 7, 11)):
        ec, eu, x, sc, _ = _inputs(shape, dev, seed=2)
        for step in STEPS:
            a_t, a_prev = O.ddim_scalars(acp, timesteps, step)
            args = (ec, eu if with_uncond else None, x, sc if with_score else None, 7.5, a_t, a_prev)
            assert torch.equal(ops.ddim_step(*args)[0], ops.cfg_ddim_step(*args))  # bitwise


def _call_ex(lib, ec, x, out, n, *, noise=None, x0=None, pred=0, flags=0, clip=0.0, std=0.0):
    p = lambda t: ctypes.c_void_p(0 if t is None else t.data_ptr())  # noqa: E731
    return lib.mc_ddim_step_ex(p(ec), p(None), p(x), p(None), p(noise), p(out), p(x0), n, pred, flags, 7.5, 0.5, 1.2, 0.9,
                               0.4, 0.5, 0.8, 2.0, clip, std, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))


def test_c_abi_contract():
    """Rejected calls return their code before any launch (launch counter unchanged, output untouched); accepted calls
    store exactly n elements of x_prev and pred_x0."""
    dev, lib = _dev(), _lib.lib()
    n, pad = 1003, 64  # n % 8 != 0
    ec, x, nz = (torch.randn(n + pad, device=dev).half() for _ in range(3))
    canary = 1234.0
    out = torch.full((n + pad,), canary, device=dev, dtype=torch.float16)
    x0 = torch.full((n + pad,), canary, device=dev, dtype=torch.float16)
    torch.cuda.synchronize()
    count = _lib.launch_count()
    rejected = [
        (dict(pred=3), -2), (dict(pred=-1), -2),            # MC_E_UNSUPPORTED: prediction type outside the three
        (dict(flags=4), -2), (dict(flags=-1), -2),          # MC_E_UNSUPPORTED: unknown flag bits
        (dict(std=0.1), -1),                                # MC_E_INVALID: std_dev != 0 with noise == NULL
        (dict(flags=1, clip=-1.0), -1), (dict(flags=1, clip=float("nan")), -1),  # MC_E_INVALID: clip range
    ]
    for kw, code in rejected:
        assert _call_ex(lib, ec, x, out, n, x0=x0, **kw) == code, kw
        assert lib.mc_last_error()
    assert _call_ex(lib, ec[1:], x, out, n) == -1  # MC_E_INVALID: 2-byte offset, not 16-byte aligned
    assert _call_ex(lib, ec, x, out, 0) == -1 and _call_ex(lib, None, x, out, n) == -1
    torch.cuda.synchronize()
    assert _lib.launch_count() == count  # nothing was launched
    assert bool((out == canary).all()) and bool((x0 == canary).all())
    for kw in (dict(), dict(noise=nz, std=0.1), dict(pred=2, flags=3, clip=1.0, noise=nz, std=0.1), dict(pred=1, flags=1, clip=0.5)):
        out.fill_(canary), x0.fill_(canary)
        assert _call_ex(lib, ec, x, out, n, x0=x0, **kw) == 0, kw
        torch.cuda.synchronize()
        for t in (out, x0):
            assert bool((t[n:] == canary).all()), f"{kw}: stored past n"
            assert torch.isfinite(t[:n]).all() and not bool((t[:n] == canary).any()), f"{kw}: elements below n not written"
    assert _lib.launch_count() == count + 4
    with pytest.raises(NotImplementedError):  # the Python binding maps MC_E_UNSUPPORTED as everywhere else
        _lib.check(_call_ex(lib, ec, x, out, n, pred=7), "mc_ddim_step_ex")


def _scheduler(dev, **kw):
    s = DDIMScheduler(**dict(NOISE_SCHEDULER_KWARGS, **kw))
    s.customized_set_timesteps = schedule_set_timesteps.__get__(s)
    s.customized_step = schedule_customized_step.__get__(s)
    s.customized_step_fused = schedule_customized_step_fused.__get__(s)
    s.customized_set_timesteps(50, 25, 0.3, device=dev)
    return s


@pytest.mark.parametrize("gen_device", ["cuda", "cpu"])
@pytest.mark.parametrize("skw", [dict(), dict(prediction_type="v_prediction", clip_sample=True)])
def test_step_batch_invariance(gen_device, skw):
    """B = 3 with three generators equals the three B = 1 calls bit for bit, for generators on either device: sample s of
    the batch gets the noise its own generator gives alone, and the kernel is elementwise."""
    dev = _dev()
    s = _scheduler(dev, **skw)
    ec, eu, x, sc, _ = _inputs((3, 4, 8, 16, 16), dev, seed=3)
    gens = lambda: [torch.Generator(device=gen_device).manual_seed(100 + i) for i in range(3)]  # noqa: E731
    for step in (3, 30, 49):
        score = sc if step < 25 else None
        n0 = _lib.launch_count()
        batch = s.customized_step_fused(ec, eu, 7.5, step, x, score=score, eta=0.5, generator=gens())
        assert _lib.launch_count() == n0 + 1  # CFG combine + step of the whole batch: one launch
        alone = [s.customized_step_fused(ec[i:i + 1], eu[i:i + 1], 7.5, step, x[i:i + 1],
                                         score=None if score is None else score[i:i + 1], eta=0.5, generator=g)
                 for i, g in enumerate(gens())]
        assert torch.equal(batch, torch.cat(alone))  # bitwise
        plain = s.customized_step_fused(ec, eu, 7.5, step, x, score=score, eta=0.0, generator=gens())
        assert (step == 49) == torch.equal(plain, batch)  # the noise is really added, except where std_dev_t = 0


def test_step_eta_zero_leaves_generator_untouched_and_tuple():
    dev = _dev()
    ec, _, x, sc, nz = _inputs((1, 4, 8, 16, 16), dev, seed=4)
    for gen_device in ("cuda", "cpu"):
        g = torch.Generator(device=gen_device).manual_seed(9)
        state = g.get_state()
        prev, x0, a_prev = _scheduler(dev).customized_step(ec, 5, x, eta=0.0, generator=g, score=sc)
        assert torch.equal(g.get_state(), state)
        assert x0 is None and float(a_prev) == float(O.ddim_scalars(O.alphas_cumprod(), O.uneven_timesteps(50, 25, 0.3), 5)[1])
        prev2, x02, _ = _scheduler(dev).customized_step(ec, 5, x, eta=0.5, generator=g, score=sc)
        assert not torch.equal(g.get_state(), state) and x02 is not None and not torch.equal(prev, prev2)
    s = _scheduler(dev, clip_sample=True, clip_sample_range=0.75)
    prev, x0, _ = s.customized_step(ec, 5, x, variance_noise=nz, eta=1.0, use_clipped_model_output=True)
    assert x0.abs().max().item() == 0.75  # pred_original_sample is the clipped x0
    assert torch.equal(s.customized_step(ec, 5, x, variance_noise=nz, eta=1.0, use_clipped_model_output=True,
                                         return_dict=False)[0], prev)


# ---------------------------------------------------------------------------------------------------------------
# end to end on the reference's runs
# ---------------------------------------------------------------------------------------------------------------
def _rel(a, b):
    a, b = a.float().cpu(), torch.as_tensor(b).float()
    return ((a - b).abs().max() / (b.abs().max() + 1e-12)).item()


def _pipeline(case, dev, **kw):
    import motionclone_b200 as mc
    g = np.load(os.path.join(GOLDEN, f"ref_{case}.npz"))
    meta = json.loads(str(g["meta"]))
    icfg = dict(meta["infer"])
    inp = synthetic_inputs(icfg["video_length"], icfg["height"], icfg["width"], UNET_TINY_CONFIG["cross_attention_dim"],
                           meta["input_seed"])
    icfg.update(video_latents=inp["clip_latents"].half(), video_noise=inp["clip_noise"].half(), new_prompt="synthetic")
    pipe = mc.build_pipeline(UNET_TINY_CONFIG, icfg, device=dev, weight_seed=meta["weight_seed"],
                             scheduler_kwargs=meta["scheduler_kwargs"], **kw)
    pipe.set_prompt_embeds(inp["text_embeddings"].to(dev, torch.float16))
    pipe.motion_representation_dict = {str(n): [torch.from_numpy(g[f"repr_val_{i}"]).half(),
                                                torch.from_numpy(g[f"repr_idx_{i}"])]
                                       for i, n in enumerate(g["repr_names"])}
    return pipe, g, meta, inp


@pytest.mark.parametrize("case", ["tiny8_eta", "tiny8_vpred", "tiny8_clip"])
def test_sampling_loop_vs_reference(case):
    """sample_video under the case's scheduler configuration and eta, on the reference's motion representation, each
    step fed the variance noise the reference drew at that step (extra_step_kwargs["variance_noise"])."""
    dev = _dev()
    pipe, g, meta, inp = _pipeline(case, dev)
    per_step = []
    step = pipe.single_step_video

    def rec(lat, i, t, extra):
        if meta["eta"] > 0:
            extra = dict(extra, variance_noise=torch.from_numpy(g["variance_noise"][i]).to(dev, torch.float16))
        per_step.append(step(lat, i, t, extra))
        return per_step[-1]

    pipe.single_step_video = rec
    final = pipe.sample_video(eta=meta["eta"], noisy_latents=inp["noisy_latents"].to(dev, torch.float16),
                              return_latents=True)
    ref = g["latents_per_step"]
    rels = [_rel(p, ref[i]) for i, p in enumerate(per_step)]
    print(case, "per-step latent rel err vs reference fp32:", rels)
    assert len(per_step) == len(ref) and torch.isfinite(final).all()
    assert rels[0] < 1.5e-2  # one step: fp16 UNet vs fp32 (the bar of test_pipeline_gpu.py)
    if case != "tiny8_clip":
        assert rels[-1] < 5e-2   # final latents, relative to max |x| (the bar of test_pipeline_gpu.py)
        return
    # clip_sample with range 1 on this random-init UNet saturates: from the third step on nearly every x0 is +-1 by the
    # sign of a value amplified by 1 / sqrt(a_t), so an fp16-sized difference moves single elements from -1 to +1 and a
    # max-error bar says nothing (measured on an H100: 1.3e-2, 2.9e-2, 5.6e-2, 0.26, 1.3, 1.4). What holds: the second step
    # within 5 % of max |x|, and the last step (alpha_prev = 1, so x_prev = h(clamp(x0))) inside the range exactly. The
    # clamp's arithmetic itself is pinned bit for bit in test_ddim_step_variants_bit_exact and test_direct_step_vs_reference.
    assert rels[1] < 5e-2
    assert final.abs().max().item() <= CLIP_RANGE


@pytest.mark.parametrize("case", ["tiny8_eta", "tiny8_vpred", "tiny8_clip"])
def test_direct_step_vs_reference(case):
    """customized_step(use_clipped_model_output=True, eta=0.3, variance_noise, score) as the reference ran it in fp32."""
    dev = _dev()
    g = np.load(os.path.join(GOLDEN, f"ref_{case}.npz"))
    meta = json.loads(str(g["meta"]))
    d, icfg = meta["direct"], meta["infer"]
    s = DDIMScheduler(**dict(NOISE_SCHEDULER_KWARGS, **meta["scheduler_kwargs"]))
    schedule_set_timesteps(s, icfg["inference_steps"], icfg["guidance_steps"], icfg["guidance_scale"], device=dev)
    h = lambda k: torch.from_numpy(g[k]).to(dev, torch.float16)  # noqa: E731
    prev, x0, a_prev = schedule_customized_step(
        s, h("direct_model_output"), d["step_index"], h("direct_sample"), eta=d["eta"], variance_noise=h("direct_noise"),
        score=h("direct_score"), use_clipped_model_output=d["use_clipped_model_output"], guidance_scale=d["guidance_scale"])
    r_prev, r_x0 = _rel(prev, g["direct_prev_sample"]), _rel(x0, g["direct_pred_original_sample"])
    print(case, "direct step rel err vs reference fp32: x_prev", r_prev, "x0", r_x0)
    # fp16 inputs against fp32 ones: x0 = (x - sb*e) / sqrt(a_t) multiplies half an fp16 spacing of |x| ~ 4 (1e-3) by
    # 1 / sqrt(a_850) ~ 7; in the clip case that is measured against max |x0| = 1: 2 % of the largest value
    assert r_prev < 2e-2 and r_x0 < 2e-2
    c = lambda k: h(k).cpu()  # noqa: E731
    cpu, cpu_x0 = S.ddim_step_fp16_sequence(
        c("direct_model_output"), None, c("direct_sample"), c("direct_score"), 0.0, *O.ddim_scalars(
            O.alphas_cumprod(), s.timesteps_host, d["step_index"]), d["guidance_scale"], eta=d["eta"],
        variance_noise=c("direct_noise"), use_clipped_model_output=True,
        **S.step_kwargs_of(dict(NOISE_SCHEDULER_KWARGS, **meta["scheduler_kwargs"])))
    assert torch.equal(prev.cpu(), cpu) and torch.equal(x0.cpu(), cpu_x0)  # bitwise: the CPU statement of the roundings
    assert float(a_prev) == float(g["direct_alpha_prod_t_prev"])


def test_sample_video_eta_reproducible_and_graph_invariant():
    """sample_video(eta=0.5, generator=g): the same seed gives the same latents bit for bit, with CUDA graphs on and off
    (the scheduler step and its noise draw are outside the captured UNet forwards), for generators on either device."""
    dev = _dev()
    outs = {}
    for graphs in (False, True):
        pipe, g, meta, inp = _pipeline("tiny8_eta", dev, use_cuda_graphs=graphs)
        x = inp["noisy_latents"].to(dev, torch.float16)
        for gen_device in ("cuda", "cpu"):
            runs = [pipe.sample_video(eta=0.5, generator=torch.Generator(device=gen_device).manual_seed(77),
                                      noisy_latents=x, return_latents=True).clone() for _ in range(2)]
            assert torch.equal(runs[0], runs[1])  # bitwise
            outs[graphs, gen_device] = runs[0]
        other = pipe.sample_video(eta=0.5, generator=torch.Generator(device="cuda").manual_seed(78), noisy_latents=x,
                                  return_latents=True)
        assert not torch.equal(other, outs[graphs, "cuda"])  # the seed matters
        assert not torch.equal(pipe.sample_video(eta=0.0, noisy_latents=x, return_latents=True), outs[graphs, "cuda"])
    for gen_device in ("cuda", "cpu"):
        assert torch.equal(outs[False, gen_device], outs[True, gen_device])  # bitwise


def test_sample_video_batch_noise_per_generator(monkeypatch):
    """B = 2 with a list of generators: every step is ONE fused launch over the whole batch, and sample s reads the noise
    its own generator gives in a B = 1 run."""
    dev, ops = _dev(), _ops()
    pipe, g, meta, inp = _pipeline("tiny8_eta", dev)
    x = inp["noisy_latents"].to(dev, torch.float16)
    pipe.set_prompt_embeds(pipe.prompt_embeds.repeat_interleave(2, dim=0))  # [u, u, c, c]
    calls = []
    fused = ops.ddim_step

    def spy(*a, **k):
        n0 = _lib.launch_count()
        out = fused(*a, **k)
        calls.append((k["noise"].clone(), _lib.launch_count() - n0))
        return out

    monkeypatch.setattr(ops, "ddim_step", spy)
    gens = [torch.Generator(device="cuda").manual_seed(s) for s in (5, 6)]
    out = pipe.sample_video(eta=0.5, generator=gens, noisy_latents=torch.cat([x, x]), return_latents=True)
    assert out.shape[0] == 2 and torch.isfinite(out).all()
    assert len(calls) == meta["infer"]["inference_steps"] and all(n == 1 for _, n in calls)
    alone = [torch.Generator(device="cuda").manual_seed(s) for s in (5, 6)]
    for noise, _ in calls:
        for i, ga in enumerate(alone):
            assert torch.equal(noise[i:i + 1], torch.randn(x.shape, generator=ga, device=dev, dtype=torch.float16))
