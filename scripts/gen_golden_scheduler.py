"""Generates the scheduler-step fixtures tests/golden/ref_tiny8_{eta,vpred,clip}.npz by running the UNMODIFIED reference on
the CPU, through oracle/gen_golden.py's writer (same inputs, same checks: regenerating must reproduce every committed
tensor bit for bit). TEST INFRASTRUCTURE: needs the reference tree, like oracle/gen_golden.py.

  python scripts/gen_golden_scheduler.py [tiny8_eta tiny8_vpred tiny8_clip]

The cases are the branches of customized_step (utils/motionclone_functions.py:285-409) off the shipped configuration:
  tiny8_eta    sample_video(eta=0.5, generator=<CPU generator>): the stochastic step (:391-404);
  tiny8_vpred  noise_scheduler_kwargs prediction_type: v_prediction (:345-347);
  tiny8_clip   noise_scheduler_kwargs clip_sample: true, clip_sample_range: 1.0 (:357-360).
Every tensor the reference's randn_tensor returns during sampling is stored (`variance_noise`, one per step), so a
consumer replays the step with the reference's own noise. sample_video never passes use_clipped_model_output, so every
case also records one direct call of the bound customized_step with use_clipped_model_output=True, eta = 0.3, a score
and given variance noise (`direct_*` keys; return_dict=True, so pred_original_sample is recorded too).
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from motionclone_b200 import synthetic  # noqa: E402
from motionclone_b200.synthetic import synthetic_normal  # noqa: E402
from oracle import gen_golden, ref_runner  # noqa: E402
from oracle.gen_golden import BASE, ROOT  # noqa: E402

_TINY8 = dict(BASE, inference_steps=6, guidance_steps=3, guidance_scale=0.3, video_length=8, height=128, width=128)
CASES = {
    # name: (unet config name, inference cfg, input seed), as oracle/gen_golden.py's CASES
    "tiny8_eta": ("tiny", dict(_TINY8), 152),
    "tiny8_vpred": ("tiny", dict(_TINY8), 162),
    "tiny8_clip": ("tiny", dict(_TINY8), 172),
}
# what each case changes: sample_video's eta (+ the seed of its CPU generator) and the scheduler's configuration
VARIANTS = {
    "tiny8_eta": dict(eta=0.5, generator_seed=1234, scheduler_kwargs={}),
    "tiny8_vpred": dict(eta=0.0, generator_seed=None, scheduler_kwargs=dict(prediction_type="v_prediction")),
    "tiny8_clip": dict(eta=0.0, generator_seed=None, scheduler_kwargs=dict(clip_sample=True, clip_sample_range=1.0)),
}
DIRECT = dict(step_index=1, eta=0.3, use_clipped_model_output=True, guidance_scale=1.0)


def _direct_call(pipeline, shape, seed):
    """One customized_step call with use_clipped_model_output=True on seeded inputs of the latent shape."""
    model_output, sample, noise = (synthetic_normal(tag, shape, seed) for tag in ("direct_eps", "direct_x", "direct_noise"))
    score = 0.05 * synthetic_normal("direct_score", shape, seed)
    prev, x0, a_prev = pipeline.scheduler.customized_step(
        model_output, DIRECT["step_index"], sample, eta=DIRECT["eta"], variance_noise=noise, score=score,
        use_clipped_model_output=DIRECT["use_clipped_model_output"], guidance_scale=DIRECT["guidance_scale"])
    return dict(direct_model_output=model_output, direct_sample=sample, direct_score=score, direct_noise=noise,
                direct_prev_sample=prev, direct_pred_original_sample=x0, direct_alpha_prod_t_prev=a_prev)


def _runner(variant, seed):
    """oracle/ref_runner.run_reference with the case's scheduler configuration, eta and generator; the noise the reference
    draws while sampling and the direct call are added to what it returns."""
    def run(ucfg, icfg, inp, repr_path, **kw):
        drawn = []
        build = ref_runner.build_reference_pipeline
        shipped = synthetic.NOISE_SCHEDULER_KWARGS

        def build_hooked(*a, **k):
            pipeline, mf = build(*a, **k)
            from diffusers.utils.torch_utils import randn_tensor  # the reference's import (:12), importable from here on
            extract, sample = pipeline.obtain_motion_representation, pipeline.sample_video

            def record(*a, **k):
                t = randn_tensor(*a, **k)
                drawn.append(t.detach().float().cpu().clone())
                return t

            def extract_hooked(*a, **k):  # extraction runs on the preset clip noise; sampling draws from the generator
                r = extract(*a, **k)
                mf.randn_tensor = record
                return r

            def sample_hooked(**k):
                g = None if variant["generator_seed"] is None else torch.Generator().manual_seed(variant["generator_seed"])
                return sample(**dict(k, eta=variant["eta"], generator=g))

            pipeline.obtain_motion_representation, pipeline.sample_video = extract_hooked, sample_hooked
            return pipeline, mf

        ref_runner.build_reference_pipeline = build_hooked
        synthetic.NOISE_SCHEDULER_KWARGS = dict(shipped, **variant["scheduler_kwargs"])
        try:
            out, pipeline = ref_runner.run_reference(ucfg, icfg, inp, repr_path, **kw)
        finally:
            ref_runner.build_reference_pipeline = build
            synthetic.NOISE_SCHEDULER_KWARGS = shipped
        assert len(drawn) == (icfg["inference_steps"] if variant["eta"] > 0 else 0)
        if drawn:
            out["variance_noise"] = torch.stack(drawn)
        out.update({k: torch.as_tensor(v).detach().float().cpu()
                    for k, v in _direct_call(pipeline, tuple(inp["noisy_latents"].shape), seed).items()})
        return out, pipeline
    return run


if __name__ == "__main__":
    names = sys.argv[1:] or list(CASES)
    unknown = [n for n in names if n not in CASES]
    if unknown:
        raise SystemExit(f"unknown case(s) {unknown}; choose from {list(CASES)}")
    gen_golden.CASES.update(CASES)
    shipped_runner = gen_golden.run_reference
    for name in names:
        gen_golden.run_reference = _runner(VARIANTS[name], CASES[name][2])
        try:
            gen_golden.main([name])
        finally:
            gen_golden.run_reference = shipped_runner
        path = os.path.join(ROOT, "tests", "golden", f"ref_{name}.npz")
        with np.load(path) as g:  # record what the case changed (meta is not compared on regeneration)
            arrays = {k: g[k] for k in g.files}
        meta = json.loads(str(arrays["meta"]))
        meta.update(VARIANTS[name], direct=DIRECT, generator="scripts/gen_golden_scheduler.py")
        arrays["meta"] = np.array(json.dumps(meta))
        np.savez_compressed(path, **arrays)
