"""Batched steps at the bench configuration (16 x 512 x 512, SD1.5 + v3_sd15_mm widths): one guided and one plain DDIM
step of a batch of two samples against the B = 1 step of each sample, with the bench-config bars of
test_zzz_benchconfig_gpu.py: max |diff| <= 4 ulp(max |x|), mean |diff| <= 0.5 ulp, guidance-gradient cosine >= 0.995.
The project's kernels give each sample its single-sample bits; what remains is cuBLAS / cuDNN choosing algorithms by
batch size."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from motionclone_b200.synthetic import UNET_SD15_CONFIG, synthetic_inputs, synthetic_normal  # noqa: E402

ICFG = dict(cfg_scale=7.5, negative_prompt="", warm_up_steps=10, cool_up_steps=10, motion_guidance_weight=2000,
            motion_guidance_blocks=["up_blocks.1"], add_noise_step=400, inference_steps=50, guidance_steps=30,
            guidance_scale=0.4, height=512, width=512, new_prompt="synthetic", video_length=16)


def _ulp(x: float) -> float:
    return 2.0 ** (math.floor(math.log2(max(x, 2.0 ** -14))) - 10)


@pytest.fixture(scope="module")
def batch2():
    import motionclone_b200 as mc
    dev = torch.device("cuda:0")
    h = lambda t: t.to(dev, torch.float16)  # noqa: E731
    inp = [synthetic_inputs(16, 512, 512, 768, seed) for seed in (42, 142)]
    icfg = dict(ICFG, video_latents=inp[0]["clip_latents"].half(), video_noise=inp[0]["clip_noise"].half())
    pipe = mc.build_pipeline(UNET_SD15_CONFIG, icfg, device=dev, weight_seed=42)
    pipe.set_prompt_embeds(h(inp[0]["text_embeddings"]))
    rep = pipe.obtain_motion_representation()
    texts = [h(inp[0]["text_embeddings"]), h(inp[1]["text_embeddings"])]
    texts[1][1] = h(synthetic_normal("text", (2, 77, 768), 245)[1])
    yield dict(pipe=pipe, rep=rep, lat=[h(i["noisy_latents"]) for i in inp], texts=texts)
    torch.cuda.empty_cache()


def _step(pipe, rep, lats, texts, step_index):
    pipe.motion_representation_dict = rep
    pipe.text_embeddings = torch.cat([t[:1] for t in texts] + [t[1:] for t in texts])
    pipe.motion_scale = ICFG["motion_guidance_weight"]
    pipe.add_controlnet = False
    out = pipe.single_step_video(torch.cat(lats), step_index, pipe.scheduler.timesteps[step_index], {})
    grad = pipe.last_gradient.clone() if step_index < ICFG["guidance_steps"] else None
    return out.clone(), grad


@pytest.mark.parametrize("kind", ["guided", "plain"])
def test_batched_step_matches_single_sample_steps(batch2, kind):
    c = batch2
    step_index = 0 if kind == "guided" else ICFG["guidance_steps"]
    lats = c["lat"] if kind == "guided" else [(x * 8.0).half() for x in c["lat"]]  # plain: the loop's magnitude there
    out, grad = _step(c["pipe"], c["rep"], lats, c["texts"], step_index)
    for s in range(2):
        one, grad1 = _step(c["pipe"], c["rep"], [lats[s]], [c["texts"][s]], step_index)
        mag = one.float().abs().max().item()
        ulp = _ulp(mag)
        diff = (out[s:s + 1].float() - one.float()).abs()
        print(f"{kind} step, sample {s}: max|x|={mag:.2f} (ulp {ulp:.4f}); max diff {diff.max().item() / ulp:.2f} ulp, "
              f"mean {diff.mean().item() / ulp:.3f} ulp")
        assert torch.isfinite(out[s]).all()
        assert diff.max().item() <= 4 * ulp and diff.mean().item() <= 0.5 * ulp
        if grad is not None:
            cos = torch.nn.functional.cosine_similarity(grad[s].float().flatten(), grad1[0].float().flatten(), dim=0).item()
            print(f"guided step, sample {s}: gradient cosine vs B = 1 {cos:.6f}")
            assert cos >= 0.995
    torch.cuda.empty_cache()
