"""Parity at the bench configuration (16 x 512 x 512, SD1.5 + motion-module widths) with frame-pooled GroupNorm
(use_inflated_groupnorm=False): motion extraction and one guided and one plain DDIM step of this package against
`oracle.single_step` in fp16 on the same device, with the reference's pooled norms (torch.nn.GroupNorm on the 5-D tensor
for the resnet and output norms). Same bars as test_zzz_benchconfig_gpu.py: steps within 4 ulp max and 0.5 ulp mean,
guidance-gradient cosine >= 0.995 and max-abs error <= 8 %, and the extraction index-set rule.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import mc_oracle as O  # noqa: E402
from motionclone_b200.synthetic import UNET_SD15_POOLED_GN_CONFIG, synthetic_inputs, synthetic_state_dict  # noqa: E402
from test_zzz_benchconfig_gpu import BASE, _ulp  # noqa: E402
# the extraction index-set test; collected in this module it takes the `bench_case` fixture defined below
from test_zzz_benchconfig_gpu import test_extraction_index_sets_vs_device_oracle  # noqa: E402,F401


@pytest.fixture(scope="module", autouse=True)
def pooled_oracle():
    """The oracle with the reference's use_inflated_groupnorm=False resnet and output norms."""
    per_frame = O._gn
    O._gn = lambda sd, name, x, groups, eps: F.group_norm(x, groups, sd[name + ".weight"], sd[name + ".bias"], eps)
    yield
    O._gn = per_frame


@pytest.fixture(scope="module")
def bench_case(pooled_oracle):
    import motionclone_b200 as mc
    dev = torch.device("cuda:0")
    icfg = dict(BASE, video_length=16)
    inp = synthetic_inputs(16, 512, 512, 768, 42)
    h = lambda t: t.to(dev, torch.float16)  # noqa: E731
    icfg.update(video_latents=inp["clip_latents"].half(), video_noise=inp["clip_noise"].half())
    pipe = mc.build_pipeline(UNET_SD15_POOLED_GN_CONFIG, icfg, device=dev, weight_seed=42)
    pipe.set_prompt_embeds(h(inp["text_embeddings"]))
    shapes = {k: v.shape for k, v in pipe.unet.state_dict().items()}
    sd = {k: h(v) for k, v in synthetic_state_dict(shapes, 42).items()}
    rep = pipe.obtain_motion_representation(motion_representation_path=None)
    with torch.no_grad():
        rep_o, probs_o = O.obtain_motion_representation(sd, UNET_SD15_POOLED_GN_CONFIG, h(inp["clip_latents"]),
                                                        h(inp["clip_noise"]), h(inp["text_embeddings"][[0]]),
                                                        icfg["add_noise_step"])
    torch.cuda.empty_cache()
    return dict(name="pooledgn_16x512x512", pipe=pipe, sd=sd, icfg=icfg, inp=inp, rep=rep, rep_o=rep_o,
                probs_o=probs_o, dev=dev, h=h)


@pytest.mark.parametrize("kind", ["guided", "plain"])
def test_pooled_single_step_vs_device_oracle(bench_case, kind):
    c = bench_case
    pipe, icfg, inp, h = c["pipe"], c["icfg"], c["inp"], c["h"]
    step_index = 0 if kind == "guided" else icfg["guidance_steps"]
    timesteps = O.uneven_timesteps(icfg["inference_steps"], icfg["guidance_steps"], icfg["guidance_scale"])
    acp = O.alphas_cumprod()
    lat = h(inp["noisy_latents"])
    if kind == "plain":  # a latent of the magnitude the loop has at the first plain step (after 30 guided steps)
        lat = (lat * 8.0).half()
    rep = {n: [v[0].clone(), v[1].clone()] for n, v in c["rep_o"].items()}
    pipe.motion_representation_dict = rep
    pipe._repr_on_device = None
    pipe.scheduler.customized_set_timesteps(icfg["inference_steps"], icfg["guidance_steps"], icfg["guidance_scale"],
                                            device=c["dev"], timestep_spacing_type="uneven")
    pipe.text_embeddings = h(inp["text_embeddings"])
    pipe.motion_scale = icfg["motion_guidance_weight"]
    pipe.add_controlnet = False
    ours = pipe.single_step_video(lat, step_index, pipe.scheduler.timesteps[step_index], {})
    stats = {}
    want = O.single_step(c["sd"], UNET_SD15_POOLED_GN_CONFIG, icfg, lat, step_index, timesteps, acp,
                         h(inp["text_embeddings"]), rep, stats=stats)
    mag = want.float().abs().max().item()
    ulp = _ulp(mag)
    diff = (ours.float() - want.float()).abs()
    print(f"{c['name']} {kind} step: max|x|={mag:.2f} (fp16 ulp {ulp:.4f}); max abs diff {diff.max().item():.4f} = "
          f"{diff.max().item() / ulp:.2f} ulp; mean abs diff {diff.mean().item():.5f} = "
          f"{diff.mean().item() / ulp:.3f} ulp")
    assert torch.isfinite(ours).all()
    assert diff.max().item() <= 4 * ulp and diff.mean().item() <= 0.5 * ulp
    if kind == "guided":
        g_o = stats["grad"][step_index].to(c["dev"])
        g = pipe.last_gradient.float()
        cos = torch.nn.functional.cosine_similarity(g.flatten(), g_o.flatten(), dim=0).item()
        rel = (g - g_o).abs().max().item() / g_o.abs().max().item()
        print(f"{c['name']} guidance gradient: cosine {cos:.6f}, max-abs rel err {rel:.4f}")
        assert cos >= 0.995 and rel <= 8e-2
    torch.cuda.empty_cache()
