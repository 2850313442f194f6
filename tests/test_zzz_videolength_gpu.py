"""A 24-frame clip at full size (24 x 512 x 512, SD1.5 + v3_sd15_mm widths): the temporal attention runs ragged in
32-frame tiles at all four UNet levels. Extraction, then one guided and one plain DDIM step through this package against
the reference's op sequence in fp16 on the same device (oracle/mc_oracle.py), with the bars and the tests of
test_zzz_benchconfig_gpu.py, collected here a second time with this module's `bench_case` fixture:
  * steps: max |x_ours - x_oracle| <= 4 ulp(max |x|), mean <= 0.5 ulp;
  * guidance gradient: cosine >= 0.995;
  * extraction: < 1 % of top-1 rows differ from the oracle's, each a near-tie in the oracle's own probabilities.
The file sorts last, with the other full-size tests, so its memory use does not affect the smaller ones.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import mc_oracle as O  # noqa: E402
from motionclone_b200.synthetic import UNET_SD15_CONFIG, synthetic_inputs, synthetic_state_dict  # noqa: E402
from test_zzz_benchconfig_gpu import BASE  # noqa: E402
# collected in this module, these take the `bench_case` fixture defined below
from test_zzz_benchconfig_gpu import (test_extraction_index_sets_vs_device_oracle,  # noqa: E402,F401
                                      test_single_step_vs_device_oracle)


@pytest.fixture(scope="module", params=["c6_video24_24x512x512"])
def bench_case(request):
    import motionclone_b200 as mc
    dev = torch.device("cuda:0")
    icfg = dict(BASE, video_length=24)
    inp = synthetic_inputs(24, 512, 512, 768, 42)
    h = lambda t: t.to(dev, torch.float16)  # noqa: E731
    icfg.update(video_latents=inp["clip_latents"].half(), video_noise=inp["clip_noise"].half())
    pipe = mc.build_pipeline(UNET_SD15_CONFIG, icfg, device=dev, weight_seed=42)
    pipe.set_prompt_embeds(h(inp["text_embeddings"]))
    shapes = {k: v.shape for k, v in pipe.unet.state_dict().items()}
    sd = {k: h(v) for k, v in synthetic_state_dict(shapes, 42).items()}
    rep = pipe.obtain_motion_representation(motion_representation_path=None)
    with torch.no_grad():
        rep_o, probs_o = O.obtain_motion_representation(sd, UNET_SD15_CONFIG, h(inp["clip_latents"]), h(inp["clip_noise"]),
                                                        h(inp["text_embeddings"][[0]]), icfg["add_noise_step"])
    assert all(v[1].shape[-2] == 24 for v in rep.values())
    torch.cuda.empty_cache()
    return dict(name=request.param, pipe=pipe, sd=sd, icfg=icfg, inp=inp, rep=rep, rep_o=rep_o, probs_o=probs_o, cn=None,
                dev=dev, h=h)
