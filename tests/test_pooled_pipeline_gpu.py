"""End to end with frame-pooled GroupNorm (use_inflated_groupnorm=False): this package on the GPU against the UNMODIFIED
reference's fixtures ref_tiny8_pooledgn, ref_tiny12_pooledgn (12 frames: also a ragged temporal-attention tile) and
ref_c2mini_pooledgn (SD1.5 widths, 16 frames), written by scripts/gen_golden_pooled_groupnorm.py.

The end-to-end tests are those of test_pipeline_gpu.py, collected here a second time with this module's `run` fixture,
so the pooled fixtures are held to exactly the same bars. Their same-device fp16 oracle runs with the pooled norms of the
reference (torch.nn.GroupNorm on the 5-D tensor for the resnet and output norms) for the whole module. This file also
checks CUDA-graph replay and a B = 2 batched sample against the B = 1 fixture bars.
"""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import mc_oracle as O  # noqa: E402
from motionclone_b200.synthetic import (UNET_SD15_POOLED_GN_CONFIG, UNET_TINY_POOLED_GN_CONFIG,  # noqa: E402
                                        synthetic_inputs)
from test_pipeline_gpu import _rel  # noqa: E402
# the end-to-end tests of test_pipeline_gpu.py; collected in this module they take the `run` fixture defined below
from test_pipeline_gpu import (test_guidance_loss_and_gradient_vs_reference, test_latents_vs_reference,  # noqa: E402,F401
                               test_latents_vs_same_device_oracle, test_motion_representation_vs_reference,
                               test_unet_forward_vs_reference)

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
CONFIGS = {"UNET_TINY_POOLED_GN_CONFIG": UNET_TINY_POOLED_GN_CONFIG,
           "UNET_SD15_POOLED_GN_CONFIG": UNET_SD15_POOLED_GN_CONFIG}


@pytest.fixture(scope="module", autouse=True)
def pooled_oracle():
    """The oracle with the reference's use_inflated_groupnorm=False norms (models/resnet.py:143-146, 162-165,
    models/unet.py:244-247); the transformer and motion-module norms do not go through O._gn and stay per frame."""
    per_frame = O._gn
    O._gn = lambda sd, name, x, groups, eps: F.group_norm(x, groups, sd[name + ".weight"], sd[name + ".bias"], eps)
    yield
    O._gn = per_frame


def _load(case):
    g = np.load(os.path.join(GOLDEN, f"ref_{case}.npz"))
    return g, json.loads(str(g["meta"]))


def _build(case, dev, use_cuda_graphs=True):
    import motionclone_b200 as mc
    g, meta = _load(case)
    ucfg = CONFIGS[meta["unet_config"]]
    icfg = dict(meta["infer"])
    inp = synthetic_inputs(icfg["video_length"], icfg["height"], icfg["width"], ucfg["cross_attention_dim"],
                           meta["input_seed"])
    icfg.update(video_latents=inp["clip_latents"].half(), video_noise=inp["clip_noise"].half(), new_prompt="synthetic")
    pipe = mc.build_pipeline(ucfg, icfg, device=dev, weight_seed=meta["weight_seed"], use_cuda_graphs=use_cuda_graphs)
    pipe.set_prompt_embeds(inp["text_embeddings"].to(dev, torch.float16))
    return pipe, g, meta, inp, ucfg


def _fixture_repr(g):
    return {str(n): [torch.from_numpy(g[f"repr_val_{i}"]).half(), torch.from_numpy(g[f"repr_idx_{i}"])]
            for i, n in enumerate(g["repr_names"])}


@pytest.fixture(scope="module", params=["tiny8_pooledgn", "tiny12_pooledgn", "c2mini_pooledgn"])
def run(request):
    """As test_pipeline_gpu.run: one UNet forward, the package's own extraction, and the sampling loop on the
    reference's motion representation, recording every step's latents and the guided steps' losses and gradients."""
    assert torch.cuda.is_available()
    dev = torch.device("cuda:0")
    pipe, g, meta, inp, ucfg = _build(request.param, dev)
    assert not ucfg["use_inflated_groupnorm"]
    with torch.no_grad():
        fwd = pipe.unet(inp["noisy_latents"].to(dev, torch.float16), 500,
                        encoder_hidden_states=inp["text_embeddings"][[1]].to(dev, torch.float16)).sample
    rep = pipe.obtain_motion_representation(motion_representation_path=None)
    pipe.motion_representation_dict = _fixture_repr(g)
    per_step, losses, grads = [], [], {}
    step = pipe.single_step_video

    def rec(lat, i, t, extra):
        out = step(lat, i, t, extra)
        per_step.append(out)
        if i < meta["infer"]["guidance_steps"]:
            losses.append(pipe.last_loss.float().item())
            grads[i] = pipe.last_gradient
        return out

    pipe.single_step_video = rec
    final = pipe.sample_video(noisy_latents=inp["noisy_latents"].to(dev, torch.float16), return_latents=True)
    return dict(case=request.param, pipe=pipe, g=g, meta=meta, inp=inp, ucfg=ucfg, fwd=fwd, rep=rep,
                per_step=per_step, losses=losses, grads=grads, final=final, dev=dev)


def test_pooled_cuda_graph_replay_is_bit_identical():
    """Graph replay of the plain and unconditional forwards with pooled norms equals eager launches bit for bit."""
    dev = torch.device("cuda:0")
    outs = []
    for graphs in (False, True):
        pipe, g, meta, inp, _ = _build("tiny12_pooledgn", dev, use_cuda_graphs=graphs)
        pipe.obtain_motion_representation(motion_representation_path=None)
        finals = [pipe.sample_video(noisy_latents=inp["noisy_latents"].to(dev, torch.float16), return_latents=True)
                  .clone() for _ in range(2)]  # the second sample replays the graphs captured by the first
        assert torch.equal(finals[0], finals[1])
        outs.append(finals[1])
        assert ("_unet_graphs" in pipe.__dict__) == graphs
    assert torch.equal(outs[0], outs[1])


def test_pooled_batched_sampling_meets_fixture_bars():
    """B = 2 in one loop (guided steps at b = 2, plain steps at b = 4 with two tiling samples of 2f frames, each holding
    two pools of f): both samples meet the B = 1 fixture bars on their latents."""
    dev = torch.device("cuda:0")
    pipe, g, meta, inp, _ = _build("tiny8_pooledgn", dev)
    te = inp["text_embeddings"].to(dev, torch.float16)
    pipe.set_prompt_embeds(torch.cat([te[[0]], te[[0]], te[[1]], te[[1]]]))
    noisy = inp["noisy_latents"].to(dev, torch.float16)
    per_step = []
    step = pipe.single_step_video

    def rec(lat, i, t, extra):
        out = step(lat, i, t, extra)
        per_step.append(out)
        return out

    pipe.single_step_video = rec
    final = pipe.sample_video(noisy_latents=torch.cat([noisy, noisy]), return_latents=True,
                              motion_representation=_fixture_repr(g))
    assert final.shape[0] == 2 and torch.isfinite(final).all()
    ref = g["latents_per_step"]
    for s in range(2):
        r0, r_end = _rel(per_step[0][[s]], ref[0]), _rel(final[[s]], ref[-1])
        print(f"pooled B=2 sample {s}: latent rel err vs reference after step 0 {r0:.4f}, at the end {r_end:.4f}")
        assert r0 < 1.5e-2 and r_end < 5e-2
