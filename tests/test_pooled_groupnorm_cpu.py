"""Frame-pooled GroupNorm (use_inflated_groupnorm=False) on the CPU: the oracle restatement with pooled resnet and output
norms against the UNMODIFIED reference's fixtures (tests/golden/ref_*_pooledgn.npz, scripts/gen_golden_pooled_groupnorm.py),
and the structure of a pooled UNet: which norms pool, its state dict, and the per-frame norms of a ControlNet built
from it."""
import json
import os
from contextlib import contextmanager

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from motionclone_b200.synthetic import UNET_TINY_POOLED_GN_CONFIG, synthetic_inputs, synthetic_state_dict
from oracle import mc_oracle as O

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


@contextmanager
def pooled_oracle():
    """The oracle with the reference's use_inflated_groupnorm=False norms: resnet norm1 / norm2 and conv_norm_out are
    torch.nn.GroupNorm on the 5-D [b, c, f, h, w] tensor (models/resnet.py:143-146, 162-165, models/unet.py:244-247).
    The transformer and motion-module norms do not go through O._gn and stay per frame."""
    per_frame = O._gn
    O._gn = lambda sd, name, x, groups, eps: F.group_norm(x, groups, sd[name + ".weight"], sd[name + ".bias"], eps)
    try:
        yield
    finally:
        O._gn = per_frame


def _case(case):
    g = np.load(os.path.join(GOLDEN, f"ref_{case}.npz"))
    meta = json.loads(str(g["meta"]))
    assert meta["unet_config"] == "UNET_TINY_POOLED_GN_CONFIG"
    shapes = json.load(open(os.path.join(GOLDEN, "ref_state_dict_shapes_tiny.json")))
    sd = synthetic_state_dict(shapes, meta["weight_seed"])
    icfg = meta["infer"]
    inp = synthetic_inputs(icfg["video_length"], icfg["height"], icfg["width"],
                           UNET_TINY_POOLED_GN_CONFIG["cross_attention_dim"], meta["input_seed"])
    return g, meta, sd, icfg, inp


def _close(a, b, tol=1e-5):
    b = torch.as_tensor(b)
    assert (a - b).abs().max().item() <= tol * (b.abs().max().item() + 1e-12)


@pytest.mark.parametrize("case", ["tiny8_pooledgn", "tiny12_pooledgn"])
def test_pooled_oracle_extraction_and_unet_forward(case):
    g, meta, sd, icfg, inp = _case(case)
    with pooled_oracle():
        rep, probs = O.obtain_motion_representation(sd, UNET_TINY_POOLED_GN_CONFIG, inp["clip_latents"],
                                                    inp["clip_noise"], inp["text_embeddings"][[0]],
                                                    icfg["add_noise_step"])
        with torch.no_grad():
            y = O.unet_forward(sd, UNET_TINY_POOLED_GN_CONFIG, inp["noisy_latents"], 500, inp["text_embeddings"][[1]])
    assert list(rep.keys()) == [str(n) for n in g["repr_names"]]
    for i, n in enumerate(rep):
        _close(rep[n][0], g[f"repr_val_{i}"])
        assert torch.equal(rep[n][1], torch.from_numpy(g[f"repr_idx_{i}"]))  # index sets: exact
    _close(probs[next(iter(probs))], g["extract_probs_0"])
    _close(y, g["unet_fwd_t500_cond"])
    # the per-frame oracle does not reproduce the pooled reference: the fixtures discriminate between the modes
    with torch.no_grad():
        y_pf = O.unet_forward(sd, UNET_TINY_POOLED_GN_CONFIG, inp["noisy_latents"], 500, inp["text_embeddings"][[1]])
    ref = torch.as_tensor(g["unet_fwd_t500_cond"])
    assert (y_pf - ref).abs().max().item() > 1e-2 * ref.abs().max().item()


@pytest.mark.parametrize("case", ["tiny8_pooledgn", "tiny12_pooledgn"])
def test_pooled_oracle_guided_sampling_loop(case):
    g, meta, sd, icfg, inp = _case(case)
    rep = {str(n): [torch.from_numpy(g[f"repr_val_{i}"]), torch.from_numpy(g[f"repr_idx_{i}"])]
           for i, n in enumerate(g["repr_names"])}
    stats = {}
    with pooled_oracle():  # guided steps, the guided->plain boundary and the first plain step
        steps = O.sample_loop(sd, UNET_TINY_POOLED_GN_CONFIG, icfg, inp["noisy_latents"], inp["text_embeddings"], rep,
                              stats=stats, max_steps=icfg["guidance_steps"] + 1)
    for i, s in enumerate(steps):
        _close(s, g["latents_per_step"][i])
    _close(torch.stack(stats["loss_unscaled"]), g["losses"][: len(stats["loss_unscaled"])])
    _close(stats["grad"][0], g["grad_step_0"])


def test_c2mini_pooled_fixture_consistent():
    g = np.load(os.path.join(GOLDEN, "ref_c2mini_pooledgn.npz"))
    meta = json.loads(str(g["meta"]))
    assert meta["unet"] == "sd15" and meta["unet_config"] == "UNET_SD15_POOLED_GN_CONFIG"
    assert meta["infer"]["video_length"] == 16 and meta["infer"]["inference_steps"] == 4
    assert list(g["timesteps"]) == list(O.uneven_timesteps(4, 2, 0.4))
    assert np.isfinite(g["latents_per_step"]).all() and np.isfinite(g["grad_step_0"]).all()
    assert g["repr_idx_0"].dtype == np.uint8 and g["repr_idx_0"].max() < 16


def _tiny_unet(**over):
    from motionclone_b200.unet3d import UNet3DConditionModel
    return UNet3DConditionModel(**dict(UNET_TINY_POOLED_GN_CONFIG, **over))


def test_pooled_unet_norm_modules():
    from motionclone_b200.spatial import FramePooledGroupNormNHWC
    from motionclone_b200.unet3d import FramePooledGroupNorm, InflatedGroupNorm
    unet = _tiny_unet()
    pooled, per_frame = [], []
    for name, m in unet.named_modules():
        if isinstance(m, torch.nn.GroupNorm):
            (pooled if isinstance(m, FramePooledGroupNormNHWC) else per_frame).append(name)
    resnet_norms = {n for n, _ in unet.named_modules() if n.endswith((".norm1", ".norm2")) and ".resnets." in n}
    assert set(pooled) == resnet_norms | {"conv_norm_out"}
    assert len(resnet_norms) == 2 * (4 * 2 + 2 + 4 * 3)  # 22 resnets: down 4 x 2, mid 2, up 4 x 3
    assert all(isinstance(unet.get_submodule(n), FramePooledGroupNorm) for n in pooled)
    assert per_frame and all(n.endswith(".norm") for n in per_frame)  # transformer / motion-module input norms
    assert all(".attentions." in n or ".motion_modules." in n for n in per_frame)
    inflated = _tiny_unet(use_inflated_groupnorm=True)
    assert not any(isinstance(m, FramePooledGroupNormNHWC) for m in inflated.modules())
    assert isinstance(inflated.conv_norm_out, InflatedGroupNorm)


def test_pooled_unet_state_dict_matches_reference():
    shapes = json.load(open(os.path.join(GOLDEN, "ref_state_dict_shapes_tiny.json")))
    sd = _tiny_unet().state_dict()
    assert {k: list(v.shape) for k, v in sd.items()} == shapes


def test_controlnet_from_pooled_unet_has_per_frame_norms():
    from motionclone_b200.controlnet import SparseControlNetModel
    from motionclone_b200.spatial import FramePooledGroupNormNHWC
    from motionclone_b200.synthetic import SPARSECTRL_LATENT_KWARGS
    from motionclone_b200.unet3d import InflatedGroupNorm
    cn = SparseControlNetModel.from_unet(_tiny_unet(), controlnet_additional_kwargs=SPARSECTRL_LATENT_KWARGS)
    norms = [m for n, m in cn.named_modules() if ".resnets." in n and n.endswith((".norm1", ".norm2"))]
    assert norms and all(isinstance(m, InflatedGroupNorm) for m in norms)
    assert not any(isinstance(m, FramePooledGroupNormNHWC) for m in cn.modules())


def test_pooled_norm_needs_a_frame_count():
    from motionclone_b200.spatial import FramePooledGroupNormNHWC
    gn = FramePooledGroupNormNHWC(4, 32)
    x = torch.zeros(6, 32, 2, 2).contiguous(memory_format=torch.channels_last)
    for frames in (None, 0, 4):
        with pytest.raises(ValueError):
            gn(x, frames=frames)
