"""Batched sampling, host side (no kernel runs here): every malformed batch is refused before the loop starts, the
plain step pairs each sample with its own prompt rows, and the per-sample motion representations are concatenated in
the temporal kernel's row order."""
import pytest
import torch

import motionclone_b200 as mc
from motionclone_b200 import guidance, ops
from motionclone_b200.synthetic import UNET_TINY_CONFIG
from motionclone_b200.unet3d import UNet3DConditionOutput

F = 8
ICFG = dict(cfg_scale=7.5, negative_prompt="", warm_up_steps=10, cool_up_steps=10, motion_guidance_weight=2000,
            motion_guidance_blocks=["up_blocks.1"], add_noise_step=400, inference_steps=4, guidance_steps=2,
            guidance_scale=0.3, video_length=F, height=64, width=64, new_prompt="batch")


@pytest.fixture(scope="module")
def pipe():
    p = mc.build_pipeline(UNET_TINY_CONFIG, ICFG, device="cpu", dtype=torch.float32, use_cuda_graphs=False)

    def no_loop(*a, **k):
        raise AssertionError("the sampling loop started on a malformed batch")

    p.single_step_video = no_loop
    return p


def _rep(pipe, seed, frames=F, n=4):
    g = torch.Generator().manual_seed(seed)
    return {name: [torch.rand(n, 8, frames, 1, generator=g),
                   torch.randint(0, frames, (n, 8, frames, 1), generator=g).to(torch.uint8)]
            for name in guidance.guided_modules(pipe)}


def _text(b, c=UNET_TINY_CONFIG["cross_attention_dim"]):
    return torch.randn(2 * b, 77, c)


def _lat(b):
    return torch.randn(b, 4, F, 8, 8)


def _call(pipe, b_text, **kw):
    pipe.set_prompt_embeds(_text(b_text))
    pipe.motion_representation_dict, pipe.motion_representation_path = _rep(pipe, 0), None
    return pipe.sample_video(return_latents=True, **kw)


def test_prompt_latent_count_mismatch(pipe):
    with pytest.raises(ValueError, match="batch size mismatch"):
        _call(pipe, 2, noisy_latents=_lat(3))
    with pytest.raises(ValueError, match="batch size mismatch"):
        _call(pipe, 1, noisy_latents=_lat(2))


def test_prompt_rows_must_be_2b(pipe):
    pipe.set_prompt_embeds(torch.randn(3, 77, UNET_TINY_CONFIG["cross_attention_dim"]))
    pipe.motion_representation_dict = _rep(pipe, 0)
    with pytest.raises(ValueError, match=r"\[2B, 77, c\]"):
        pipe.sample_video(noisy_latents=_lat(1), return_latents=True)


def test_latents_must_be_5d(pipe):
    with pytest.raises(ValueError, match="noisy_latents"):
        _call(pipe, 1, noisy_latents=torch.randn(4, F, 8, 8))


def test_generator_list_length(pipe):
    gens = [torch.Generator().manual_seed(i) for i in range(3)]
    with pytest.raises(ValueError, match="generators 3"):
        _call(pipe, 2, generator=gens)


def test_representation_list_length(pipe):
    with pytest.raises(ValueError, match="motion representations 3"):
        _call(pipe, 2, noisy_latents=_lat(2), motion_representation=[_rep(pipe, i) for i in range(3)])


def test_representation_index_out_of_range(pipe):
    bad = _rep(pipe, 2)
    name = next(iter(bad))
    bad[name][1][0, 0, 0, 0] = F
    with pytest.raises(ValueError, match=f"index {F} >= video_length {F}"):
        _call(pipe, 2, noisy_latents=_lat(2), motion_representation=[_rep(pipe, 1), bad])


def test_representation_frame_count(pipe):
    with pytest.raises(ValueError, match="frames"):
        _call(pipe, 2, noisy_latents=_lat(2), motion_representation=_rep(pipe, 1, frames=F + 4))


def test_representation_missing_module(pipe):
    partial = _rep(pipe, 1)
    partial.pop(next(iter(partial)))
    with pytest.raises(ValueError, match="no entry for guided module"):
        _call(pipe, 2, noisy_latents=_lat(2), motion_representation=[_rep(pipe, 1), partial])


def test_sparsectrl_batch_not_implemented(pipe):
    with pytest.raises(NotImplementedError, match="SparseCtrl"):
        _call(pipe, 2, noisy_latents=_lat(2), add_controlnet=True)


def test_frame_cap_of_the_plain_pass(pipe):
    # 2 * B * f frames go through one GroupNorm call of the plain step: 2 * 65 * 8 = 1040 > 1024
    with pytest.raises(ValueError, match="at most 64 samples"):
        _call(pipe, 65, noisy_latents=_lat(65))


def test_plain_step_pairs_each_sample_with_its_prompts(pipe, monkeypatch):
    """b = 2B pass over [x_1..B, x_1..B] against [uncond_1..B, cond_1..B]; CFG gets eps_cond = rows B.., eps_uncond =
    rows ..B; the GroupNorm sample count of the pass is B."""
    B = 3
    seen = {}

    def fake_forward(sample, timestep, encoder_hidden_states=None, **kw):
        seen["sample"], seen["text"], seen["samples"] = sample.clone(), encoder_hidden_states.clone(), ops._gn_samples
        tag = encoder_hidden_states[:, 0, 0].view(-1, 1, 1, 1, 1)
        return UNet3DConditionOutput(sample=sample * 0 + tag)

    def fake_step(eps_cond, eps_uncond, cfg_scale, step_index, sample, score=None, **kw):
        seen["cond"], seen["uncond"], seen["x"] = eps_cond.clone(), eps_uncond.clone(), sample.clone()
        return sample

    monkeypatch.setattr(pipe.unet, "forward", fake_forward)
    monkeypatch.setattr(pipe.scheduler, "customized_step_fused", fake_step)
    text, x = _text(B), _lat(B)
    pipe.text_embeddings = text
    guidance.single_step_video(pipe, x, ICFG["guidance_steps"], 10, {})
    assert seen["samples"] == B and ops._gn_samples == 1
    assert torch.equal(seen["sample"], torch.cat([x, x])) and torch.equal(seen["text"], text)
    for s in range(B):
        assert torch.all(seen["uncond"][s] == text[s, 0, 0])
        assert torch.all(seen["cond"][s] == text[B + s, 0, 0])
    assert torch.equal(seen["x"], x)


def test_representation_concatenation_row_order(pipe):
    a, b = _rep(pipe, 10), _rep(pipe, 11)
    pipe.motion_representation_dict = a
    pipe._sample_reps = [a, b, a]
    try:
        dev_reps, cat_idx = guidance._device_batch(pipe, torch.device("cpu"), 3)
    finally:
        pipe._sample_reps = None
    assert dev_reps[0] is dev_reps[2]  # a shared dict is copied once
    for name in a:
        want = torch.cat([a[name][1], b[name][1], a[name][1]])
        assert cat_idx[name].dtype == torch.uint8 and torch.equal(cat_idx[name], want)
        assert torch.equal(dev_reps[1][name][0], b[name][0].half())
    # cached: the same dicts give the same device tensors
    pipe._sample_reps = [a, b, a]
    try:
        again = guidance._device_batch(pipe, torch.device("cpu"), 3)[1]
    finally:
        pipe._sample_reps = None
    assert all(again[n] is cat_idx[n] for n in a)


def test_batch_samples_context():
    assert ops._gn_samples == 1
    with ops.batch_samples(4):
        assert ops._gn_samples == 4
        with ops.batch_samples(2):
            assert ops._gn_samples == 2
        assert ops._gn_samples == 4
    assert ops._gn_samples == 1
    with pytest.raises(ValueError):
        with ops.batch_samples(0):
            pass
