"""End-to-end GPU parity: this package (fp16, CUDA kernels) against
  (a) the golden fixtures written by the UNMODIFIED reference in fp32 (tests/golden/ref_*.npz, oracle/gen_golden.py),
  (b) the oracle restatement run in fp16 on the same device (the reference's op sequence on this GPU).
Tolerances are fp16 tolerances (north_star: "within a stated fp16 tolerance"), stated at each assert, relative to the
tensor's max magnitude because the random-init UNet drives latents to |x| ~ 1e2 (fp16 spacing there is 6e-2).
"""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import mc_oracle as O  # noqa: E402
from motionclone_b200.synthetic import (SPARSECTRL_IMAGE_KWARGS, SPARSECTRL_LATENT_KWARGS, UNET_SD15_CONFIG,  # noqa: E402
                                        UNET_TINY_CONFIG, synthetic_condition, synthetic_inputs, synthetic_state_dict)

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _load(case):
    g = np.load(os.path.join(GOLDEN, f"ref_{case}.npz"))
    meta = json.loads(str(g["meta"]))
    return g, meta


def _rel(a, b):
    a, b = a.float().cpu(), torch.as_tensor(b).float()
    return ((a - b).abs().max() / (b.abs().max() + 1e-12)).item()


def _build(case, dev):
    import motionclone_b200 as mc
    g, meta = _load(case)
    ucfg = UNET_TINY_CONFIG if meta["unet"] == "tiny" else UNET_SD15_CONFIG
    icfg = dict(meta["infer"])
    inp = synthetic_inputs(icfg["video_length"], icfg["height"], icfg["width"], ucfg["cross_attention_dim"],
                           meta["input_seed"])
    icfg.update(video_latents=inp["clip_latents"].half(), video_noise=inp["clip_noise"].half(), new_prompt="synthetic")
    cn_kwargs = None
    if icfg.get("sparsectrl"):  # SparseCtrl cases (BASELINE configs[3], [4] topology): synthetic condition inputs
        kind = icfg["sparsectrl"]
        cn_kwargs = SPARSECTRL_LATENT_KWARGS if kind == "latent" else SPARSECTRL_IMAGE_KWARGS
        cond = synthetic_condition(kind, len(icfg["image_index"]), icfg["height"], icfg["width"], icfg["video_length"],
                                   meta["input_seed"] + 5)
        inp.update(cond)
        images = cond["cond_latents"] if kind == "latent" else cond["cond_images"]
        inp["controlnet_images"] = images.permute(1, 0, 2, 3).unsqueeze(0)  # [1, c, n_img, h, w]
        icfg.update(controlnet_images=inp["controlnet_images"].half(), video_pixels=cond.get("clip_pixels"))
    pipe = mc.build_pipeline(ucfg, icfg, device=dev, weight_seed=meta["weight_seed"], controlnet_kwargs=cn_kwargs)
    pipe.set_prompt_embeds(inp["text_embeddings"].to(dev, torch.float16))
    inp["cn_kwargs"] = cn_kwargs
    return pipe, g, meta, inp, ucfg


def _oracle_controlnet(run_or_pipe, meta, inp, dev):
    """dict for the oracle's controlnet arguments (fp16 on device), or None for the t2v cases."""
    if inp.get("cn_kwargs") is None:
        return None
    pipe = run_or_pipe
    shapes = {k: v.shape for k, v in pipe.controlnet.state_dict().items()}
    sdc = {k: v.to(dev, torch.float16) for k, v in synthetic_state_dict(shapes, meta["weight_seed"] + 1).items()}
    return dict(sd=sdc, kwargs=inp["cn_kwargs"], image_index=meta["infer"]["image_index"],
                scale=meta["infer"]["controlnet_scale"], images=inp["controlnet_images"].to(dev, torch.float16))


@pytest.fixture(scope="module", params=["tiny8", "tiny16", "c1", "tiny8_i2v_latent", "tiny8_i2v_image", "c2mini"])
def run(request):
    assert torch.cuda.is_available()
    dev = torch.device("cuda:0")
    pipe, g, meta, inp, ucfg = _build(request.param, dev)
    with torch.no_grad():
        fwd = pipe.unet(inp["noisy_latents"].to(dev, torch.float16), 500,
                        encoder_hidden_states=inp["text_embeddings"][[1]].to(dev, torch.float16)).sample
    use_cn = inp.get("cn_kwargs") is not None
    rep = pipe.obtain_motion_representation(motion_representation_path=None, use_controlnet=use_cn)
    # the sampling loop is compared with the reference on the REFERENCE's motion representation (identical inputs);
    # the package's own extraction is checked separately in test_motion_representation_vs_reference
    pipe.motion_representation_dict = {str(n): [torch.from_numpy(g[f"repr_val_{i}"]).half(),
                                                torch.from_numpy(g[f"repr_idx_{i}"])]
                                       for i, n in enumerate(g["repr_names"])}
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
    final = pipe.sample_video(noisy_latents=inp["noisy_latents"].to(dev, torch.float16), return_latents=True,
                              add_controlnet=use_cn)
    return dict(case=request.param, pipe=pipe, g=g, meta=meta, inp=inp, ucfg=ucfg, fwd=fwd, rep=rep,
                per_step=per_step, losses=losses, grads=grads, final=final, dev=dev)


def test_unet_forward_vs_reference(run):
    r = _rel(run["fwd"], run["g"]["unet_fwd_t500_cond"])
    print(run["case"], "unet fwd rel err vs reference fp32:", r)
    assert r < 2e-2  # fp16 storage through ~150 layers vs fp32: 2 % of max |eps|


def test_motion_representation_vs_reference(run):
    g = run["g"]
    names = list(run["rep"].keys())
    assert names == [str(n) for n in g["repr_names"]]
    total, mismatch, worst_gaps = 0, 0, []
    for i, n in enumerate(names):
        val, idx = run["rep"][n]
        ref_val, ref_idx = torch.from_numpy(g[f"repr_val_{i}"]), torch.from_numpy(g[f"repr_idx_{i}"])
        assert val.shape == ref_val.shape and idx.dtype == torch.uint8
        bad = idx.cpu() != ref_idx
        total += bad.numel()
        mismatch += int(bad.sum())
        # values: fp16 probabilities vs fp32 ones, 1e-2 absolute (inputs to the softmax carry fp16 error of the UNet)
        assert (val.float().cpu() - ref_val).abs().max().item() < 2.5e-2
        # every index mismatch, in EVERY guided module, must sit on a row that is a near-tie in the REFERENCE's own fp32
        # probabilities (fixture key extract_top2gap_i = top-1 minus top-2 probability of the reference's rows). The
        # bound is an fp16 statement: q, k reach the softmax through ~100 fp16 layers, so two probabilities closer than
        # the accumulated fp16 error of a score can legitimately swap order (8e-3 is ~64 fp16 ulps of a probability ~ 1/L).
        gap = torch.from_numpy(g[f"extract_top2gap_{i}"]).unsqueeze(-1)
        worst = float(gap[bad].max()) if bool(bad.any()) else 0.0
        worst_gaps.append(worst)
        assert worst < 8e-3, f"module {i}: top-1 index differs where the reference's top-2 gap is {worst:.3e}"
    print(run["case"], f"top-1 index mismatches vs fp32 reference: {mismatch}/{total}; largest reference top-2 gap on a "
          f"mismatching row, per module: {[f'{w:.2e}' for w in worst_gaps]}")
    assert mismatch / total < 0.02


def test_guidance_loss_and_gradient_vs_reference(run):
    g, meta = run["g"], run["meta"]
    icfg = meta["infer"]
    want = []
    for i, raw in enumerate(g["losses"]):  # the fixture stores compute_temp_loss's return (unscaled)
        want.append(float(raw) * icfg["motion_guidance_weight"] *
                    O.loss_scale(i, icfg["guidance_steps"], icfg["warm_up_steps"], icfg["cool_up_steps"]))
    print(run["case"], "loss:", run["losses"], "reference:", want)
    assert abs(run["losses"][0] - want[0]) <= 2e-2 * abs(want[0])  # step 0 shares identical inputs
    r = _rel(run["grads"][0], g["grad_step_0"])
    ref_g = torch.from_numpy(g["grad_step_0"]).flatten()
    cos = torch.nn.functional.cosine_similarity(run["grads"][0].float().cpu().flatten(), ref_g, dim=0).item()
    # yardstick: the reference's own op sequence in fp16 on this device (oracle), against the same fp32 gradient
    dev, inp, ucfg = run["dev"], run["inp"], run["ucfg"]
    shapes = {k: v.shape for k, v in run["pipe"].unet.state_dict().items()}
    sd = {k: v.to(dev, torch.float16) for k, v in synthetic_state_dict(shapes, meta["weight_seed"]).items()}
    h = lambda t: t.to(dev, torch.float16)  # noqa: E731
    rep = {str(n): [h(torch.from_numpy(g[f"repr_val_{i}"])), torch.from_numpy(g[f"repr_idx_{i}"]).to(dev)]
           for i, n in enumerate(g["repr_names"])}
    stats = {}
    O.sample_loop(sd, ucfg, icfg, h(inp["noisy_latents"]), h(inp["text_embeddings"]), rep, stats=stats, max_steps=1,
                  controlnet=_oracle_controlnet(run["pipe"], meta, inp, dev))
    r_eager = _rel(stats["grad"][0], g["grad_step_0"])
    print(run["case"], f"grad step 0: rel max err {r:.4f} (eager fp16 op sequence: {r_eager:.4f}), cosine {cos:.6f}")
    # fp16 backward through ~60 % of the UNet vs fp32 autograd: no worse than 1.5x the eager fp16 path's own error
    assert r < max(6e-2, 1.5 * r_eager) and cos > 0.995


def test_latents_vs_reference(run):
    ref = run["g"]["latents_per_step"]
    kept = run["g"]["latents_steps_kept"] if "latents_steps_kept" in run["g"] else range(len(ref))
    rels = [_rel(run["per_step"][int(s)], ref[j]) for j, s in enumerate(kept)]
    print(run["case"], "per-step latent rel err vs reference fp32:", rels)
    assert rels[0] < 1.5e-2  # one step: fp16 UNet (+ fp16 SparseCtrl in the i2v cases) vs fp32
    assert rels[-1] < 5e-2
    assert torch.isfinite(run["final"]).all()


def test_latents_vs_same_device_oracle(run):
    """The oracle in fp16 on this GPU = the reference's op sequence (baddbmm/softmax/bmm attention, eager elementwise
    ops) on identical weights and inputs."""
    dev, meta, inp, ucfg = run["dev"], run["meta"], run["inp"], run["ucfg"]
    shapes = {k: v.shape for k, v in run["pipe"].unet.state_dict().items()}
    sd = {k: v.to(dev, torch.float16) for k, v in synthetic_state_dict(shapes, meta["weight_seed"]).items()}
    icfg = meta["infer"]
    h = lambda t: t.to(dev, torch.float16)  # noqa: E731
    cn = _oracle_controlnet(run["pipe"], meta, inp, dev)
    rep, _ = O.obtain_motion_representation(sd, ucfg, h(inp["clip_latents"]), h(inp["clip_noise"]),
                                            h(inp["text_embeddings"][[0]]), icfg["add_noise_step"], controlnet=cn,
                                            clip_pixels=None if inp.get("clip_pixels") is None else h(inp["clip_pixels"]))
    mism = sum(int((rep[n][1] != run["rep"][n][1]).sum()) for n in rep)
    tot = sum(rep[n][1].numel() for n in rep)
    g = run["g"]
    gold = {str(n): [h(torch.from_numpy(g[f"repr_val_{i}"])), torch.from_numpy(g[f"repr_idx_{i}"]).to(dev)]
            for i, n in enumerate(g["repr_names"])}
    steps = O.sample_loop(sd, ucfg, icfg, h(inp["noisy_latents"]), h(inp["text_embeddings"]), gold, controlnet=cn)
    rels = [_rel(run["per_step"][i], steps[i].cpu()) for i in range(len(steps))]
    print(run["case"], f"vs fp16 oracle on device: index mismatches {mism}/{tot}; per-step latent rel err {rels}")
    assert mism / tot < 0.02
    assert rels[-1] < 5e-2


def test_cuda_graph_replay_is_bit_identical():
    """The captured no-grad UNet forwards (plain step, unconditional forward of guided steps) replay the same kernels on
    the same data: the sampled latents must equal the eager launches bit for bit."""
    import motionclone_b200 as mc
    dev = torch.device("cuda:0")
    g, meta = _load("tiny16")
    icfg = dict(meta["infer"])
    inp = synthetic_inputs(icfg["video_length"], icfg["height"], icfg["width"], UNET_TINY_CONFIG["cross_attention_dim"],
                           meta["input_seed"])
    icfg.update(video_latents=inp["clip_latents"].half(), video_noise=inp["clip_noise"].half(), new_prompt="synthetic")
    outs = []
    for graphs in (False, True):
        pipe = mc.build_pipeline(UNET_TINY_CONFIG, icfg, device=dev, weight_seed=meta["weight_seed"], use_cuda_graphs=graphs)
        pipe.set_prompt_embeds(inp["text_embeddings"].to(dev, torch.float16))
        pipe.obtain_motion_representation(motion_representation_path=None)
        finals = [pipe.sample_video(noisy_latents=inp["noisy_latents"].to(dev, torch.float16), return_latents=True).clone()
                  for _ in range(2)]  # second sample replays the graphs captured by the first
        assert torch.equal(finals[0], finals[1])
        outs.append(finals[1])
        assert ("_unet_graphs" in pipe.__dict__) == graphs
    assert torch.equal(outs[0], outs[1])

