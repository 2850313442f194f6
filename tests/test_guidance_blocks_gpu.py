"""Motion guidance from other UNet blocks than the shipped ['up_blocks.1'], on the GPU:
  * the loss kernels at 1..64 modules of mixed sizes, bitwise against the CPU statement of the reference's rounding, and
    their refusal of M = 0 and M = 65;
  * end to end against the UNMODIFIED reference's fixtures ref_tiny8_up12, ref_tiny4_all40, ref_tiny8_midv2 and
    ref_c2mini8_up3 (scripts/gen_golden_guidance_blocks.py), with the bars of test_pipeline_gpu.py: its end-to-end tests
    are collected here a second time with this module's `run` fixture;
  * CUDA-graph replay with all 40 temporal attentions guided.
"""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import mc_oracle as O  # noqa: E402
from oracle.guidance_blocks_oracle import mid_block_motion_module  # noqa: E402
from motionclone_b200.synthetic import (UNET_SD15_CONFIG, UNET_TINY_CONFIG, UNET_TINY_MIDV2_CONFIG,  # noqa: E402
                                        synthetic_inputs)
# the end-to-end tests of test_pipeline_gpu.py; collected in this module they take the `run` fixture defined below
from test_pipeline_gpu import (test_guidance_loss_and_gradient_vs_reference, test_latents_vs_reference,  # noqa: E402,F401
                               test_latents_vs_same_device_oracle, test_motion_representation_vs_reference,
                               test_unet_forward_vs_reference)

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
CONFIGS = {"UNET_TINY_CONFIG": UNET_TINY_CONFIG, "UNET_TINY_MIDV2_CONFIG": UNET_TINY_MIDV2_CONFIG,
           "UNET_SD15_CONFIG": UNET_SD15_CONFIG}
# temporal-attention sizes n = positions * heads * frames of every UNet level at 16 x 512 x 512 (64x64 .. 8x8)
LEVEL_N = [4096 * 8 * 16, 1024 * 8 * 16, 256 * 8 * 16, 64 * 8 * 16]


# ---------------------------------------------------------------------------------------------------------------
# loss kernels
# ---------------------------------------------------------------------------------------------------------------
def _loss_operands(M, seed):
    g = torch.Generator().manual_seed(seed)
    n = [LEVEL_N[(m * 7 + seed) % 4] for m in range(M)]
    cur = [torch.rand(k // 128, 8, 16, 1, generator=g).half() for k in n]
    ref = [torch.rand(k // 128, 8, 16, 1, generator=g).half() for k in n]
    return cur, ref


def _cpu_statement(cur, ref):
    """Each module's term as F.mse_loss on half tensors rounds it: fp16(cur - ref), squared to fp16, then the mean, here
    in fp64. The kernel sums the fp16 squares in fp32 over a fixed tree, so its fp16 mean is held to one fp16 rounding
    of this value; the total and the gradients are held bitwise below."""
    h = lambda t: t.half().float()  # noqa: E731
    per = []
    for c, r in zip(cur, ref):
        sq = h(h(c.float() - r.float()) ** 2)
        per.append(sq.double().mean())
    return per


@pytest.mark.parametrize("M", [1, 6, 16, 17, 40, 64])
def test_motion_loss_any_module_count_bitwise(M):
    from motionclone_b200 import ops
    dev = torch.device("cuda:0")
    cur, ref = _loss_operands(M, M)
    cur_d = [c.to(dev).requires_grad_(True) for c in cur]
    ref_d = [r.to(dev) for r in ref]
    loss = ops.motion_loss(cur_d, ref_d)
    # per-module terms of the kernel: one module per call (M = 1) returns that module's fp16 mean
    per = [ops.motion_loss([c.detach()], [r]).float().item() for c, r in zip(cur_d, ref_d)]
    truth = _cpu_statement(cur, ref)
    for p, t in zip(per, truth):  # fp16 of an fp32 tree sum of fp16 squares: within one fp16 rounding of the fp64 mean
        assert abs(p - float(t)) <= 2 ** -10 * abs(float(t)) + 1e-7
    total = torch.tensor(0.0)
    for p in per:  # stack().sum() on half: fp32 accumulation in module order, one rounding to fp16
        total = total + torch.tensor(p, dtype=torch.float32)
    assert loss.item() == total.half().item()  # bitwise: the total is the module-order fp16 sum of the M terms
    # and the same bits as the eager CUDA ops of the reference for the total's module-order sum of the kernel's terms
    eager = torch.stack([torch.tensor(p, dtype=torch.float16, device=dev) for p in per]).sum()
    assert loss.item() == eager.item()
    grads = torch.autograd.grad(2000 * loss, cur_d)
    gout = (2000 * torch.ones((), dtype=torch.float16)).float()
    for gr, c, r in zip(grads, cur, ref):
        want = ((gout * 2.0 / c.numel()) * (c.float() - r.float())).half()  # the kernel's closed form, fp32 then fp16
        assert torch.equal(gr.cpu(), want)


@pytest.mark.parametrize("M", [0, 65])
def test_motion_loss_rejects_module_count(M):
    from motionclone_b200 import _lib
    dev = torch.device("cuda:0")
    cur, ref = _loss_operands(max(M, 1), 3)
    cur = [c.to(dev) for c in cur]
    ref = [r.to(dev) for r in ref]
    d = [torch.empty_like(c) for c in cur]
    arr = lambda ts: (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])  # noqa: E731
    n = (ctypes.c_int64 * len(cur))(*[c.numel() for c in cur])
    per = torch.empty(max(M, 1), dtype=torch.float16, device=dev)
    total = torch.empty((), dtype=torch.float16, device=dev)
    gout = torch.ones((), dtype=torch.float16, device=dev)
    n0 = _lib.launch_count()
    lib = _lib.lib()
    st = lib.mc_motion_loss_fwd(M, arr(cur), arr(ref), n, ctypes.c_void_p(per.data_ptr()), ctypes.c_void_p(total.data_ptr()), None)
    assert st != 0 and "1 <= M <= 64" in lib.mc_last_error().decode()
    st = lib.mc_motion_loss_bwd(M, arr(cur), arr(ref), n, ctypes.c_void_p(gout.data_ptr()), arr(d), None)
    assert st != 0 and "1 <= M <= 64" in lib.mc_last_error().decode()
    assert _lib.launch_count() == n0


def test_motion_loss_gradient_with_inputs_without_grad():
    """Guided modules after the cut run under no_grad in the conditional pass and keep their loss terms without a
    gradient: the gradients of the others are those of the all-grad call, and the loss is the same."""
    from motionclone_b200 import ops
    dev = torch.device("cuda:0")
    cur, ref = _loss_operands(12, 5)
    ref = [r.to(dev) for r in ref]
    all_grad = [c.to(dev).requires_grad_(True) for c in cur]
    some = [c.to(dev).requires_grad_(m % 3 != 0) for m, c in enumerate(cur)]
    l_all, l_some = ops.motion_loss(all_grad, ref), ops.motion_loss(some, ref)
    assert l_all.item() == l_some.item()
    g_all = torch.autograd.grad(l_all, all_grad)
    g_some = torch.autograd.grad(l_some, [c for c in some if c.requires_grad])
    assert all(torch.equal(a, b) for a, b in zip([g for m, g in enumerate(g_all) if m % 3 != 0], g_some))


# ---------------------------------------------------------------------------------------------------------------
# end to end against the reference's fixtures
# ---------------------------------------------------------------------------------------------------------------
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


@pytest.fixture(scope="module", params=["tiny8_up12", "tiny4_all40", "tiny8_midv2", "c2mini8_up3"])
def run(request):
    """As test_pipeline_gpu.run. While a case's tests run, the same-device oracle extracts with the case's guidance
    blocks, and with the v2 mid block for ref_tiny8_midv2."""
    assert torch.cuda.is_available()
    dev = torch.device("cuda:0")
    pipe, g, meta, inp, ucfg = _build(request.param, dev)
    with torch.no_grad():
        fwd = pipe.unet(inp["noisy_latents"].to(dev, torch.float16), 500,
                        encoder_hidden_states=inp["text_embeddings"][[1]].to(dev, torch.float16)).sample
    rep = pipe.obtain_motion_representation(motion_representation_path=None)
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
    final = pipe.sample_video(noisy_latents=inp["noisy_latents"].to(dev, torch.float16), return_latents=True)
    extract = O.obtain_motion_representation
    blocks = tuple(meta["infer"]["motion_guidance_blocks"])
    O.obtain_motion_representation = lambda *a, **k: extract(*a, **dict(k, guidance_blocks=blocks))
    mid = mid_block_motion_module() if ucfg["motion_module_mid_block"] else None
    if mid is not None:
        mid.__enter__()
    try:
        yield dict(case=request.param, pipe=pipe, g=g, meta=meta, inp=inp, ucfg=ucfg, fwd=fwd, rep=rep,
                   per_step=per_step, losses=losses, grads=grads, final=final, dev=dev)
    finally:
        O.obtain_motion_representation = extract
        if mid is not None:
            mid.__exit__(None, None, None)


def test_cuda_graph_replay_is_bit_identical_all40():
    """Graph replay of the plain and unconditional forwards equals eager launches bit for bit with all 40 temporal
    attentions guided (the conditional pass, with its 40-module loss, runs eagerly in both)."""
    dev = torch.device("cuda:0")
    outs = []
    for graphs in (False, True):
        pipe, g, meta, inp, _ = _build("tiny4_all40", dev, use_cuda_graphs=graphs)
        pipe.obtain_motion_representation(motion_representation_path=None)
        finals = [pipe.sample_video(noisy_latents=inp["noisy_latents"].to(dev, torch.float16), return_latents=True)
                  .clone() for _ in range(2)]  # the second sample replays the graphs captured by the first
        assert torch.equal(finals[0], finals[1])
        outs.append(finals[1])
        assert ("_unet_graphs" in pipe.__dict__) == graphs
        assert len(pipe.last_loss_per_sample) == 1 and len(pipe.motion_representation_dict) == 40
    assert torch.equal(outs[0], outs[1])
