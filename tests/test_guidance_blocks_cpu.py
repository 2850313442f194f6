"""Motion guidance from other UNet blocks than the shipped ['up_blocks.1'], on the CPU:
  * the oracle against the UNMODIFIED reference's fixtures ref_tiny8_up12 (two levels), ref_tiny4_all40 (all 40 temporal
    attentions, 4 frames), ref_tiny8_midv2 (the v2 mid-block motion module) and ref_c2mini8_up3 (SD1.5 widths, 8 frames,
    the full-resolution level), written by scripts/gen_golden_guidance_blocks.py;
  * the gradient-cut rule and the refusals of a block list the path cannot run, raised before anything runs;
  * the multi-GPU representation layout at mixed levels: manifest, pack / unpack, a two-rank gloo broadcast.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import motionclone_b200 as mc
from motionclone_b200 import _lib, dist as mcdist, guidance
from motionclone_b200.synthetic import (UNET_SD15_CONFIG, UNET_TINY_CONFIG, UNET_TINY_MIDV2_CONFIG, synthetic_inputs,
                                        synthetic_state_dict)
from motionclone_b200.unet3d import UNet3DConditionModel
from oracle import mc_oracle as O
from oracle.guidance_blocks_oracle import mid_block_motion_module

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
CONFIGS = {"UNET_TINY_CONFIG": UNET_TINY_CONFIG, "UNET_TINY_MIDV2_CONFIG": UNET_TINY_MIDV2_CONFIG,
           "UNET_SD15_CONFIG": UNET_SD15_CONFIG}
CASES = {  # fixture: (guided modules, levels (h/8 >> level) they sit at)
    "tiny8_up12": (12, {2, 1}),
    "tiny4_all40": (40, {0, 1, 2, 3}),
    "tiny8_midv2": (8, {3, 2}),
    "c2mini8_up3": (6, {0}),
}
UP = ["up_blocks.0", "up_blocks.1", "up_blocks.2", "up_blocks.3"]


def _case(case):
    g = np.load(os.path.join(GOLDEN, f"ref_{case}.npz"))
    meta = json.loads(str(g["meta"]))
    ucfg = CONFIGS[meta["unet_config"]]
    sd = synthetic_state_dict({k: v.shape for k, v in UNet3DConditionModel(**ucfg).state_dict().items()},
                              meta["weight_seed"])
    icfg = meta["infer"]
    inp = synthetic_inputs(icfg["video_length"], icfg["height"], icfg["width"], ucfg["cross_attention_dim"],
                           meta["input_seed"])
    return g, meta, ucfg, sd, icfg, inp


def _close(a, b, tol=1e-5):
    b = torch.as_tensor(b)
    assert a.shape == b.shape
    assert (a - b).abs().max().item() <= tol * (b.abs().max().item() + 1e-12)


def _oracle_ctx(ucfg):
    from contextlib import nullcontext
    return mid_block_motion_module() if ucfg["motion_module_mid_block"] else nullcontext()


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_reproduces_fixture(case):
    """Extraction (values to 1e-5, index sets exact), a plain UNet forward, and the guided steps (latents, unscaled loss,
    step-0 gradient) against the reference run with the same motion_guidance_blocks. The SD1.5-width case runs its
    first guided step only, to bound the CPU time."""
    g, meta, ucfg, sd, icfg, inp = _case(case)
    blocks = tuple(icfg["motion_guidance_blocks"])
    n_modules, _ = CASES[case]
    assert len(g["repr_names"]) == n_modules
    with _oracle_ctx(ucfg):
        rep, _ = O.obtain_motion_representation(sd, ucfg, inp["clip_latents"], inp["clip_noise"],
                                                inp["text_embeddings"][[0]], icfg["add_noise_step"],
                                                guidance_blocks=blocks)
        with torch.no_grad():
            y = O.unet_forward(sd, ucfg, inp["noisy_latents"], 500, inp["text_embeddings"][[1]])
        names = [str(n) for n in g["repr_names"]]
        # the oracle records in execution order (down, mid, up); the reference keys by named_modules (down, up, mid)
        assert sorted(rep) == sorted(names) and [n for n in rep if "mid_block" not in n] == \
            [n for n in names if "mid_block" not in n]
        for i, n in enumerate(names):
            _close(rep[n][0], g[f"repr_val_{i}"])
            assert torch.equal(rep[n][1], torch.from_numpy(g[f"repr_idx_{i}"]))
        _close(y, g["unet_fwd_t500_cond"])
        gold = {str(n): [torch.from_numpy(g[f"repr_val_{i}"]), torch.from_numpy(g[f"repr_idx_{i}"])]
                for i, n in enumerate(g["repr_names"])}
        stats = {}
        max_steps = 1 if meta["unet"] == "sd15" else icfg["guidance_steps"] + 1
        steps = O.sample_loop(sd, ucfg, icfg, inp["noisy_latents"], inp["text_embeddings"], gold, stats=stats,
                              max_steps=max_steps)
    kept = list(g["latents_steps_kept"]) if "latents_steps_kept" in g.files else list(range(len(g["latents_per_step"])))
    for j, s in enumerate(kept):
        if s < len(steps):
            _close(steps[s], g["latents_per_step"][j])
    _close(torch.stack(stats["loss_unscaled"]), g["losses"][: len(stats["loss_unscaled"])])
    _close(stats["grad"][0], g["grad_step_0"])


def _pipe(ucfg, blocks, frames=8, hw=128, guidance_steps=2):
    icfg = dict(cfg_scale=7.5, negative_prompt="", warm_up_steps=1, cool_up_steps=1, motion_guidance_weight=2000,
                motion_guidance_blocks=list(blocks), add_noise_step=400, inference_steps=3,
                guidance_steps=guidance_steps, guidance_scale=0.3, video_length=frames, height=hw, width=hw,
                new_prompt="synthetic")
    inp = synthetic_inputs(frames, hw, hw, ucfg["cross_attention_dim"], 42)
    icfg.update(video_latents=inp["clip_latents"].half(), video_noise=inp["clip_noise"].half())
    pipe = mc.build_pipeline(ucfg, icfg, device=torch.device("cpu"), weight_seed=42)
    pipe.set_prompt_embeds(inp["text_embeddings"].half())
    return pipe, inp


@pytest.mark.parametrize("blocks,cut", [(["up_blocks.1"], 1), (["up_blocks.1", "up_blocks.2"], 2),
                                        (["down_blocks"] + UP, 3), (["mid_block", "up_blocks.1"], 1),
                                        (["up_blocks.2", "up_blocks.0"], 0), (["down_blocks.2"], 2),
                                        (["up_blocks.12"], 12)])
def test_cut_rule_matches_reference(blocks, cut):
    """int(motion_guidance_blocks[-1].split(".")[-1]) (motionclone_functions.py:602), whatever the entry names."""
    unet = UNet3DConditionModel(**UNET_TINY_CONFIG)
    unet.input_config = dict(motion_guidance_blocks=blocks)
    assert unet._guidance_cut() == cut == int(blocks[-1].split(".")[-1])


@pytest.mark.parametrize("last", ["mid_block", "up_blocks", "down_blocks"])
def test_cut_without_integer_suffix_raises_before_any_launch(last):
    pipe, inp = _pipe(UNET_TINY_MIDV2_CONFIG, ["up_blocks.1", last])
    with pytest.raises(ValueError) as ref_err:
        int(last.split(".")[-1])
    n0 = _lib.launch_count()
    for call in (lambda: pipe.obtain_motion_representation(motion_representation_path=None),
                 lambda: pipe.sample_video(noisy_latents=inp["noisy_latents"].half(), return_latents=True),
                 lambda: pipe.unet(inp["noisy_latents"].half(), 500, encoder_hidden_states=inp["text_embeddings"][[1]]
                                   .half())):
        with pytest.raises(ValueError) as err:
            call()
        assert str(err.value) == str(ref_err.value)  # the reference's int() error
    assert _lib.launch_count() == n0


def test_guided_block_after_cut_refused_in_extraction():
    """['up_blocks.2', 'up_blocks.1'] cuts at 1: extraction returns before up_blocks.2 runs, so it is refused up front
    with the modules and the cut named (the reference fails later, with an unrelated AttributeError)."""
    pipe, _ = _pipe(UNET_TINY_CONFIG, ["up_blocks.2", "up_blocks.1"])
    n0 = _lib.launch_count()
    with pytest.raises(ValueError, match=r"up_blocks\.2\.motion_modules\.0.*after the cut up_blocks\.1") as err:
        pipe.obtain_motion_representation(motion_representation_path=None)
    assert "'up_blocks.1'" in str(err.value) and "up_blocks.1.motion_modules" not in str(err.value)
    assert _lib.launch_count() == n0


@pytest.mark.parametrize("blocks", [["up_blocks.2", "mid_block.0"], ["up_blocks.3", "down_blocks.9.1"], ["mid_block.0"]])
def test_no_guided_module_under_grad_refused_before_sampling(blocks):
    """Every guided module lies after the cut (or none matches), so no loss term carries gradient: ValueError before
    the loop, not an autograd error at step 0."""
    pipe, inp = _pipe(UNET_TINY_CONFIG, blocks)
    n0 = _lib.launch_count()
    with pytest.raises(ValueError, match="no guided module runs under grad"):
        pipe.sample_video(noisy_latents=inp["noisy_latents"].half(), return_latents=True, motion_representation={})
    assert _lib.launch_count() == n0


def test_guided_modules_and_levels():
    """Module counts and the order of the representation's keys: the reference's named_modules order (down, up, mid),
    which is also the order the guidance loss adds the modules' terms in."""
    for ucfg, blocks, n in [(UNET_TINY_CONFIG, ["down_blocks"] + UP, 40), (UNET_TINY_MIDV2_CONFIG, ["mid_block", "up_blocks.1"], 8),
                            (UNET_TINY_MIDV2_CONFIG, ["down_blocks", "mid_block"] + UP, 42),
                            (UNET_TINY_CONFIG, ["up_blocks.1", "up_blocks.2"], 12)]:
        pipe, _ = _pipe(ucfg, blocks)
        names = list(guidance.guided_modules(pipe))
        assert len(names) == n
        order = {"down_blocks": 0, "up_blocks": 1, "mid_block": 2}  # the reference's named_modules order
        keys = [(order[s.split(".")[0]], int(s.split(".")[1]) if s.split(".")[1].isdigit() else 0) for s in names]
        assert keys == sorted(keys)


def _levels_of(manifest, hw):
    lat = hw // 8
    return {int(round(np.log2(lat / np.sqrt(v[0])))) for _, v, _ in manifest}


@pytest.mark.parametrize("case", list(CASES))
def test_manifest_for_matches_fixture_shapes(case):
    """representation_manifest_for gives every module of the reference's representation its own [N, heads, f, 1]."""
    g, meta, ucfg, _, icfg, _ = _case(case)
    unet = UNet3DConditionModel(**ucfg)
    names = [str(n) for n in g["repr_names"]]
    man = mcdist.representation_manifest_for(unet, names, icfg["height"], icfg["width"], icfg["video_length"])
    assert [m[0] for m in man] == names
    for i, (_, vshape, ishape) in enumerate(man):
        assert vshape == ishape == tuple(g[f"repr_val_{i}"].shape)
    assert _levels_of(man, icfg["height"]) == CASES[case][1]


def test_manifest_for_shipped_block_equals_fixed_manifest():
    """For up_blocks.1 at 16x512x512 the per-level builder and representation_manifest (bench.py's) agree."""
    unet = UNet3DConditionModel(**UNET_SD15_CONFIG)
    unet.input_config = dict(motion_guidance_blocks=["up_blocks.1"])
    names = [n for n, m in unet.named_modules() if type(m).__name__ == "VersatileAttention" and "up_blocks.1" in n]
    assert mcdist.representation_manifest_for(unet, names, 512, 512, 16) == \
        mcdist.representation_manifest(names, (512 // 32) * (512 // 32), 8, 16)
    all_names = [n for n, m in unet.named_modules() if type(m).__name__ == "VersatileAttention"]
    man = mcdist.representation_manifest_for(unet, all_names, 512, 512, 16)
    sizes = {n.split(".motion_modules")[0]: v[0] for n, v, _ in man}
    assert sizes == {"down_blocks.0": 4096, "down_blocks.1": 1024, "down_blocks.2": 256, "down_blocks.3": 64,
                     "up_blocks.0": 64, "up_blocks.1": 256, "up_blocks.2": 1024, "up_blocks.3": 4096}
    with pytest.raises(ValueError):
        mcdist.representation_manifest_for(unet, ["conv_in"], 512, 512, 16)


def _mixed_rep(g):
    return {str(n): [torch.from_numpy(g[f"repr_val_{i}"]).half(), torch.from_numpy(g[f"repr_idx_{i}"])]
            for i, n in enumerate(g["repr_names"])}


@pytest.mark.parametrize("case", ["tiny8_up12", "tiny4_all40", "tiny8_midv2"])
def test_mixed_level_representation_round_trips_and_checks(case):
    g, meta, ucfg, _, icfg, _ = _case(case)
    rep = _mixed_rep(g)
    buf, man = mcdist.pack_representation(rep)
    assert man == mcdist.representation_manifest_for(UNet3DConditionModel(**ucfg), list(rep), icfg["height"],
                                                     icfg["width"], icfg["video_length"])
    assert buf.numel() == mcdist.manifest_nbytes(man)
    back = mcdist.unpack_representation(buf, man)
    assert list(back) == list(rep)
    for k in rep:
        assert torch.equal(back[k][0], rep[k][0]) and torch.equal(back[k][1], rep[k][1])
    guidance._check_representation(back, icfg["video_length"])  # mixed N per module is accepted


_WORKER = r"""
import json, os, sys, numpy as np, torch
sys.path.insert(0, sys.argv[1])
from motionclone_b200 import dist as mcdist
from motionclone_b200.synthetic import UNET_TINY_CONFIG
from motionclone_b200.unet3d import UNet3DConditionModel
rank, world, local = mcdist.init_from_env("gloo")
g = np.load(os.path.join(sys.argv[1], "tests", "golden", "ref_tiny8_up12.npz"))
icfg = json.loads(str(g["meta"]))["infer"]
full = {str(n): [torch.from_numpy(g[f"repr_val_{i}"]).half(), torch.from_numpy(g[f"repr_idx_{i}"])]
        for i, n in enumerate(g["repr_names"])}
manifest = mcdist.representation_manifest_for(UNet3DConditionModel(**UNET_TINY_CONFIG), list(full), icfg["height"],
                                              icfg["width"], icfg["video_length"])
assert len({v[0] for _, v, _ in manifest}) == 2  # two levels in one buffer
got = mcdist.broadcast_representation(full if rank == 0 else None, torch.device("cpu"), manifest)
assert list(got) == list(full)
for k in full:
    assert torch.equal(got[k][0], full[k][0]) and torch.equal(got[k][1], full[k][1])
print("rank", rank, "ok")
"""


def test_two_rank_gloo_broadcast_mixed_levels(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(_WORKER)
    procs = []
    for r in range(2):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE="2", LOCAL_RANK=str(r), MASTER_ADDR="127.0.0.1",
                   MASTER_PORT="29617")
        procs.append(subprocess.Popen([sys.executable, str(script), ROOT], env=env, stdout=subprocess.PIPE,
                                      stderr=subprocess.STDOUT))
    for p in procs:
        out, _ = p.communicate(timeout=120)
        assert p.returncode == 0, out.decode()
