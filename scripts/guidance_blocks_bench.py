"""Cost of guiding more UNet blocks, on bench.py's `object` workload (16 x 512 x 512, 50-step DDIM with 30 guided steps,
guidance_scale 0.4, random-init SD1.5 + v3_sd15_mm widths, fp16):
  * full samples for motion_guidance_blocks = ['up_blocks.1'] (shipped, 6 modules), up_blocks.1 + up_blocks.2 (12) and
    all 40 temporal attentions, alternating: one warm-up call each, then `--rounds` rounds timing one call of each
    (host clock around a synchronised call); peak memory per set;
  * one guided step per set (CUDA events around single_step_video at step 0, median of `--steps` calls);
  * the motion-loss forward + backward kernels alone at the module sizes of 6 and of 40 guided modules, CUDA events
    over `--loss-iters` launch pairs, and their share of the guided step of the same set.
The card's name and power limit are read in the same run. One JSON line on stdout.

  python scripts/guidance_blocks_bench.py [--rounds 2] [--steps 5] [--loss-iters 500] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402

from batch_bench import F, HW, INFER, card  # noqa: E402

UP = ["up_blocks.0", "up_blocks.1", "up_blocks.2", "up_blocks.3"]
SETS = {"up_blocks.1": ["up_blocks.1"], "up_blocks.1+2": ["up_blocks.1", "up_blocks.2"], "all40": ["down_blocks"] + UP}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--loss-iters", type=int, default=500)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "guidance_blocks_bench.py measures the GPU; there is no CPU path"
    import motionclone_b200 as mc
    from motionclone_b200 import dist as mcdist, guidance, ops
    from motionclone_b200.synthetic import UNET_SD15_CONFIG, synthetic_inputs

    dev = torch.device("cuda:0")
    h = lambda t: t.to(dev, torch.float16)  # noqa: E731
    info = card()
    inp = synthetic_inputs(F, HW, HW, 768, 42)
    pipes, reps = {}, {}
    for name, blocks in SETS.items():
        p = mc.build_pipeline(UNET_SD15_CONFIG, dict(INFER, motion_guidance_blocks=blocks,
                                                     video_latents=h(inp["clip_latents"]),
                                                     video_noise=h(inp["clip_noise"])), device=dev, weight_seed=42)
        p.set_prompt_embeds(h(inp["text_embeddings"]))
        reps[name] = p.obtain_motion_representation()
        pipes[name] = p
    res = {n: {"times_s": [], "peak_bytes": 0, "modules": len(reps[n])} for n in SETS}

    def one(name, timed):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        out = pipes[name].sample_video(noisy_latents=h(inp["noisy_latents"]), return_latents=True)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        assert torch.isfinite(out).all()
        res[name]["peak_bytes"] = max(res[name]["peak_bytes"], torch.cuda.max_memory_allocated())
        if timed:
            res[name]["times_s"].append(dt)
        print(f"{name}: {dt:.2f} s{'' if timed else ' (warm-up)'}", file=sys.stderr, flush=True)

    for name in SETS:
        one(name, False)
    for _ in range(args.rounds):
        for name in SETS:
            one(name, True)

    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    for name, p in pipes.items():  # one guided step (step 0) per set
        lat = h(inp["noisy_latents"])
        ms = []
        for _ in range(args.steps):
            a, b = ev(), ev()
            a.record()
            p.single_step_video(lat, 0, int(p.scheduler.timesteps_host[0]), {})
            b.record()
            torch.cuda.synchronize()
            ms.append(a.elapsed_time(b))
        res[name]["guided_step_ms"] = statistics.median(ms)

    for name in ("up_blocks.1", "all40"):  # the loss kernels alone at that set's module sizes
        man = mcdist.representation_manifest_for(pipes[name].unet, list(guidance.guided_modules(pipes[name])), HW, HW, F)
        g = torch.Generator(device=dev).manual_seed(7)
        cur = [torch.rand(v, generator=g, device=dev).half().requires_grad_(True) for _, v, _ in man]
        ref = [torch.rand(v, generator=g, device=dev).half() for _, v, _ in man]
        for _ in range(10):
            torch.autograd.grad(ops.motion_loss(cur, ref), cur)
        a, b = ev(), ev()
        a.record()
        for _ in range(args.loss_iters):
            torch.autograd.grad(ops.motion_loss(cur, ref), cur)
        b.record()
        torch.cuda.synchronize()
        per = a.elapsed_time(b) / args.loss_iters
        res[name]["loss_fwd_bwd_ms"] = per
        res[name]["loss_entries"] = int(sum(torch.Size(v).numel() for _, v, _ in man))
        res[name]["loss_share_of_guided_step"] = per / res[name]["guided_step_ms"]

    rows = {}
    for name, r in res.items():
        row = dict(r, peak_memory_gib=r.pop("peak_bytes") / 2 ** 30)
        if r["times_s"]:
            row["frames_per_s"] = [F / t for t in r["times_s"]]
            row["frames_per_s_mean"] = F * len(r["times_s"]) / sum(r["times_s"])
        rows[name] = row
    line = {"workload": f"{F}x{HW}x{HW} t2v object, 50-step DDIM (30 guided, guidance_scale 0.4), random-init SD1.5 + "
                        "v3_sd15_mm widths, fp16", "card": info, "rounds": args.rounds,
            "loss_timing": "motion_loss forward + autograd backward (2 launches + torch glue) per iteration, CUDA events",
            "sets": rows}
    print(json.dumps(line))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(json.dumps(line, indent=1) + "\n")


if __name__ == "__main__":
    main()
