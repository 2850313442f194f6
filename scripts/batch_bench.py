#!/usr/bin/env python
"""Frames/s of batched sampling: full 50-step guided samples at 16 x 512 x 512 (bench.py's `object` workload: 30 guided
steps, guidance_scale 0.4, random-init SD1.5 + v3_sd15_mm widths) with B samples per sample_video call.

The batch sizes alternate within the run: one warm-up call per B (CUDA-graph capture, cuBLAS / cuDNN algorithm choice),
then `--rounds` rounds that time one call of each B in turn, so drifting clocks or a neighbour's load hit every B alike.
Frames/s = B x 16 / wall time of the call (host clock around a synchronised call). Peak memory is
torch.cuda.max_memory_allocated over each B's calls. The card's name and power limit are read in the same run. A B that
runs out of memory is reported as such. One JSON line on stdout.

  python scripts/batch_bench.py [--batches 1 2 4] [--rounds 2] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

F, HW = 16, 512
INFER = dict(cfg_scale=7.5, negative_prompt="", warm_up_steps=10, cool_up_steps=10, motion_guidance_weight=2000,
             motion_guidance_blocks=["up_blocks.1"], add_noise_step=400, inference_steps=50, guidance_steps=30,
             guidance_scale=0.4, video_length=F, height=HW, width=HW, new_prompt="synthetic")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=20).stdout.strip()
    name, power, sm = [c.strip() for c in q.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "sm_clock_max": sm, "torch_name": torch.cuda.get_device_name(0)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 2, 4])
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "batch_bench.py measures the GPU; there is no CPU path"
    import motionclone_b200 as mc
    from motionclone_b200.synthetic import UNET_SD15_CONFIG, synthetic_inputs, synthetic_normal

    dev = torch.device("cuda:0")
    h = lambda t: t.to(dev, torch.float16)  # noqa: E731
    info = card()
    inp = synthetic_inputs(F, HW, HW, 768, 42)
    pipe = mc.build_pipeline(UNET_SD15_CONFIG, dict(INFER, video_latents=h(inp["clip_latents"]),
                                                    video_noise=h(inp["clip_noise"])), device=dev, weight_seed=42)
    pipe.set_prompt_embeds(h(inp["text_embeddings"]))
    rep = pipe.obtain_motion_representation()  # one clip shared by the batch, as t2v_camera.jsonl's prompts share one

    def inputs(B, call):
        lat = torch.cat([synthetic_inputs(F, HW, HW, 768, 1000 + 16 * call + s)["noisy_latents"] for s in range(B)])
        conds = [synthetic_normal("text", (2, 77, 768), 2000 + 16 * call + s)[1:] for s in range(B)]
        text = torch.cat([inp["text_embeddings"][:1]] * B + conds)
        return h(lat), h(text)

    res = {B: {"times_s": [], "peak_bytes": 0, "status": "ok"} for B in args.batches}

    def one(B, call, timed):
        if res[B]["status"] != "ok":
            return
        lat, text = inputs(B, call)
        pipe.set_prompt_embeds(text)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        try:
            out = pipe.sample_video(noisy_latents=lat, return_latents=True, motion_representation=rep)
            torch.cuda.synchronize()
        except torch.OutOfMemoryError as e:
            res[B]["status"] = f"out of memory: {str(e).splitlines()[0][:200]}"
            pipe.invalidate_cuda_graphs()
            torch.cuda.empty_cache()
            return
        dt = time.perf_counter() - t0
        assert torch.isfinite(out).all()
        res[B]["peak_bytes"] = max(res[B]["peak_bytes"], torch.cuda.max_memory_allocated())
        if timed:
            res[B]["times_s"].append(dt)
        print(f"B={B} call {call}: {dt:.2f} s{'' if timed else ' (warm-up)'}", file=sys.stderr, flush=True)

    call = 0
    for B in args.batches:
        one(B, call, False)
        call += 1
    for _ in range(args.rounds):
        for B in args.batches:
            one(B, call, True)
            call += 1
    rows = {}
    for B, r in res.items():
        row = {"status": r["status"], "peak_memory_gib": r["peak_bytes"] / 2 ** 30, "times_s": r["times_s"]}
        if r["times_s"]:
            row["frames_per_s"] = [B * F / t for t in r["times_s"]]
            row["frames_per_s_mean"] = B * F * len(r["times_s"]) / sum(r["times_s"])
        rows[str(B)] = row
    line = {"workload": f"{F}x{HW}x{HW} t2v object, 50-step DDIM (30 guided, guidance_scale 0.4), random-init SD1.5 + "
                        "v3_sd15_mm widths, fp16, one shared motion representation",
            "card": info, "rounds": args.rounds, "batches": rows}
    print(json.dumps(line))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(json.dumps(line, indent=1) + "\n")


if __name__ == "__main__":
    main()
