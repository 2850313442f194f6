#!/usr/bin/env python
"""Cost of frame-pooled GroupNorm (use_inflated_groupnorm=False) against the per-frame GroupNorm, on the GPU.

1. Kernels, per UNet level at 16 x 512 x 512 (every resnet / output-norm shape, 16 frames, fused SiLU and time-embedding
   add as in the resnets): forward (statistics + apply) and backward (reduce + apply), per-frame (mc_groupnorm_nhwc_batched
   / _bwd_batched) against pooled over the 16 frames (mc_groupnorm_nhwc_pooled / _bwd_pooled). CUDA events around
   `--iters` calls; the two modes alternate window by window; the median over `--reps` windows is reported.
2. Full 50-step guided samples at 16 x 512 x 512 (bench.py's `object` workload) with each mode, alternating, after one
   warm-up sample each (CUDA-graph capture, cuDNN algorithm choice); frames/s = 16 / wall time of a synchronised call.

The card's name and power limit are read in the same run. One JSON line on stdout.

  python scripts/pooled_groupnorm_bench.py [--iters 50] [--reps 7] [--rounds 2] [--skip-samples] [--out FILE]
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

import torch  # noqa: E402

from batch_bench import INFER, card  # noqa: E402

F, G, EPS = 16, 32, 1e-5
# (C, h) of the resnet norm1 / norm2 and conv_norm_out inputs at 512 x 512 (latent 64)
LEVELS = [(320, 64), (640, 64), (960, 64), (320, 32), (640, 32), (960, 32), (1280, 32), (1920, 32), (640, 16),
          (1280, 16), (1920, 16), (2560, 16), (1280, 8), (2560, 8)]


def kernel_times(iters, reps):
    from motionclone_b200 import _lib, ops
    L = _lib.lib()
    dev = torch.device("cuda:0")
    rows = []
    for C, h in LEVELS:
        g = torch.Generator().manual_seed(C + h)
        x = (torch.randn(F, C, h, h, generator=g) * 2).to(dev, torch.float16).contiguous(memory_format=torch.channels_last)
        dz = torch.randn(F, C, h, h, generator=g).to(dev, torch.float16).contiguous(memory_format=torch.channels_last)
        w = (1 + 0.1 * torch.randn(C, generator=g)).to(dev, torch.float16)
        b = (0.1 * torch.randn(C, generator=g)).to(dev, torch.float16)
        cb = torch.randn(1, C, generator=g).to(dev, torch.float16)
        y, dx = torch.empty_like(x), torch.empty_like(x)
        need = int(L.mc_groupnorm_workspace_bytes(F, G))
        ws, wsb = (torch.zeros(need, dtype=torch.uint8, device=dev) for _ in range(2))
        stats = {mode: torch.empty(F, G, 2, dtype=torch.float32, device=dev) for mode in ("per_frame", "pooled")}
        p, st = ops._ptr, ops._stream

        def fwd(mode):
            if mode == "pooled":
                return L.mc_groupnorm_nhwc_pooled(p(x), p(cb), F, p(y), p(w), p(b), p(ws), need, F, h * h, C, G, 1, F,
                                                  EPS, 1, st())
            return L.mc_groupnorm_nhwc_batched(p(x), p(cb), F, p(y), p(w), p(b), p(ws), need, F, h * h, C, G, 1, EPS, 1,
                                               st())

        def bwd(mode):
            s = p(stats[mode])
            if mode == "pooled":
                return L.mc_groupnorm_nhwc_bwd_pooled(p(x), p(cb), F, p(dz), p(dx), s, p(w), p(b), p(wsb), need, F,
                                                      h * h, C, G, 1, F, 1, st())
            return L.mc_groupnorm_nhwc_bwd_batched(p(x), p(cb), F, p(dz), p(dx), s, p(w), p(b), p(wsb), need, F, h * h,
                                                   C, G, 1, 1, st())

        for mode in ("per_frame", "pooled"):  # warm-up, and the statistics each backward reads
            _lib.check(fwd(mode), "fwd")
            _lib.check(L.mc_groupnorm_nhwc_stats(p(ws), p(stats[mode]), F, h * h, G, EPS, st()), "stats")
            _lib.check(bwd(mode), "bwd")
        times = {(d, m): [] for d in ("fwd", "bwd") for m in ("per_frame", "pooled")}
        for _ in range(reps):
            for d, fn in (("fwd", fwd), ("bwd", bwd)):
                for mode in ("per_frame", "pooled"):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(iters):
                        fn(mode)
                    e1.record()
                    e1.synchronize()
                    times[(d, mode)].append(e0.elapsed_time(e1) * 1e3 / iters)
        row = {"C": C, "hw": f"{h}x{h}", "frames": F}
        for (d, mode), v in times.items():
            row[f"{d}_{mode}_us"] = round(statistics.median(v), 2)
        for d in ("fwd", "bwd"):
            row[f"{d}_pooled_over_per_frame"] = round(row[f"{d}_pooled_us"] / row[f"{d}_per_frame_us"], 3)
        rows.append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
    return rows


def sample_rates(rounds):
    import motionclone_b200 as mc
    from motionclone_b200.synthetic import UNET_SD15_CONFIG, UNET_SD15_POOLED_GN_CONFIG, synthetic_inputs
    dev = torch.device("cuda:0")
    h = lambda t: t.to(dev, torch.float16)  # noqa: E731
    inp = synthetic_inputs(F, 512, 512, 768, 42)
    pipes = {}
    for mode, ucfg in (("per_frame", UNET_SD15_CONFIG), ("pooled", UNET_SD15_POOLED_GN_CONFIG)):
        pipe = mc.build_pipeline(ucfg, dict(INFER, video_latents=h(inp["clip_latents"]), video_noise=h(inp["clip_noise"])),
                                 device=dev, weight_seed=42)
        pipe.set_prompt_embeds(h(inp["text_embeddings"]))
        pipe.obtain_motion_representation()
        pipes[mode] = pipe
    times = {m: [] for m in pipes}
    for r in range(rounds + 1):  # round 0 is the warm-up
        for mode, pipe in pipes.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = pipe.sample_video(noisy_latents=h(inp["noisy_latents"]), return_latents=True)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            assert torch.isfinite(out).all()
            if r:
                times[mode].append(dt)
            print(f"{mode} sample {r}: {dt:.2f} s{'' if r else ' (warm-up)'}", file=sys.stderr, flush=True)
    return {m: {"times_s": t, "frames_per_s": [F / x for x in t], "frames_per_s_mean": F * len(t) / sum(t)}
            for m, t in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--skip-samples", action="store_true")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "pooled_groupnorm_bench.py measures the GPU; there is no CPU path"
    line = {"card": card(), "kernels_16_frames": kernel_times(args.iters, args.reps)}
    if not args.skip_samples:
        line["samples_16x512x512"] = sample_rates(args.rounds)
    print(json.dumps(line))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(json.dumps(line, indent=1) + "\n")


if __name__ == "__main__":
    main()
