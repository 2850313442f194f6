"""Clip length on the H100: temporal-attention kernel time per length, and a full guided sample at 24 and 16 frames.

  python scripts/video_length_bench.py [--iters N] [--samples N]

Prints the card's name and power limit, then one JSON line per (L, UNet level) with the median forward and backward
time of the temporal-attention kernels (CUDA events, fused Q|K|V layout as the pipeline feeds them, L2 flushed before
every launch, warm-ups first) at the four UNet levels of a 512 x 512 clip (P = 4096 / 1024 / 256 / 64 positions,
C = 320 / 640 / 1280 / 1280) for L = 12, 16, 24, 32. Bandwidth counts the bytes of the real L: 4 B P L C x 2 B forward
(Q, K, V read, O written), 7 x backward (Q, K, V, dO read, dQ, dK, dV written). Then a 50-step guided sample (30 guided
steps, SD1.5 + motion-module widths, 512 x 512) at 24 and at 16 frames in the same process: frames per second over
`--samples` timed samples after one warm-up sample (which also captures the CUDA graphs)."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

LEVELS = [(320, 4096), (640, 1024), (1280, 256), (1280, 64)]  # (C, positions) of the four UNet levels at 512 x 512
LENGTHS = (12, 16, 24, 32)
HEADS = 8
SAMPLE = dict(cfg_scale=7.5, negative_prompt="", warm_up_steps=10, cool_up_steps=10, motion_guidance_weight=2000,
              motion_guidance_blocks=["up_blocks.1"], add_noise_step=400, inference_steps=50, guidance_steps=30,
              guidance_scale=0.4, height=512, width=512, new_prompt="synthetic")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "not available"
    return {"device": torch.cuda.get_device_name(0), "power_limit,max_sm_clock": q}


def kernel_table(iters):
    from motionclone_b200 import ops
    dev = torch.device("cuda:0")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    for L in LENGTHS:
        for C, P in LEVELS:
            qkv = torch.randn(1, L, P, 3 * C, device=dev, dtype=torch.float16)
            q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
            d_o = torch.randn(1, L, P, C, device=dev, dtype=torch.float16)
            scale = (C // HEADS) ** -0.5
            row = {"L": L, "C": C, "P": P}
            for name, fn, nb in (("fwd", lambda: ops.temporal_attention_forward(q, k, v, HEADS, scale), 4),
                                 ("bwd", lambda: ops.temporal_attention_backward(q, k, v, HEADS, scale, d_o, None, None,
                                                                                 None), 7)):
                for _ in range(3):
                    fn()
                ts = []
                for _ in range(iters):
                    flush.zero_()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    fn()
                    e1.record()
                    torch.cuda.synchronize()
                    ts.append(e0.elapsed_time(e1))
                ms = sorted(ts)[len(ts) // 2]
                nbytes = nb * P * L * C * 2
                row[f"{name}_us"] = round(ms * 1e3, 1)
                row[f"{name}_GBs"] = round(nbytes / 1e6 / ms, 1)
            print(json.dumps(row), flush=True)


def sample_rate(L, n_samples):
    import motionclone_b200 as mc
    from motionclone_b200.synthetic import UNET_SD15_CONFIG, synthetic_inputs
    dev = torch.device("cuda:0")
    inp = synthetic_inputs(L, 512, 512, 768, 42)
    h = lambda t: t.to(dev, torch.float16)  # noqa: E731
    infer = dict(SAMPLE, video_length=L, video_latents=h(inp["clip_latents"]), video_noise=h(inp["clip_noise"]))
    pipe = mc.build_pipeline(UNET_SD15_CONFIG, infer, device=dev, weight_seed=42)
    pipe.set_prompt_embeds(h(inp["text_embeddings"]))
    pipe.obtain_motion_representation()
    lat = h(inp["noisy_latents"])
    out = pipe.sample_video(noisy_latents=lat, return_latents=True)  # warm-up: module loads, graph capture
    torch.cuda.synchronize()
    times = []
    for _ in range(n_samples):
        t0 = time.perf_counter()
        out = pipe.sample_video(noisy_latents=lat, return_latents=True)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    assert torch.isfinite(out).all()
    s = sum(times) / len(times)
    print(json.dumps({"sample": f"{L}x512x512", "steps": SAMPLE["inference_steps"],
                      "guided_steps": SAMPLE["guidance_steps"], "seconds": [round(t, 3) for t in times],
                      "frames_per_s": round(L / s, 3)}), flush=True)
    del pipe, out
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--samples", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs an H100 (no CPU fallback)"
    print(json.dumps(card()), flush=True)
    kernel_table(args.iters)
    for L in (24, 16):
        sample_rate(L, args.samples)


if __name__ == "__main__":
    main()
