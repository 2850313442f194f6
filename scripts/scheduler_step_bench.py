#!/usr/bin/env python
"""Cost of the fused scheduler step (CFG combine + customized_step, motionclone_functions.py:239 + :339-404) per variant,
on the GPU, against the reference's eager op sequence for the same variant.

At [1, 4, 16, 64, 64] and [4, 4, 16, 64, 64] fp16 (one and four 16 x 512 x 512 samples), for each variant: one call of
the fused step as the sampling loop makes it, host scalar algebra + one launch (CUDA events around `--iters` calls; the
variants alternate window by window, so the shipped variant is timed next to the new ones; median over `--reps`
windows), its algorithmic bytes (reads eps_cond, eps_uncond, x, [score],
[noise]; one write) over that time against the H100 SXM's 3.35 TB/s, and the eager sequence (oracle/scheduler_oracle.py
on the same tensors): its time and its kernel launches counted by torch.profiler in a run of its own. The `randn` row is
the variance-noise draw of eta > 0 (torch's generator; not part of the fused launch).

At 1.3 / 5.2 MB per tensor this is launch-latency territory: the numbers say what a step costs, not what HBM can do.
The card's name and power limit are read in the same run. One JSON line on stdout.

  python scripts/scheduler_step_bench.py [--iters 200] [--reps 7] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from batch_bench import card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
# name: (prediction_type, clip, re-derive, score, eta)
VARIANTS = {
    "shipped plain (epsilon)": ("epsilon", False, False, False, 0.0),
    "shipped guided (epsilon + score)": ("epsilon", False, False, True, 0.0),
    "epsilon + score + eta": ("epsilon", False, False, True, 0.5),
    "v_prediction + score": ("v_prediction", False, False, True, 0.0),
    "sample + clip": ("sample", True, False, False, 0.0),
    "v_prediction + clip + re-derive + score + eta": ("v_prediction", True, True, True, 0.5),
}


def _window(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters  # us per call


def _eager_launches(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(e.count for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA)


def measure(batch, iters, reps):
    from motionclone_b200 import ops
    from oracle import mc_oracle as O
    from oracle import scheduler_oracle as S
    dev = torch.device("cuda:0")
    shape = (batch, 4, 16, 64, 64)
    g = torch.Generator().manual_seed(batch)
    ec, eu, x, sc, nz = (torch.randn(shape, generator=g).to(dev, torch.float16) for _ in range(5))
    sc = sc * 0.05
    a_t, a_prev = O.ddim_scalars(O.alphas_cumprod(), O.uneven_timesteps(50, 25, 0.3), 13)
    tensor_bytes = x.numel() * 2
    fused, eager = {}, {}
    for name, (pred, clip, rederive, with_score, eta) in VARIANTS.items():
        kw = dict(prediction_type=pred, clip_sample_range=1.0 if clip else None, use_clipped_model_output=rederive, eta=eta)
        score, noise = (sc if with_score else None), (nz if eta > 0 else None)
        if name.startswith("shipped"):  # the entry point the sampling loop takes for this configuration
            fused[name] = lambda score=score: ops.cfg_ddim_step(ec, eu, x, score, 7.5, a_t, a_prev)
        else:
            fused[name] = lambda score=score, noise=noise, kw=kw: ops.ddim_step(ec, eu, x, score, 7.5, a_t, a_prev,
                                                                                noise=noise, **kw)
        eager[name] = lambda score=score, noise=noise, kw=kw: S.ddim_step(O.cfg_combine(ec, eu, 7.5), x, score, a_t,
                                                                          a_prev, variance_noise=noise, **kw)
    gen = torch.Generator(device=dev).manual_seed(0)
    randn = lambda: torch.randn(shape, generator=gen, device=dev, dtype=torch.float16)  # noqa: E731
    for fn in list(fused.values()) + list(eager.values()) + [randn]:  # warm-up: module load, allocator
        for _ in range(10):
            fn()
    torch.cuda.synchronize()
    t_fused, t_eager, t_randn = {n: [] for n in fused}, {n: [] for n in eager}, []
    for _ in range(reps):
        for name in fused:
            t_fused[name].append(_window(fused[name], iters))
        for name in eager:
            t_eager[name].append(_window(eager[name], iters))
        t_randn.append(_window(randn, iters))
    rows = []
    for name, (pred, clip, rederive, with_score, eta) in VARIANTS.items():
        nbytes = tensor_bytes * (4 + int(with_score) + int(eta > 0))
        us = statistics.median(t_fused[name])
        rows.append({"variant": name, "fused_us": round(us, 2), "fused_us_min_max": [round(min(t_fused[name]), 2),
                                                                                     round(max(t_fused[name]), 2)],
                     "fused_launches": 1, "algorithmic_bytes": nbytes,
                     "fraction_of_3.35TBps": round(nbytes / (us * 1e-6) / HBM_BYTES_PER_S, 3),
                     "eager_us": round(statistics.median(t_eager[name]), 2), "eager_launches": _eager_launches(eager[name])})
        print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
    return {"shape": list(shape), "launches_per_window": iters, "windows": reps, "variants": rows,
            "randn_us": round(statistics.median(t_randn), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "scheduler_step_bench.py measures the GPU; there is no CPU path"
    line = {"card": card(), "sizes": [measure(b, args.iters, args.reps) for b in (1, 4)]}
    print(json.dumps(line))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(json.dumps(line, indent=1) + "\n")


if __name__ == "__main__":
    main()
