"""Microbenchmark of the text cross-attention core (reference models/attention.py:280-285 -> :535-542) at the four
layer shapes of the SD1.5 UNet (16 x 512 x 512): this package's wgmma kernels (csrc/spatial_attn_tc.cu, csrc/spatial_attn_bwd_tc.cu) next to the
library kernel that F.scaled_dot_product_attention picks for the same strided views. CUDA events, L2 flushed between
launches, 3 warm-ups, median of 20. One JSON line per shape. Algorithmic bytes: forward = Q read + O written;
backward (dQ only: the text K/V carry no gradient, weights are frozen) = Q, dO read + dQ written."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F

from motionclone_b200 import ops

dev = torch.device("cuda:0")
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
H, NK, FR = 8, 77, 16


def timeit(fn, iters=20):
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
    ts.sort()
    return ts[len(ts) // 2]


for B in (1, 2):
    for C, N in ((320, 4096), (640, 1024), (1280, 256), (1280, 64)):
        dh = C // H
        scale = dh ** -0.5
        q = torch.randn(B, FR * N, C, device=dev, dtype=torch.float16)
        kv = torch.randn(B, NK, 2 * C, device=dev, dtype=torch.float16)
        k, v = kv[..., :C], kv[..., C:]
        d_o = torch.randn_like(q)
        q4 = q.view(B, -1, H, dh).transpose(1, 2)
        k4, v4 = (t.reshape(B, NK, H, dh).transpose(1, 2) for t in (k, v))
        res = dict(B=B, C=C, N=N, MB_fwd=round(2 * q.numel() * 2 / 1e6, 1))
        res["ours_fwd_ms"] = round(timeit(lambda: ops.cross_attention_forward(q, k, v, H, scale)), 4)
        res["lib_fwd_ms"] = round(timeit(lambda: F.scaled_dot_product_attention(q4, k4, v4, scale=scale)), 4)
        o_ours = ops.cross_attention_forward(q, k, v, H, scale)
        o_lib = F.scaled_dot_product_attention(q4, k4, v4, scale=scale).transpose(1, 2).reshape(B, -1, C)
        res["fwd_maxdiff"] = round((o_ours.float() - o_lib.float()).abs().max().item(), 5)
        if hasattr(ops, "cross_attention_backward"):
            res["ours_bwd_ms"] = round(timeit(lambda: ops.cross_attention_backward(q, k, v, d_o, H, scale)), 4)
        qg = q.clone().requires_grad_(True)
        qg4 = qg.view(B, -1, H, dh).transpose(1, 2)
        og = F.scaled_dot_product_attention(qg4, k4, v4, scale=scale)
        d_o4 = d_o.view(B, -1, H, dh).transpose(1, 2)
        res["lib_bwd_ms"] = round(timeit(lambda: torch.autograd.grad(og, qg, d_o4, retain_graph=True)), 4)
        if hasattr(ops, "cross_attention_backward"):
            dq_lib = torch.autograd.grad(og, qg, d_o4, retain_graph=True)[0]
            dq = ops.cross_attention_backward(q, k, v, d_o, H, scale)
            res["bwd_maxdiff"] = round((dq.float() - dq_lib.float()).abs().max().item(), 5)
            res["bwd_ref_max"] = round(dq_lib.float().abs().max().item(), 5)
        print(json.dumps(res), flush=True)
