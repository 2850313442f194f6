"""Microbenchmark: this package's wgmma + TMA spatial self-attention against the library SDPA kernels on the UNet's
shapes (forward; forward + backward when the backward kernels exist). Profiling aid, not a bench value."""
import json
import sys
import os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
from motionclone_b200 import _lib, ops

# `--lib PATH`: time a side-by-side build of the same sources instead of the in-tree library
if "--lib" in sys.argv:
    i = sys.argv.index("--lib")
    _lib.LIB_PATH = os.path.abspath(sys.argv[i + 1])
    del sys.argv[i:i + 2]

dev = "cuda"


def bench(fn, n=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


shapes = [("self64", 16, 8, 4096, 40), ("self32", 16, 8, 1024, 80), ("self16", 16, 8, 256, 160), ("self8", 16, 8, 64, 160),
          ("self64_b2", 32, 8, 4096, 40), ("self64_L32", 32, 8, 4096, 40)]
ONLY = sys.argv[1] if len(sys.argv) > 1 else None   # e.g. `self64`: one shape, few iterations (profiler captures)
for name, B, H, N, dh in shapes:
    if ONLY and name != ONLY:
        continue
    C = H * dh
    qkv = torch.randn(B, N, 3 * C, device=dev, dtype=torch.float16)
    q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    q4, k4, v4 = (t.view(B, N, H, dh).transpose(1, 2) for t in (q, k, v))
    scale = dh ** -0.5
    flops = 4 * B * H * N * N * dh
    with torch.no_grad():
        t_lib = bench(lambda: F.scaled_dot_product_attention(q4, k4, v4, scale=scale))
        t_own = bench(lambda: ops.spatial_attention_forward(q, k, v, H, scale))
        o_lib = F.scaled_dot_product_attention(q4, k4, v4, scale=scale).transpose(1, 2).reshape(B, N, C)
        o_own, _ = ops.spatial_attention_forward(q, k, v, H, scale)
    row = dict(shape=name, B=B, H=H, N=N, dh=dh, lib_fwd_ms=t_lib, own_fwd_ms=t_own, lib_tflops=flops / t_lib / 1e9,
               own_tflops=flops / t_own / 1e9, max_abs_diff=(o_lib.float() - o_own.float()).abs().max().item())
    if hasattr(ops, "SpatialAttentionTC"):
        qg = qkv.detach().clone().requires_grad_(True)

        def fb_own():
            o = ops.SpatialAttentionTC.apply(qg[..., :C], qg[..., C:2 * C], qg[..., 2 * C:], H, scale)
            torch.autograd.grad(o, qg, torch.ones_like(o))

        def fb_lib():
            qq, kk, vv = (qg[..., i * C:(i + 1) * C].view(B, N, H, dh).transpose(1, 2) for i in range(3))
            o = F.scaled_dot_product_attention(qq, kk, vv, scale=scale)
            torch.autograd.grad(o, qg, torch.ones_like(o))
        row.update(lib_fwdbwd_ms=bench(fb_lib, 10), own_fwdbwd_ms=bench(fb_own, 10))
    print(json.dumps(row), flush=True)
