"""Cold-L2 microbenchmark of the temporal-attention kernels at the four layer shapes of the SD1.5 UNet
(16 x 512 x 512, b=1 and b=2), fused-QKV layout as the pipeline uses it. CUDA events, L2 flushed between launches
(256 MB write), >= 3 warm-ups. Prints one JSON line per shape; `python scripts/kernel_bench.py --ncu` runs each kernel
twice only (for use under ncu)."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from motionclone_b200 import ops

ncu = "--ncu" in sys.argv
dev = torch.device("cuda:0")
peak = 3350.0  # GB/s, H100 SXM data sheet (HBM3); MEASURED_PEAKS.json overrides it
try:
    peak = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    pass
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
L, H = 16, 8
shapes = [(320, 4096), (640, 1024), (1280, 256), (1280, 64)]
if "--l32" in sys.argv:
    L = 32
iters = 2 if ncu else 20
tot = {"fwd": [0.0, 0.0], "bwd": [0.0, 0.0]}
for B in (1, 2):
    for C, D in shapes:
        qkv = torch.randn(B, L, D, 3 * C, device=dev, dtype=torch.float16)
        q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
        d_o = torch.randn(B, L, D, C, device=dev, dtype=torch.float16)
        scale = (C // H) ** -0.5
        res = {}
        for name, fn, nb in (("fwd", lambda: ops.temporal_attention_forward(q, k, v, H, scale), 4),
                             ("bwd", lambda: ops.temporal_attention_backward(q, k, v, H, scale, d_o, None, None, None), 7)):
            for _ in range(1 if ncu else 3):
                fn()
            ts = []
            for _ in range(iters):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); fn(); e1.record(); torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            ts.sort()
            ms = ts[len(ts) // 2]
            nbytes = nb * B * L * D * C * 2
            res[name] = dict(ms=round(ms, 4), GBs=round(nbytes / 1e6 / ms, 1), frac=round(nbytes / 1e6 / ms / peak, 3), MB=round(nbytes / 1e6, 1))
            if B == 1:
                mult = 10
                tot[name][0] += mult * nbytes; tot[name][1] += mult * ms
        print(json.dumps(dict(B=B, C=C, D=D, L=L, **res)))
for name in tot:
    b, ms = tot[name]
    print(json.dumps(dict(summary=name, per_forward_MB=round(b / 1e6, 1), per_forward_ms=round(ms, 3), GBs=round(b / 1e6 / ms, 1), frac=round(b / 1e6 / ms / peak, 3),
                          note="40 calls of one b=1 UNet forward (10 per shape), cold L2, launch-to-launch")))
