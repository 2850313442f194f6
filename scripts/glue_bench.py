"""Microbenchmark of the memory-bound glue kernels (GroupNorm NHWC fwd/bwd, LayerNorm, GEGLU) at UNet shapes
(16 x 512 x 512): achieved GB/s of ALGORITHMIC bytes (GroupNorm fwd: 2 reads + 1 write of the tensor; bwd: x, dz read
twice + dx written; LayerNorm: 1 read + 1 write; GEGLU: [T, 2I] read + [T, I] written) against the measured HBM peak.
In-situ style (no L2 flush: the producer's output is usually L2-warm in the UNet too) and cold (L2 flushed)."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from motionclone_b200 import ops

dev = torch.device("cuda:0")
peak = 3350.0  # GB/s, H100 SXM data sheet (HBM3); MEASURED_PEAKS.json overrides it
try:
    peak = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    pass
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)


def timeit(fn, cold, iters=15):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(iters):
        if cold:
            flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def report(name, shape, nbytes, fn):
    r = dict(kernel=name, shape=shape, MB=round(nbytes / 1e6, 1))
    for cold in (True, False):
        ms = timeit(fn, cold)
        r["cold" if cold else "warm"] = dict(us=round(ms * 1e3, 1), GBs=round(nbytes / 1e6 / ms, 0), frac=round(nbytes / 1e6 / ms / peak, 3))
    print(json.dumps(r), flush=True)


for N, C, H, W in ((16, 320, 64, 64), (16, 640, 64, 64), (16, 960, 64, 64), (32, 320, 64, 64), (16, 640, 32, 32), (16, 1280, 32, 32),
                   (16, 1280, 16, 16), (16, 2560, 16, 16), (16, 1280, 8, 8)):
    x = torch.randn(N, C, H, W, device=dev, dtype=torch.float16).contiguous(memory_format=torch.channels_last)
    w = torch.randn(C, device=dev, dtype=torch.float16)
    b = torch.randn(C, device=dev, dtype=torch.float16)
    cb = torch.randn(N // 16, C, device=dev, dtype=torch.float16)
    nb = x.numel() * 2
    report("groupnorm_fwd_silu_temb", [N, C, H, W], 3 * nb, lambda: ops.groupnorm_nhwc(x, w, b, 32, 1e-5, True, cb))
    xg = x.clone().requires_grad_(True)
    y = ops.GroupNormNHWCFn.apply(xg, w, b, cb, 32, 1e-5, True)
    dz = torch.randn_like(x)
    report("groupnorm_bwd_silu_temb", [N, C, H, W], 5 * nb, lambda: torch.autograd.grad(y, xg, dz, retain_graph=True))
for rows, C in ((65536, 320), (16384, 640), (4096, 1280)):
    x = torch.randn(rows, C, device=dev, dtype=torch.float16)
    w = torch.randn(C, device=dev, dtype=torch.float16)
    b = torch.randn(C, device=dev, dtype=torch.float16)
    report("layernorm", [rows, C], 2 * x.numel() * 2, lambda: ops.layernorm(x, w, b, 1e-5))
for T, I in ((65536, 1280), (16384, 2560), (4096, 5120)):
    x = torch.randn(T, 2 * I, device=dev, dtype=torch.float16)
    report("geglu", [T, I], 3 * T * I * 2, lambda: ops.geglu(x))
