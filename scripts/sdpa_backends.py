"""Which library SDPA backend is fastest on the H100 for the spatial attention shapes of the SD1.5 UNet (fwd and fwd+bwd)?"""
import torch, time
from torch.nn.attention import sdpa_kernel, SDPBackend
import torch.nn.functional as F
dev = "cuda"
def bench(fn, n=10):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n
shapes = [("self64", 16, 8, 4096, 4096, 40), ("self32", 16, 8, 1024, 1024, 80), ("self16", 16, 8, 256, 256, 160), ("self8", 16, 8, 64, 64, 160),
          ("cross64", 1, 8, 65536, 77, 40), ("cross32", 1, 8, 16384, 77, 80), ("cross16", 1, 8, 4096, 77, 160)]
for name, B, H, Nq, Nk, dh in shapes:
    # strided like the pipeline: q/k/v views of a fused projection
    if Nq == Nk:
        qkv = torch.randn(B, Nq, 3, H, dh, device=dev, dtype=torch.float16)
        q, k, v = (qkv[:, :, i].transpose(1, 2) for i in range(3))
    else:
        q = torch.randn(B, Nq, H, dh, device=dev, dtype=torch.float16).transpose(1, 2)
        k = torch.randn(B, Nk, H, dh, device=dev, dtype=torch.float16).transpose(1, 2)
        v = torch.randn(B, Nk, H, dh, device=dev, dtype=torch.float16).transpose(1, 2)
    flops = 4 * B * H * Nq * Nk * dh
    row = [name]
    for be in (SDPBackend.CUDNN_ATTENTION, SDPBackend.FLASH_ATTENTION, SDPBackend.EFFICIENT_ATTENTION):
        try:
            with sdpa_kernel([be]):
                with torch.no_grad():
                    t_f = bench(lambda: F.scaled_dot_product_attention(q, k, v, scale=dh ** -0.5))
                qg, kg, vg = (t.detach().clone().requires_grad_(True) for t in (q, k, v))
                def fb():
                    o = F.scaled_dot_product_attention(qg, kg, vg, scale=dh ** -0.5)
                    torch.autograd.grad(o, (qg, kg, vg), torch.ones_like(o))
                t_fb = bench(fb)
            row.append(f"{be.name[:6]}: fwd {t_f:.3f} ms ({flops/t_f/1e9:.0f} TF/s) fwd+bwd {t_fb:.3f} ms")
        except Exception as e:
            row.append(f"{be.name[:6]}: ERR {str(e)[:50]}")
    print(" | ".join(row), flush=True)
