"""Spatial self-attention (csrc/spatial_attn_tc.cu, wgmma + tensor-map TMA) through the C ABI against
  (a) the math statement of the reference seam in fp64 (attention.py:461-490 on the same fp16 inputs), and
  (b) the library kernel the reference's xformers call maps to on this torch (F.scaled_dot_product_attention).
Tolerance: fp16 output rounding (half an ulp of |o| <= 4 is 2e-3) plus fp16 rounding of the probabilities fed to P V.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from motionclone_b200 import ops  # noqa: E402


def _ref_fp64(q, k, v, heads, scale):
    B, N, C = q.shape
    dh = C // heads
    q4, k4, v4 = (t.double().view(B, N, heads, dh).transpose(1, 2) for t in (q, k, v))
    s = torch.matmul(q4, k4.transpose(-1, -2)) * scale
    lse = torch.logsumexp(s, dim=-1)
    o = torch.matmul(torch.softmax(s, dim=-1), v4)
    return o.transpose(1, 2).reshape(B, N, C), lse


CASES = [  # (frames, heads, tokens, head dim)
    (2, 8, 4096, 40), (2, 8, 1024, 80), (3, 8, 256, 160), (3, 8, 64, 160),   # the four UNet levels at 512 x 512
    (2, 8, 256, 40), (2, 8, 64, 80), (2, 8, 16, 160),                        # 128 x 128 (c2mini)
    (2, 8, 1024, 8), (2, 8, 256, 16), (2, 8, 64, 32), (1, 8, 16, 32), (1, 8, 4, 32),  # tiny-config widths
    (1, 2, 200, 64), (1, 3, 129, 40), (2, 1, 385, 80), (1, 1, 1, 16),       # ragged token counts
]


@pytest.mark.parametrize("B,H,N,dh", CASES)
@pytest.mark.parametrize("fused", [True, False])
def test_spatial_attention_forward(B, H, N, dh, fused):
    torch.manual_seed(N * 7 + dh)
    dev = torch.device("cuda:0")
    C = H * dh
    if fused:  # column blocks of one fused QKV projection, as the UNet calls it
        qkv = torch.randn(B, N, 3 * C, device=dev, dtype=torch.float16)
        q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    else:      # separate tensors with unrelated strides
        q = torch.randn(B, N, C, device=dev, dtype=torch.float16)
        k = torch.randn(B, N + 3, C + 8, device=dev, dtype=torch.float16)[:, :N, :C]
        v = (torch.randn(B, N, C, device=dev, dtype=torch.float16) * 2).contiguous()
    q = q * 2.0  # scores with a healthy spread (std ~ 2 after scaling)
    q = q.contiguous() if not fused else q
    scale = dh ** -0.5
    o, lse = ops.spatial_attention_forward(q, k, v, H, scale, want_lse=True)
    want, want_lse = _ref_fp64(q, k, v, H, scale)
    err = (o.double() - want).abs().max().item()
    err_lse = (lse.double() - want_lse).abs().max().item()
    lib = F.scaled_dot_product_attention(*(t.reshape(B, N, H, dh).transpose(1, 2) for t in (q, k, v)), scale=scale)
    err_lib = (lib.transpose(1, 2).reshape(B, N, C).double() - want).abs().max().item()
    print(f"B={B} H={H} N={N} dh={dh} fused={fused}: max abs err {err:.3e} (library kernel {err_lib:.3e}), lse {err_lse:.3e}")
    # |v| <= ~9 (2 sigma-scaled randn): output ulp/2 <= 4e-3; P in fp16 adds <= 2^-11 relative
    assert err < 8e-3 and err <= max(4e-3, 3 * err_lib)
    assert err_lse < 2e-3
    assert torch.isfinite(o).all()


def test_spatial_attention_large_scores():
    """Rows whose maximum jumps by orders of magnitude between key tiles: the online softmax must rescale the running
    O and row sum (held in registers) by exp2(m_old - m_new) on every tile where the maximum grows."""
    dev = torch.device("cuda:0")
    B, H, N, dh = 1, 2, 512, 40
    C = H * dh
    torch.manual_seed(0)
    q = torch.randn(B, N, C, device=dev, dtype=torch.float16)
    k = torch.randn(B, N, C, device=dev, dtype=torch.float16)
    k[:, 128:256] *= 4   # tile 1 dominates tile 0
    k[:, 384:] *= 12     # tile 3 dominates everything
    v = torch.randn(B, N, C, device=dev, dtype=torch.float16)
    o, lse = ops.spatial_attention_forward(q, k, v, H, 1.0, want_lse=True)
    want, want_lse = _ref_fp64(q, k, v, H, 1.0)
    assert (o.double() - want).abs().max().item() < 8e-3
    assert (lse.double() - want_lse).abs().max().item() < 1e-2


def test_spatial_attention_rejects_bad_arguments():
    dev = torch.device("cuda:0")
    x = torch.randn(1, 16, 8 * 24, device=dev, dtype=torch.float16)
    with pytest.raises(NotImplementedError):
        ops.spatial_attention_forward(x, x, x, 8, 1.0)  # head dim 24
    with pytest.raises(TypeError):
        ops.spatial_attention_forward(x.float(), x.float(), x.float(), 8, 1.0)


BWD_CASES = [(1, 8, 4096, 40), (2, 8, 1024, 80), (2, 8, 256, 160), (2, 8, 64, 160), (2, 8, 256, 40), (2, 8, 16, 160),
             (2, 8, 256, 16), (1, 8, 64, 32), (1, 2, 200, 64), (1, 3, 129, 40), (1, 1, 385, 80), (1, 2, 4, 8)]


@pytest.mark.parametrize("B,H,N,dh", BWD_CASES)
def test_spatial_attention_backward(B, H, N, dh):
    """dQ, dK, dV of the wgmma backward against fp64 autograd of the math statement on the same fp16 inputs; the
    library kernel's own error against the same truth is the yardstick."""
    torch.manual_seed(N * 3 + dh)
    dev = torch.device("cuda:0")
    C = H * dh
    qkv = torch.randn(B, N, 3 * C, device=dev, dtype=torch.float16)
    qkv[..., :C] *= 2.0
    d_o = torch.randn(B, N, C, device=dev, dtype=torch.float16)
    scale = dh ** -0.5
    x = qkv.clone().requires_grad_(True)
    o = ops.SpatialAttentionFusedTC.apply(x, H, scale)
    (g,) = torch.autograd.grad(o, x, d_o)
    # separate-view form must give the same gradient (autograd accumulates the three views)
    x2 = qkv.clone().requires_grad_(True)
    o2 = ops.SpatialAttentionTC.apply(x2[..., :C], x2[..., C:2 * C], x2[..., 2 * C:], H, scale)
    (g2,) = torch.autograd.grad(o2, x2, d_o)
    assert torch.equal(g, g2)
    # truth: fp64 autograd
    xd = qkv.double().requires_grad_(True)
    q4, k4, v4 = (xd[..., i * C:(i + 1) * C].reshape(B, N, H, dh).transpose(1, 2) for i in range(3))
    od = torch.matmul(torch.softmax(torch.matmul(q4, k4.transpose(-1, -2)) * scale, dim=-1), v4)
    (gd,) = torch.autograd.grad(od.transpose(1, 2).reshape(B, N, C), xd, d_o.double())
    # yardstick: the library kernel in fp16
    xl = qkv.clone().requires_grad_(True)
    ql, kl, vl = (xl[..., i * C:(i + 1) * C].reshape(B, N, H, dh).transpose(1, 2) for i in range(3))
    ol = F.scaled_dot_product_attention(ql, kl, vl, scale=scale).transpose(1, 2).reshape(B, N, C)
    (gl,) = torch.autograd.grad(ol, xl, d_o)
    for name, sl in (("dq", slice(0, C)), ("dk", slice(C, 2 * C)), ("dv", slice(2 * C, 3 * C))):
        ref = gd[..., sl]
        err = (g[..., sl].double() - ref).abs().max().item() / ref.abs().max().item()
        err_lib = (gl[..., sl].double() - ref).abs().max().item() / ref.abs().max().item()
        print(f"B={B} H={H} N={N} dh={dh} {name}: rel max err {err:.3e} (library {err_lib:.3e})")
        assert err < max(4e-3, 3 * err_lib), name
    assert torch.isfinite(g).all()
