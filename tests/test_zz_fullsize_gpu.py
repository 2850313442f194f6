"""Properties at BASELINE.json's FULL layer sizes (16 x 512 x 512: 16 frames, 64 x 64 latent positions, C = 320) that need
no oracle run of that size: the hot path is a batch of independent (position, head) / (query row) / (frame) problems, so
permuting the independent axis of the inputs must permute the outputs BIT FOR BIT (no dependence on which tile, CTA or
pipeline stage a unit lands in, no cross-unit leakage, deterministic reductions), and the fused epilogues must agree
with their stand-alone statements. Spatial and text cross-attention are also held to fp64 math on a sample (the first
and last frame, a few thousand query rows), computed one head at a time. The oracle-checked versions of the same kernels at oracle-sized inputs are in
test_kernels_gpu.py; end-to-end parity against the reference fixtures is in test_pipeline_gpu.py.
(File name sorts last on purpose: these are the heaviest tests.)"""
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import mc_oracle as O  # noqa: E402


def _ops():
    from motionclone_b200 import ops
    return ops


def _dev():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    return torch.device("cuda:0")


L, H, C, D = 16, 8, 320, 64 * 64  # frames, heads, channels, positions of the down0 / up3 motion modules


def test_temporal_attention_full_size_position_permutation_and_top1():
    """VersatileAttention core (models/motion_module.py:309-332) + top-1 extraction (utils/motionclone_functions.py:79)
    + gathered probabilities (:91-92), forward and backward, at [1, 16, 4096, 320]."""
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(11)
    qkv = torch.randn(1, L, D, 3 * C, generator=g).to(dev, torch.float16)
    perm = torch.randperm(D, generator=g).to(dev)
    qkv_p = qkv[:, :, perm].contiguous()
    scale = (C // H) ** -0.5
    split = lambda t: (t[..., :C], t[..., C:2 * C], t[..., 2 * C:])  # noqa: E731

    o, probs, top, _ = ops.temporal_attention_forward(*split(qkv), H, scale, want_probs=True, want_top1=True)
    o_p, probs_p, top_p, _ = ops.temporal_attention_forward(*split(qkv_p), H, scale, want_probs=True, want_top1=True)
    assert torch.equal(o_p, o[:, :, perm]), "attention output depends on where a position sits in the launch"
    assert torch.equal(probs_p, probs[perm]) and torch.equal(top_p[1], top[1][perm]) and torch.equal(top_p[0], top[0][perm])
    # fused top-1 epilogue == lowest-index argmax of the kernel's own probabilities (the index-set bar), full size
    wv, wi = O.top1_lowest_index(probs)
    assert torch.equal(top[1], wi) and torch.equal(top[0], wv)
    # gathered-probability epilogue == torch.gather on the probabilities
    idx = torch.randint(0, L, (D, H, L, 1), generator=g).to(dev, torch.uint8)
    _, _, _, gathered = ops.temporal_attention_forward(*split(qkv), H, scale, gather_idx=idx)
    assert torch.equal(gathered, torch.gather(probs, -1, idx.long()))
    # rows of a softmax sum to one (fp16 rounding of 16 terms)
    assert (probs.float().sum(-1) - 1).abs().max().item() <= 4e-3

    # backward: dO branch + one-hot gathered branch (closed form of gather + mse_loss backward)
    d_o = torch.randn(1, L, D, C, generator=g).to(dev, torch.float16)
    d_g = (0.01 * torch.randn(D, H, L, 1, generator=g)).to(dev, torch.float16)
    dqkv = ops.temporal_attention_backward(*split(qkv), H, scale, d_o, None, idx, d_g, return_fused=True)
    dqkv_p = ops.temporal_attention_backward(*split(qkv_p), H, scale, d_o[:, :, perm].contiguous(), None,
                                             idx[perm].contiguous(), d_g[perm].contiguous(), return_fused=True)
    assert torch.isfinite(dqkv).all()
    assert torch.equal(dqkv_p, dqkv[:, :, perm]), "attention gradient depends on where a position sits in the launch"


def _attn_fp64_by_head(q, k, v, d_o, heads, scale):
    """fp64 softmax(scale q k^T) v of ONE frame, one head at a time (a 4096 x 4096 fp64 score matrix is 134 MB per head):
    q, d_o [Nq, C], k, v [Nk, C] fp16 -> o [Nq, C], lse [heads, Nq], and with d_o the gradients (dq, dk, dv)."""
    Nq, Cq = q.shape
    dh = Cq // heads
    o = torch.empty(Nq, Cq, dtype=torch.float64, device=q.device)
    lse = torch.empty(heads, Nq, dtype=torch.float64, device=q.device)
    grads = tuple(torch.empty(t.shape, dtype=torch.float64, device=q.device) for t in (q, k, v)) if d_o is not None else None
    for h in range(heads):
        cols = slice(h * dh, (h + 1) * dh)
        qh, kh, vh = (t[:, cols].double().requires_grad_(d_o is not None) for t in (q, k, v))
        s = qh @ kh.T * scale
        lse[h] = torch.logsumexp(s, -1).detach()
        oh = torch.softmax(s, -1) @ vh
        o[:, cols] = oh.detach()
        if d_o is not None:
            for dst, gr in zip(grads, torch.autograd.grad(oh, (qh, kh, vh), d_o[:, cols].double())):
                dst[:, cols] = gr
    return o, lse, grads


def _sdpa_rows(q, k, v, d_o, heads, scale):
    """the library's fp16 attention on [B, N, C] tensors (and, with d_o, its gradients): the yardstick of the bars."""
    leaves = [t.detach().clone().requires_grad_(d_o is not None) for t in (q, k, v)]
    B, Nq, Cq = q.shape
    o = torch.nn.functional.scaled_dot_product_attention(
        *(t.reshape(B, -1, heads, Cq // heads).transpose(1, 2) for t in leaves), scale=scale).transpose(1, 2).reshape(B, Nq, Cq)
    return o.detach(), (torch.autograd.grad(o, leaves, d_o) if d_o is not None else None)


# spatial self-attention at 16 x 512 x 512: (tokens per frame, channels) of the four UNet levels, 8 heads
SPATIAL_LEVELS = [(D, C), (D // 4, 2 * C), (D // 16, 4 * C), (D // 64, 4 * C)]


@pytest.mark.parametrize("N,Cs", SPATIAL_LEVELS)
def test_spatial_attention_full_size_forward(N, Cs):
    """attn1 forward (models/attention.py:271-278 -> :535-542) at 32 frames (the CFG pair of 16): fp64 parity on the first
    and last frame, bitwise invariance under a frame permutation, bitwise identical repeated runs."""
    ops, dev = _ops(), _dev()
    B, dh = 2 * L, Cs // H
    g = torch.Generator(device=dev).manual_seed(15 + N)
    qkv = torch.randn(B, N, 3 * Cs, generator=g, device=dev, dtype=torch.float16)
    perm = torch.randperm(B, generator=g, device=dev)
    scale = dh ** -0.5
    split = lambda t: (t[..., :Cs], t[..., Cs:2 * Cs], t[..., 2 * Cs:])  # noqa: E731
    o, lse = ops.spatial_attention_forward(*split(qkv), H, scale, want_lse=True)
    o2, lse2 = ops.spatial_attention_forward(*split(qkv), H, scale, want_lse=True)
    assert torch.equal(o, o2) and torch.equal(lse, lse2), "spatial attention forward is not run-to-run deterministic"
    o_p, lse_p = ops.spatial_attention_forward(*split(qkv[perm].contiguous()), H, scale, want_lse=True)
    assert torch.equal(o_p, o[perm]) and torch.equal(lse_p, lse[perm]), "output depends on where a frame sits in the grid"
    ends = [0, B - 1]
    lib_o, _ = _sdpa_rows(*split(qkv[ends]), None, H, scale)
    for i, b in enumerate(ends):
        ref_o, ref_lse, _ = _attn_fp64_by_head(*split(qkv[b]), None, H, scale)
        err = (o[b].double() - ref_o).abs().max().item()
        err_lib = (lib_o[i].double() - ref_o).abs().max().item()
        err_lse = (lse[b].double() - ref_lse).abs().max().item()
        print(f"[{B}, {N}, {Cs}] frame {b}: o {err:.3e} (library {err_lib:.3e}) lse {err_lse:.3e}")
        assert err < 8e-3 and err <= max(4e-3, 3 * err_lib) and err_lse < 2e-3


@pytest.mark.parametrize("N,Cs", SPATIAL_LEVELS)
def test_spatial_attention_full_size_backward(N, Cs):
    """attn1 backward through SpatialAttentionFusedTC at the 16 frames of the guided pass: fp64 parity of dq | dk | dv on
    the first and last frame, bitwise invariance under a frame permutation, bitwise identical repeated runs (the dQ and
    dK/dV kernels use no atomics)."""
    ops, dev = _ops(), _dev()
    B, dh = L, Cs // H
    g = torch.Generator(device=dev).manual_seed(16 + N)
    qkv = torch.randn(B, N, 3 * Cs, generator=g, device=dev, dtype=torch.float16)
    d_o = torch.randn(B, N, Cs, generator=g, device=dev, dtype=torch.float16)
    perm = torch.randperm(B, generator=g, device=dev)
    scale = dh ** -0.5

    def run(x, dd):
        xg = x.clone().requires_grad_(True)
        o = ops.SpatialAttentionFusedTC.apply(xg, H, scale)
        (dx,) = torch.autograd.grad(o, xg, dd)
        return o.detach(), dx

    o, dqkv = run(qkv, d_o)
    o2, dqkv2 = run(qkv, d_o)
    assert torch.equal(o, o2) and torch.equal(dqkv, dqkv2), "spatial attention backward is not run-to-run deterministic"
    o_p, dqkv_p = run(qkv[perm].contiguous(), d_o[perm].contiguous())
    assert torch.equal(o_p, o[perm]) and torch.equal(dqkv_p, dqkv[perm]), "gradient depends on where a frame sits in the grid"
    assert torch.isfinite(dqkv).all()
    split = lambda t: (t[..., :Cs], t[..., Cs:2 * Cs], t[..., 2 * Cs:])  # noqa: E731
    ends = [0, B - 1]
    _, lib_g = _sdpa_rows(*split(qkv[ends]), d_o[ends], H, scale)
    for i, b in enumerate(ends):
        _, _, ref_g = _attn_fp64_by_head(*split(qkv[b]), d_o[b], H, scale)
        for name, got, ref, lib in zip(("dq", "dk", "dv"), split(dqkv[b]), ref_g, lib_g):
            top = ref.abs().max().item()
            err = (got.double() - ref).abs().max().item() / top
            err_lib = (lib[i].double() - ref).abs().max().item() / top
            print(f"[{B}, {N}, {Cs}] frame {b} {name}: rel max err {err:.3e} (library {err_lib:.3e})")
            assert err < max(4e-3, 3 * err_lib), (b, name)


def test_cross_attention_full_size_row_permutation():
    """attn2 on the wgmma kernels (models/attention.py:280-285 -> :535-542): 16 x 4096 query rows against the 77 text keys."""
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(12)
    nq = L * D
    q = torch.randn(1, nq, C, generator=g).to(dev, torch.float16)
    kv = torch.randn(1, 77, 2 * C, generator=g).to(dev, torch.float16)
    k, v = kv[..., :C], kv[..., C:]
    d_o = torch.randn(1, nq, C, generator=g).to(dev, torch.float16)
    perm = torch.randperm(nq, generator=g).to(dev)
    scale = (C // H) ** -0.5
    o = ops.cross_attention_forward(q, k, v, H, scale)
    o_p = ops.cross_attention_forward(q[:, perm].contiguous(), k, v, H, scale)
    assert torch.isfinite(o).all()
    assert torch.equal(o_p, o[:, perm]), "cross-attention output depends on the row's place in its 128-row tile"
    dq = ops.cross_attention_backward(q, k, v, d_o, H, scale)
    dq_p = ops.cross_attention_backward(q[:, perm].contiguous(), k, v, d_o[:, perm].contiguous(), H, scale)
    assert torch.isfinite(dq).all()
    assert torch.equal(dq_p, dq[:, perm])
    # a convex combination of the value rows: every output lies inside the per-channel range of V (+ one fp16 ulp)
    vh = v.float()
    assert (o.float() <= vh.amax(dim=1, keepdim=True) + 1e-2).all() and (o.float() >= vh.amin(dim=1, keepdim=True) - 1e-2).all()
    # fp64 parity on a sample of rows (rows are independent problems), next to the library kernel's own error
    rows = perm[:4096]
    ref_o, _, ref_g = _attn_fp64_by_head(q[0, rows], k[0], v[0], d_o[0, rows], H, scale)
    lib_o, lib_g = _sdpa_rows(q[:, rows], k, v, d_o[:, rows], H, scale)
    err = (o[0, rows].double() - ref_o).abs().max().item()
    err_lib = (lib_o[0].double() - ref_o).abs().max().item()
    top = ref_g[0].abs().max().item()
    err_dq = (dq[0, rows].double() - ref_g[0]).abs().max().item() / top
    err_dq_lib = (lib_g[0][0].double() - ref_g[0]).abs().max().item() / top
    print(f"cross-attention, {rows.numel()} sampled rows: o {err:.3e} (library {err_lib:.3e}), "
          f"dq rel {err_dq:.3e} (library {err_dq_lib:.3e})")
    assert err < 8e-3 and err <= max(4e-3, 3 * err_lib)
    assert err_dq < max(4e-3, 3 * err_dq_lib)


def test_groupnorm_full_size_frame_permutation_and_determinism():
    """InflatedGroupNorm + temb add + SiLU (models/resnet.py:21-29, :186-204) at [16, 320, 64, 64], forward and input
    gradient: frames are independent; split partials are folded in a fixed order whichever CTA finishes last."""
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(13)
    x = (torch.randn(L, C, 64, 64, generator=g) * 2 + 0.5).to(dev, torch.float16).contiguous(memory_format=torch.channels_last)
    w = (1 + 0.1 * torch.randn(C, generator=g)).to(dev, torch.float16)
    b = (0.1 * torch.randn(C, generator=g)).to(dev, torch.float16)
    temb = torch.randn(1, C, generator=g).to(dev, torch.float16)
    dz = torch.randn(L, C, 64, 64, generator=g).to(dev, torch.float16).contiguous(memory_format=torch.channels_last)
    perm = torch.randperm(L, generator=g).to(dev)

    def run(xx, dd):
        xg = xx.clone().requires_grad_(True)
        y = ops.GroupNormNHWCFn.apply(xg, w, b, temb, 32, 1e-5, True)
        (dx,) = torch.autograd.grad(y, xg, dd)
        return y.detach(), dx

    y, dx = run(x, dz)
    y2, dx2 = run(x, dz)
    assert torch.equal(y, y2) and torch.equal(dx, dx2), "GroupNorm is not run-to-run deterministic"
    xp = x[perm].contiguous(memory_format=torch.channels_last)
    dp = dz[perm].contiguous(memory_format=torch.channels_last)
    yp, dxp = run(xp, dp)
    assert torch.equal(yp, y[perm]) and torch.equal(dxp, dx[perm])
    with torch.no_grad():
        assert torch.equal(ops.groupnorm_nhwc(x, w, b, 32, 1e-5, True, temb), y)  # inference entry point, same kernels
    # the normalised pre-activation has zero mean / unit variance per (frame, group): check through the no-SiLU path
    with torch.no_grad():
        z = ops.groupnorm_nhwc(x, torch.ones_like(w), torch.zeros_like(b), 32, 1e-5, False)
    zz = z.float().permute(0, 2, 3, 1).reshape(L, 64 * 64, 32, C // 32)
    assert zz.mean(dim=(1, 3)).abs().max().item() <= 2e-3
    assert (zz.var(dim=(1, 3), unbiased=False) - 1).abs().max().item() <= 5e-3


def test_geglu_lookup_table_path_full_size():
    """diffusers FeedForward GEGLU (models/attention.py:211) at the [65536 / 4, 8 * 320] projection of a C = 320 layer: this
    size takes the shared-memory lookup-table kernel (csrc/norm_act.cu), which must reproduce the eager pair
    `F.gelu(gate)` (fp16) -> `h * gelu` (fp16) with the same rounding points."""
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(14)
    T, I = 16384, 4 * C
    x = (torch.randn(T, 2 * I, generator=g) * 2).to(dev, torch.float16)
    with torch.no_grad():
        y = ops.geglu(x)
    h, gate = x.chunk(2, dim=-1)
    eager = h * torch.nn.functional.gelu(gate)
    ref = h.float() * torch.nn.functional.gelu(gate.float())
    assert (y.float() - ref).abs().max().item() <= max(1.6e-2, 1.5 * (eager.float() - ref).abs().max().item())
    assert (y != eager).float().mean().item() < 1e-3
    # and bit-identical to the erf kernel (small launches take it): same device code built the table
    small = ops.geglu(x[:256].contiguous())
    assert torch.equal(small, y[:256])
