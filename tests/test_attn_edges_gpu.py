"""Edges of the wgmma attention kernels (csrc/spatial_attn_tc.cu: forward of spatial self- and text cross-attention;
csrc/spatial_attn_bwd_tc.cu: spatial dQ / dK / dV, cross-attention dQ), each checked against fp64 math on the same fp16
inputs:
  * score offsets: every score of a row shifted by delta nats (softmax unchanged, log-sum-exp shifted), so the kernels
    see very negative and very positive row statistics, on aligned and ragged token counts;
  * rows with an exact answer: one-hot rows (o and dV are copies of input rows, bit for bit), uniform rows (q = 0) and
    constant values (dQ = dK = 0), which catch tile-column and layout mistakes that a tolerance would absorb;
  * token and key counts around every tile edge the kernels have (32, 64, 80, 128 rows);
  * stores: every output written into the interior of a canary-filled buffer with padded strides, through the C ABI.
The bars are those of test_spatial_attn_gpu.py: forward <= 8e-3 abs and <= 3x the library kernel's own error, lse
<= 2e-3 abs, gradients <= max(4e-3, 3x library) of max|reference|; tighter where the answer is exact.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from motionclone_b200 import _lib, ops  # noqa: E402

HEAD_DIMS = ops.SPATIAL_ATTN_HEAD_DIMS


def _dev():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    return torch.device("cuda:0")


# ---------------------------------------------------------------------------------------------------------------
# references and bars
# ---------------------------------------------------------------------------------------------------------------
def _ref(q, k, v, d_o, H, scale):
    """fp64 softmax(scale q k^T) v per head on the given fp16 values: q [B, Nq, C], k / v [B, Nk, C], d_o [B, Nq, C] or
    None -> o [B, Nq, C], lse [B, H, Nq], (dq, dk, dv) or None."""
    B, Nq, C = q.shape
    Nk, dh = k.shape[1], C // H
    leaves = [t.double().requires_grad_(d_o is not None) for t in (q, k, v)]
    qh, kh, vh = (t.reshape(B, -1, H, dh).transpose(1, 2) for t in leaves)
    s = qh @ kh.transpose(-1, -2) * scale
    lse = torch.logsumexp(s, -1)
    o = (torch.softmax(s, -1) @ vh).transpose(1, 2).reshape(B, Nq, C)
    grads = torch.autograd.grad(o, leaves, d_o.double()) if d_o is not None else None
    return o.detach(), lse.detach(), grads


def _library(q, k, v, d_o, H, scale):
    """The library's fp16 attention (F.scaled_dot_product_attention) and its gradients: the yardstick of the bars."""
    leaves = [t.detach().clone().requires_grad_(d_o is not None) for t in (q, k, v)]
    B, Nq, C = q.shape
    o = F.scaled_dot_product_attention(*(t.reshape(B, -1, H, C // H).transpose(1, 2) for t in leaves), scale=scale)
    o = o.transpose(1, 2).reshape(B, Nq, C)
    grads = torch.autograd.grad(o, leaves, d_o) if d_o is not None else None
    return o.detach(), grads


def _rel(x, ref, cols=None):
    """max |x - ref| / max |ref|; the absolute error where the reference is exactly zero (one key: dS = 0)."""
    if cols is not None:
        x, ref = x[..., cols], ref[..., cols]
    err, top = (x.double() - ref).abs().max().item(), ref.abs().max().item()
    return err / top if top > 0 else err


def _check_forward(tag, o, ref_o, lib_o, lse=None, ref_lse=None):
    err = (o.double() - ref_o).abs().max().item()
    err_lib = (lib_o.double() - ref_o).abs().max().item()
    err_lse = (lse.double() - ref_lse).abs().max().item() if lse is not None else 0.0
    print(f"{tag}: o {err:.3e} (library {err_lib:.3e}) lse {err_lse:.3e}")
    assert torch.isfinite(o).all(), tag
    assert err < 8e-3 and err <= max(4e-3, 3 * err_lib), (tag, err, err_lib)
    if lse is not None:
        assert torch.isfinite(lse).all(), tag
        assert err_lse < 2e-3, (tag, err_lse)


def _check_grads(tag, got, ref, lib, cols=None):
    """got / ref / lib: {name: gradient}; `cols` restricts the dk comparison to some channels."""
    errs = {n: (_rel(got[n], ref[n], cols if n == "dk" else None), _rel(lib[n], ref[n], cols if n == "dk" else None))
            for n in got}
    print(tag + ": " + " ".join(f"{n} {e:.3e} (library {el:.3e})" for n, (e, el) in errs.items()))
    for n, (e, el) in errs.items():
        assert torch.isfinite(got[n]).all(), (tag, n, "non-finite gradient")
        assert e < max(4e-3, 3 * el), (tag, n, e, el)


def _spatial(q, k, v, d_o, H, scale):
    """kernel forward (o, lse) and, with d_o, backward {dq, dk, dv} through the ops entry points."""
    o, lse = ops.spatial_attention_forward(q, k, v, H, scale, want_lse=True)
    if d_o is None:
        return o, lse, None
    C = q.shape[-1]
    g = ops.spatial_attention_backward(q, k, v, o, lse, d_o, H, scale)
    return o, lse, {"dq": g[..., :C], "dk": g[..., C:2 * C], "dv": g[..., 2 * C:]}


def _fused(q, k, v, dev):
    """q | k | v as the column blocks of one fused [B, N, 3C] fp16 buffer (the UNet's projection layout)."""
    C = q.shape[-1]
    qkv = torch.cat([q, k, v], -1).to(dev, torch.float16)
    return qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]


def _kv(k, v, dev):
    """text K | V as the column blocks of one [B, Nk, 2C] buffer."""
    C = k.shape[-1]
    kv = torch.cat([k, v], -1).to(dev, torch.float16)
    return kv[..., :C], kv[..., C:]


def _quantized(shape, g):
    """Nonzero multiples of 1/16 in [-4, 4]: every product of two and every sum of up to 4096 such products is exact in
    fp32, whatever the summation order, and no value has a sign-of-zero ambiguity."""
    mag = torch.randint(1, 65, shape, generator=g).double()
    sign = torch.randint(0, 2, shape, generator=g).double() * 2 - 1
    return mag * sign / 16


def _ulp16(x):
    """fp16 spacing at |x| (x fp64): 2^(e - 11) with |x| = m 2^e, m in [0.5, 1); 2^-24 in the subnormal range."""
    _, e = torch.frexp(x.abs())
    ulp = torch.exp2((e - 11).double()).clamp_min(2.0 ** -24)
    return torch.where(x == 0, torch.full_like(ulp, 2.0 ** -24), ulp)


# ---------------------------------------------------------------------------------------------------------------
# 1. score offsets
# ---------------------------------------------------------------------------------------------------------------
DELTAS = [-100.0, -60.0, -20.0, -8.0, 0.0, 8.0, 30.0]
OFFSET_SPATIAL = [  # (frames, heads, tokens, head dim): ragged and 64-aligned token counts
    (2, 2, 16, 160), (2, 2, 40, 40), (1, 2, 129, 40), (2, 2, 160, 80), (1, 2, 200, 8), (1, 2, 385, 80),
    (2, 2, 64, 8), (1, 2, 256, 160), (1, 2, 256, 40)]
OFFSET_CROSS = [  # (batch, heads, queries, keys, head dim)
    (1, 2, 200, 77, 40), (1, 2, 129, 16, 160), (1, 2, 64, 80, 8), (1, 2, 300, 65, 80), (2, 2, 100, 64, 40)]


def _offset_inputs(B, Nq, Nk, H, dh, delta, seed, kappa=1.0):
    """randn q, k, v, d_o with channel 0 of every head carrying kappa in every key and delta / (kappa scale) in every
    query: every scaled score of a row is shifted by the same delta (up to fp16 rounding of the query value), which
    moves the row's log-sum-exp by delta and leaves its softmax unchanged."""
    g = torch.Generator().manual_seed(seed)
    C, scale = H * dh, dh ** -0.5
    q, k, v = (torch.randn(B, n, C, generator=g) for n in (Nq, Nk, Nk))
    d_o = torch.randn(B, Nq, C, generator=g)
    k[..., ::dh] = kappa
    q[..., ::dh] = delta / (kappa * scale)
    return q, k, v, d_o, scale


@pytest.mark.parametrize("delta", DELTAS)
@pytest.mark.parametrize("B,H,N,dh", OFFSET_SPATIAL)
def test_spatial_attention_score_offset(B, H, N, dh, delta):
    """Forward and backward with every row's scores shifted by delta. The dQ kernel scores the zero-filled keys past the
    end of a ragged last tile against the row's own statistics: unmasked, p = exp(-lse) overflows at very negative lse
    and inf x 0 turns dQ into NaN."""
    dev = _dev()
    q, k, v, d_o, scale = _offset_inputs(B, N, N, H, dh, delta, seed=N * 13 + dh)
    q, k, v = _fused(q, k, v, dev)
    d_o = d_o.to(dev, torch.float16)
    o, lse, got = _spatial(q, k, v, d_o, H, scale)
    ref_o, ref_lse, (gq, gk, gv) = _ref(q, k, v, d_o, H, scale)
    lib_o, (lq, lk, lv) = _library(q, k, v, d_o, H, scale)
    tag = f"B={B} H={H} N={N} dh={dh} delta={delta:+g}"
    # the offset channel of dK is q_c * column sums of dS (q_c up to ~1.3e3): its magnitude would set the relative bar
    # of the whole tensor, so dK is measured on the other channels
    cols = torch.tensor([c for c in range(H * dh) if c % dh], device=dev)
    _check_grads(tag, got, {"dq": gq, "dk": gk, "dv": gv}, {"dq": lq, "dk": lk, "dv": lv}, cols=cols)
    _check_forward(tag, o, ref_o, lib_o, lse, ref_lse)


@pytest.mark.parametrize("delta", DELTAS)
@pytest.mark.parametrize("B,H,Nq,Nk,dh", OFFSET_CROSS)
def test_cross_attention_score_offset(B, H, Nq, Nk, dh, delta):
    """Text cross-attention forward (two key tiles above 64 keys) and dQ (the whole key axis as one tile) with every
    row's scores shifted by delta."""
    dev = _dev()
    q, k, v, d_o, scale = _offset_inputs(B, Nq, Nk, H, dh, delta, seed=Nq * 17 + Nk + dh)
    q, d_o = q.to(dev, torch.float16), d_o.to(dev, torch.float16)
    k, v = _kv(k, v, dev)
    o = ops.cross_attention_forward(q, k, v, H, scale)
    dq = ops.cross_attention_backward(q, k, v, d_o, H, scale)
    ref_o, _, (gq, _, _) = _ref(q, k, v, d_o, H, scale)
    lib_o, (lq, _, _) = _library(q, k, v, d_o, H, scale)
    tag = f"B={B} H={H} Nq={Nq} Nk={Nk} dh={dh} delta={delta:+g}"
    _check_grads(tag, {"dq": dq}, {"dq": gq}, {"dq": lq})
    _check_forward(tag, o, ref_o, lib_o)


# ---------------------------------------------------------------------------------------------------------------
# 2. rows with an exact answer
# ---------------------------------------------------------------------------------------------------------------
ONEHOT_SCALE = 40.0


def _onehot_inputs(B, Nq, Nk, H, dh, seed):
    """Key j encodes its index in binary over channel pairs (b, 1 - b); query i of (frame, head) copies key tau(i).
    Then s[i, tau(i)] = bits and every other score is <= bits - 1, exactly in fp16 and fp32; at scale 40 the dominant
    key leads by >= 40 nats, so the softmax is one-hot to far below fp16 resolution. tau covers every key (a permutation
    when Nq == Nk), so the dominant key visits every column of every key tile: the MUFU and the polynomial exp2 columns
    and the partial last tile. v and d_o are quantized (_quantized), which makes every product in the backward exact."""
    g = torch.Generator().manual_seed(seed)
    bits = max(1, (Nk - 1).bit_length())
    assert 2 * bits <= dh, "head dim too small for the key code"
    code = ((torch.arange(Nk)[:, None] >> torch.arange(bits)) & 1).double()
    enc = torch.zeros(Nk, dh, dtype=torch.float64)
    enc[:, 0:2 * bits:2], enc[:, 1:2 * bits:2] = code, 1 - code
    reps = -(-Nq // Nk)
    tau = torch.stack([torch.stack([torch.cat([torch.randperm(Nk, generator=g) for _ in range(reps)])[:Nq]
                                    for _ in range(H)]) for _ in range(B)])  # [B, H, Nq]
    k = enc.repeat(B, 1, H)                                                  # [B, Nk, H * dh]
    q = enc[tau].permute(0, 2, 1, 3).reshape(B, Nq, H * dh)                 # q[b, i, h] = enc[tau[b, h, i]]
    v = _quantized((B, Nk, H * dh), g)
    d_o = _quantized((B, Nq, H * dh), g)
    return q, k, v, d_o, tau, bits


def _gather_rows(x, idx, dh):
    """x [B, N, H*dh], idx [B, H, M] -> y [B, M, H*dh] with y[b, i, h] = x[b, idx[b, h, i], h]."""
    B, N, C = x.shape
    H = C // dh
    xh = x.reshape(B, N, H, dh).permute(0, 2, 1, 3)                          # [B, H, N, dh]
    y = torch.gather(xh, 2, idx[..., None].expand(-1, -1, -1, dh))
    return y.permute(0, 2, 1, 3).reshape(B, -1, C)


ONEHOT_SPATIAL = [(2, 2, 16, 8), (1, 2, 129, 16), (1, 2, 100, 32), (2, 2, 200, 40), (1, 2, 256, 64), (1, 2, 385, 80),
                  (2, 2, 64, 160), (1, 2, 191, 160)]
ONEHOT_CROSS = [(1, 2, 200, 77, 40), (1, 2, 160, 80, 160), (1, 2, 129, 65, 16), (2, 2, 64, 16, 8), (1, 2, 100, 1, 8),
                (1, 2, 300, 64, 80), (1, 2, 128, 33, 32)]


@pytest.mark.parametrize("B,H,N,dh", ONEHOT_SPATIAL)
def test_spatial_attention_one_hot_rows(B, H, N, dh):
    """o == v[tau] and dV == dO[tau^-1] bit for bit, lse == bits * scale, dQ = dK = 0: a wrong tile-column mapping, row
    placement or head offset moves a copied row and breaks the equality."""
    dev = _dev()
    q, k, v, d_o, tau, bits = _onehot_inputs(B, N, N, H, dh, seed=N * 5 + dh)
    q, k, v = _fused(q, k, v, dev)
    d_o, tau = d_o.to(dev, torch.float16), tau.to(dev)
    o, lse, got = _spatial(q, k, v, d_o, H, ONEHOT_SCALE)
    assert torch.equal(o.view(torch.int16), _gather_rows(v, tau, dh).view(torch.int16)), "o != v[tau]"
    want_lse = bits * ONEHOT_SCALE
    assert ((lse.double() - want_lse).abs() <= 1e-6 * want_lse).all(), (lse.min().item(), lse.max().item(), want_lse)
    inv = torch.argsort(tau, dim=-1)
    assert torch.equal(got["dv"].view(torch.int16), _gather_rows(d_o, inv, dh).view(torch.int16)), "dv != d_o[tau^-1]"
    bar = 1e-4 * got["dv"].abs().max().item()
    assert got["dq"].abs().max().item() <= bar and got["dk"].abs().max().item() <= bar


@pytest.mark.parametrize("B,H,Nq,Nk,dh", ONEHOT_CROSS)
def test_cross_attention_one_hot_rows(B, H, Nq, Nk, dh):
    dev = _dev()
    q, k, v, d_o, tau, _ = _onehot_inputs(B, Nq, Nk, H, dh, seed=Nq * 3 + Nk + dh)
    q, d_o, tau = q.to(dev, torch.float16), d_o.to(dev, torch.float16), tau.to(dev)
    k, v = _kv(k, v, dev)
    o = ops.cross_attention_forward(q, k, v, H, ONEHOT_SCALE)
    assert torch.equal(o.view(torch.int16), _gather_rows(v, tau, dh).view(torch.int16)), "o != v[tau]"
    dq = ops.cross_attention_backward(q, k, v, d_o, H, ONEHOT_SCALE)
    assert dq.abs().max().item() <= 1e-4 * d_o.abs().max().item()


def _uniform_closed_form(k, v, d_o, H, scale):
    """q = 0: P = 1/Nk everywhere, lse = ln Nk, o = mean_j v_j, dV_j = mean_i dO_i, dK = 0 and
    dQ_i = (scale / Nk) sum_j (dO_i . (v_j - mean v)) k_j, per head, in fp64."""
    B, Nk, C = k.shape
    dh = C // H
    kh, vh, gh = (t.double().reshape(B, -1, H, dh).transpose(1, 2) for t in (k, v, d_o))
    vbar = vh.mean(2, keepdim=True)                                          # [B, H, 1, dh]
    dp = gh @ (vh - vbar).transpose(-1, -2)                                  # [B, H, Nq, Nk]
    dq = (scale / Nk) * dp @ kh
    dv = gh.sum(2, keepdim=True).expand_as(vh) / Nk
    merge = lambda t: t.transpose(1, 2).reshape(B, t.shape[2], C)  # noqa: E731
    return merge(vbar.expand(-1, -1, d_o.shape[1], -1)), merge(dq), merge(dv)


@pytest.mark.parametrize("B,H,N,dh", [(2, 2, 64, 8), (1, 2, 129, 40), (1, 2, 200, 80), (1, 2, 97, 160), (1, 2, 2, 16)])
def test_spatial_attention_uniform_rows(B, H, N, dh):
    """q = 0: lse == ln N; o within one fp16 ulp of the fp64 mean of v (a quarter of the exponentials come from the
    polynomial exp2, whose value at 0 is 0.99999928, not 1); dK == 0 exactly (dK = dS^T Q); dQ, dV in closed form."""
    dev = _dev()
    g = torch.Generator().manual_seed(N + dh)
    C, scale = H * dh, dh ** -0.5
    q = torch.zeros(B, N, C, dtype=torch.float64)
    k = torch.randn(B, N, C, generator=g)
    v = _quantized((B, N, C), g)
    q, k, v = _fused(q, k, v, dev)
    d_o = torch.randn(B, N, C, generator=g).to(dev, torch.float16)
    o, lse, got = _spatial(q, k, v, d_o, H, scale)
    want_o, want_dq, want_dv = _uniform_closed_form(k, v, d_o, H, scale)
    assert ((lse.double() - math.log(N)).abs() <= 1e-6 * max(1.0, math.log(N))).all()
    assert ((o.double() - want_o).abs() <= _ulp16(want_o)).all(), (o.double() - want_o).abs().max().item()
    assert (got["dk"] == 0).all(), "dK = dS^T Q must vanish with Q = 0"
    assert torch.isfinite(got["dq"]).all() and torch.isfinite(got["dv"]).all()
    # dV: every P is the same fp16 value (<= 2^-11 off 1/N) and dV is rounded once
    assert _rel(got["dv"], want_dv) <= 2e-3 and _rel(got["dq"], want_dq) <= 4e-3


@pytest.mark.parametrize("B,H,Nq,Nk,dh", [(1, 2, 200, 77, 40), (1, 2, 100, 80, 160), (2, 2, 64, 17, 8), (1, 2, 64, 1, 16)])
def test_cross_attention_uniform_rows(B, H, Nq, Nk, dh):
    dev = _dev()
    g = torch.Generator().manual_seed(Nq + Nk + dh)
    C, scale = H * dh, dh ** -0.5
    q = torch.zeros(B, Nq, C, device=dev, dtype=torch.float16)
    k, v = _kv(torch.randn(B, Nk, C, generator=g), _quantized((B, Nk, C), g), dev)
    d_o = torch.randn(B, Nq, C, generator=g).to(dev, torch.float16)
    o = ops.cross_attention_forward(q, k, v, H, scale)
    dq = ops.cross_attention_backward(q, k, v, d_o, H, scale)
    want_o, want_dq, _ = _uniform_closed_form(k, v, d_o, H, scale)
    assert ((o.double() - want_o).abs() <= _ulp16(want_o)).all(), (o.double() - want_o).abs().max().item()
    assert torch.isfinite(dq).all() and _rel(dq, want_dq) <= 4e-3


def _constant_v_bars(q, k, v0, d_o, H, scale):
    """Bounds on |dQ|, |dK| when every key carries the value row v0. dS_ij = scale P_ij dO_i . (v0 - O_i) and the kernel's
    O_i = v0 (sum_j fp16(P_ij) / sum_j P_ij), rounded once: |O_i - v0| <= 2^-10 |v0| per element, so
    |dS_ij| <= 2^-10 scale P_ij sum_e |dO_ie v0_e|. Summed against K (rows of P sum to 1) and against Q (over the column
    sums of P), with a factor 4 of margin for the fp32 and fp16 roundings of dP, D and dS."""
    B, Nq, C = q.shape
    dh = C // H
    qh, kh = (t.double().reshape(B, -1, H, dh).transpose(1, 2) for t in (q, k))
    p = torch.softmax(qh @ kh.transpose(-1, -2) * scale, -1)                 # [B, H, Nq, Nk]
    a = (d_o.double().reshape(B, Nq, H, dh).abs() * v0.double().reshape(B, 1, H, dh).abs()).sum(-1)  # [B, Nq, H]
    amax = a.max().item()
    bar_dq = 2.0 ** -8 * scale * amax * k.abs().max().item()
    bar_dk = 2.0 ** -8 * scale * amax * q.abs().max().item() * p.sum(2).max().item()
    return bar_dq, bar_dk


@pytest.mark.parametrize("B,H,N,dh", [(2, 2, 129, 40), (1, 2, 256, 80), (1, 2, 100, 160), (2, 2, 40, 8)])
def test_spatial_attention_constant_values(B, H, N, dh):
    """Every key carries the same value row: o = v0 (up to the fp16 rounding of P), dQ = dK = 0 (dP_ij = D_i)."""
    dev = _dev()
    g = torch.Generator().manual_seed(N * 11 + dh)
    C, scale = H * dh, dh ** -0.5
    q, k = (torch.randn(B, N, C, generator=g) * 2 for _ in range(2))
    v0 = _quantized((B, 1, C), g)
    q, k, v = _fused(q, k, v0.expand(B, N, C), dev)
    d_o = _quantized((B, N, C), g).to(dev, torch.float16)
    o, lse, got = _spatial(q, k, v, d_o, H, scale)
    v0 = v0.to(dev)
    assert ((o.double() - v0).abs() <= 2.0 ** -9 * v0.abs()).all(), (o.double() - v0).abs().max().item()
    bar_dq, bar_dk = _constant_v_bars(q, k, v0, d_o, H, scale)
    print(f"B={B} H={H} N={N} dh={dh}: |dq| {got['dq'].abs().max().item():.3e} (bar {bar_dq:.3e}), "
          f"|dk| {got['dk'].abs().max().item():.3e} (bar {bar_dk:.3e})")
    assert got["dq"].abs().max().item() <= bar_dq and got["dk"].abs().max().item() <= bar_dk
    _, _, (_, _, gv) = _ref(q, k, v, d_o, H, scale)
    assert _rel(got["dv"], gv) < 4e-3


@pytest.mark.parametrize("B,H,Nq,Nk,dh", [(1, 2, 200, 77, 40), (1, 2, 129, 80, 160), (2, 2, 64, 65, 8)])
def test_cross_attention_constant_values(B, H, Nq, Nk, dh):
    dev = _dev()
    g = torch.Generator().manual_seed(Nq * 11 + Nk + dh)
    C, scale = H * dh, dh ** -0.5
    q = (torch.randn(B, Nq, C, generator=g) * 2).to(dev, torch.float16)
    v0 = _quantized((B, 1, C), g)
    k, v = _kv(torch.randn(B, Nk, C, generator=g) * 2, v0.expand(B, Nk, C), dev)
    d_o = _quantized((B, Nq, C), g).to(dev, torch.float16)
    o = ops.cross_attention_forward(q, k, v, H, scale)
    dq = ops.cross_attention_backward(q, k, v, d_o, H, scale)
    v0 = v0.to(dev)
    assert ((o.double() - v0).abs() <= 2.0 ** -9 * v0.abs()).all(), (o.double() - v0).abs().max().item()
    bar_dq, _ = _constant_v_bars(q, k, v0, d_o, H, scale)
    assert dq.abs().max().item() <= bar_dq, (dq.abs().max().item(), bar_dq)


# ---------------------------------------------------------------------------------------------------------------
# 3. token and key counts around the tile edges
# ---------------------------------------------------------------------------------------------------------------
CROSS_KEYS = [1, 2, 8, 15, 16, 17, 63, 64, 65, 76, 77, 78, 79, 80]


@pytest.mark.parametrize("dh", [8, 40, 160])
@pytest.mark.parametrize("Nk", CROSS_KEYS)
def test_cross_attention_key_count(Nk, dh):
    """1..80 text keys: the forward splits more than 64 keys into two 64-key tiles, the dQ kernel takes all of them as one
    80-wide tile; both mask the keys past the end."""
    dev = _dev()
    B, H, Nq = 1, 2, 200
    g = torch.Generator().manual_seed(Nk * 7 + dh)
    C, scale = H * dh, dh ** -0.5
    q = (torch.randn(B, Nq, C, generator=g) * 2).to(dev, torch.float16)
    k, v = _kv(torch.randn(B, Nk, C, generator=g), torch.randn(B, Nk, C, generator=g), dev)
    d_o = torch.randn(B, Nq, C, generator=g).to(dev, torch.float16)
    o = ops.cross_attention_forward(q, k, v, H, scale)
    dq = ops.cross_attention_backward(q, k, v, d_o, H, scale)
    ref_o, _, (gq, _, _) = _ref(q, k, v, d_o, H, scale)
    lib_o, (lq, _, _) = _library(q, k, v, d_o, H, scale)
    tag = f"Nk={Nk} dh={dh}"
    _check_forward(tag, o, ref_o, lib_o)
    _check_grads(tag, {"dq": dq}, {"dq": gq}, {"dq": lq})


def test_cross_attention_rejects_81_keys():
    dev = _dev()
    q = torch.randn(1, 64, 80, device=dev, dtype=torch.float16)
    k = torch.randn(1, 81, 80, device=dev, dtype=torch.float16)
    with pytest.raises(NotImplementedError):
        ops.cross_attention_forward(q, k, k, 2, 40 ** -0.5)
    with pytest.raises(NotImplementedError):
        ops.cross_attention_backward(q, k, k, q, 2, 40 ** -0.5)


SPATIAL_TOKENS = ([(N, dh) for dh in (40, 160) for N in (63, 64, 65, 127, 128, 129, 191, 193)]
                  + [(N, 160) for N in (31, 33, 97)])  # DH = 160: 64-key dK/dV CTAs and 32-query tiles


@pytest.mark.parametrize("N,dh", SPATIAL_TOKENS)
def test_spatial_attention_token_count(N, dh):
    dev = _dev()
    B, H = 2, 2
    g = torch.Generator().manual_seed(N * 19 + dh)
    C, scale = H * dh, dh ** -0.5
    q, k, v = _fused(torch.randn(B, N, C, generator=g) * 2, torch.randn(B, N, C, generator=g),
                     torch.randn(B, N, C, generator=g), dev)
    d_o = torch.randn(B, N, C, generator=g).to(dev, torch.float16)
    o, lse, got = _spatial(q, k, v, d_o, H, scale)
    ref_o, ref_lse, (gq, gk, gv) = _ref(q, k, v, d_o, H, scale)
    lib_o, (lq, lk, lv) = _library(q, k, v, d_o, H, scale)
    tag = f"N={N} dh={dh}"
    _check_forward(tag, o, ref_o, lib_o, lse, ref_lse)
    _check_grads(tag, got, {"dq": gq, "dk": gk, "dv": gv}, {"dq": lq, "dk": lk, "dv": lv})


# ---------------------------------------------------------------------------------------------------------------
# 4. stores stay inside their outputs (C ABI, padded strides, canary-filled guards)
# ---------------------------------------------------------------------------------------------------------------
CANARY16 = 0x7E5B        # an fp16 NaN: no kernel writes it
CANARY32 = 0x7FC5A5A5    # an fp32 NaN


class _Canary:
    """A logical [B, rows, cols] output inside a larger buffer pre-filled with a NaN bit pattern: rows `pad_cols` wider
    than the view, frames `pad_rows` rows longer, and `guard` elements before and after."""

    def __init__(self, B, rows, cols, dev, bits=16, pad_cols=24, pad_rows=3, guard=64):
        dtype, canary = (torch.int16, CANARY16) if bits == 16 else (torch.int32, CANARY32)
        self.sr = cols + pad_cols
        self.sb = (rows + pad_rows) * self.sr
        total = guard + B * self.sb + guard
        self.buf = torch.full((total,), canary, dtype=dtype, device=dev)
        self.canary = canary
        self.inside = torch.zeros(total, dtype=torch.bool, device=dev)
        frames = slice(guard, guard + B * self.sb)
        self.view = self.buf[frames].view(B, rows + pad_rows, self.sr)[:, :rows, :cols]
        self.inside[frames].view(B, rows + pad_rows, self.sr)[:, :rows, :cols] = True
        self.ptr = ctypes.c_void_p(self.buf.data_ptr() + guard * self.buf.element_size())

    def check(self, want, what):
        """every element outside the view still holds the canary; the view holds `want` bit for bit."""
        bits = torch.int16 if self.buf.dtype == torch.int16 else torch.int32
        assert (self.buf[~self.inside] == self.canary).all(), f"{what}: store outside the output"
        assert (self.view != self.canary).all(), f"{what}: element of the output never written"
        assert torch.equal(self.view, want.contiguous().view(bits).reshape(self.view.shape)), f"{what}: wrong bits"


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


@pytest.mark.parametrize("dh", HEAD_DIMS)
def test_spatial_attention_stores_stay_in_bounds(dh):
    """mc_spatial_attn_fwd / mc_spatial_attn_bwd with o, lse, dq, dk, dv inside canary buffers (dq | dk | dv as three
    buffers sharing one stride pattern, so a dQ store past its column block is not overwritten by the dK/dV kernel). The
    bits must equal the ops path's (contiguous outputs): the output strides change where results go, nothing else."""
    dev = _dev()
    B, H, N = 2, 2, 100
    C, scale = H * dh, dh ** -0.5
    g = torch.Generator().manual_seed(dh)
    q, k, v = _fused(torch.randn(B, N, C, generator=g) * 2, torch.randn(B, N, C, generator=g),
                     torch.randn(B, N, C, generator=g), dev)
    d_o = torch.randn(B, N, C, generator=g).to(dev, torch.float16)
    o, lse, got = _spatial(q, k, v, d_o, H, scale)
    L = _lib.lib()

    co, cl = _Canary(B, N, C, dev), _Canary(1, 1, B * H * N, dev, bits=32, pad_cols=0, pad_rows=0)
    st = L.mc_spatial_attn_fwd(_p(q), _p(k), _p(v), co.ptr, cl.ptr, B, N, H, dh, q.stride(0), q.stride(1), k.stride(0),
                               k.stride(1), v.stride(0), v.stride(1), co.sb, co.sr, float(scale), _stream())
    _lib.check(st, "mc_spatial_attn_fwd")
    torch.cuda.synchronize()
    co.check(o, f"dh={dh} o")
    cl.check(lse, f"dh={dh} lse")

    grads = {n: _Canary(B, N, C, dev) for n in ("dq", "dk", "dv")}
    ws = torch.empty(int(L.mc_spatial_attn_bwd_workspace_bytes(B, N, H)), dtype=torch.uint8, device=dev)
    st = L.mc_spatial_attn_bwd(_p(q), _p(k), _p(v), _p(o), _p(d_o), _p(lse), grads["dq"].ptr, grads["dk"].ptr,
                               grads["dv"].ptr, _p(ws), B, N, H, dh, q.stride(0), q.stride(1), k.stride(0), k.stride(1),
                               v.stride(0), v.stride(1), o.stride(0), o.stride(1), d_o.stride(0), d_o.stride(1),
                               grads["dq"].sb, grads["dq"].sr, float(scale), _stream())
    _lib.check(st, "mc_spatial_attn_bwd")
    torch.cuda.synchronize()
    for n, c in grads.items():
        c.check(got[n], f"dh={dh} {n}")


@pytest.mark.parametrize("dh", HEAD_DIMS)
def test_cross_attention_stores_stay_in_bounds(dh):
    """mc_cross_attn_fwd / mc_cross_attn_bwd_dq with o and dq inside canary buffers."""
    dev = _dev()
    B, H, Nq, Nk = 2, 2, 100, 77
    C, scale = H * dh, dh ** -0.5
    g = torch.Generator().manual_seed(dh + 1)
    q = (torch.randn(B, Nq, C, generator=g) * 2).to(dev, torch.float16)
    k, v = _kv(torch.randn(B, Nk, C, generator=g), torch.randn(B, Nk, C, generator=g), dev)
    d_o = torch.randn(B, Nq, C, generator=g).to(dev, torch.float16)
    o = ops.cross_attention_forward(q, k, v, H, scale)
    dq = ops.cross_attention_backward(q, k, v, d_o, H, scale)
    L = _lib.lib()

    co = _Canary(B, Nq, C, dev)
    st = L.mc_cross_attn_fwd(_p(q), _p(k), _p(v), co.ptr, B, Nq, Nk, H, dh, q.stride(0), q.stride(1), k.stride(0),
                             k.stride(1), co.sb, co.sr, float(scale), _stream())
    _lib.check(st, "mc_cross_attn_fwd")
    cq = _Canary(B, Nq, C, dev)
    st = L.mc_cross_attn_bwd_dq(_p(q), _p(k), _p(v), _p(d_o), cq.ptr, B, Nq, Nk, H, dh, q.stride(0), q.stride(1),
                                k.stride(0), k.stride(1), d_o.stride(0), d_o.stride(1), cq.sb, cq.sr, float(scale),
                                _stream())
    _lib.check(st, "mc_cross_attn_bwd_dq")
    torch.cuda.synchronize()
    co.check(o, f"dh={dh} o")
    cq.check(dq, f"dh={dh} dq")
