"""GPU parity of every C-ABI kernel against the oracle (oracle/mc_oracle.py) on seeded inputs.

Bars (stated per test): bit-exact for the elementwise update, the index sets and — on exactly-representable inputs —
the probabilities; fp16-rounding tolerances elsewhere, written next to each assert.
"""
import itertools

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


def _to_oracle(t):  # [B,F,P,C] -> [(B P), F, C]  (reference layout after 'b f d c -> (b d) f c', motion_module.py:279)
    B, F, P, C = t.shape
    return t.permute(0, 2, 1, 3).reshape(B * P, F, C)


def _from_oracle(t, B, P):  # [(B P), F, C] -> [B,F,P,C]
    BP, F, C = t.shape
    return t.reshape(B, P, F, C).permute(0, 2, 1, 3)


def _make_qkv(B, F, P, C, seed, fused, exact=False, dev=None):
    g = torch.Generator(device="cpu").manual_seed(seed)
    shape = (B, F, P, 3 * C) if fused else (3, B, F, P, C)
    if exact:  # every product and partial sum is exactly representable -> no accumulation-order dependence
        x = torch.randint(-2, 3, shape, generator=g).float() * 0.5
    else:
        x = torch.randn(shape, generator=g)
    x = x.to(dev, torch.float16)
    if fused:
        return x[..., :C], x[..., C:2 * C], x[..., 2 * C:]
    return x[0], x[1], x[2]


# ---------------------------------------------------------------------------------------------------------------
# E1: CFG + guided DDIM update, add_noise  — bit-exact
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("with_score", [True, False])
@pytest.mark.parametrize("n_shape", [(1, 4, 16, 64, 64), (1, 4, 8, 17, 3)])
def test_cfg_ddim_step_bit_exact(with_score, n_shape):
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(1)
    ec, eu, x, sc = (torch.randn(n_shape, generator=g).to(dev, torch.float16) for _ in range(4))
    sc = sc * 0.05
    acp = O.alphas_cumprod()
    timesteps = O.uneven_timesteps(50, 25, 0.3)
    for step in (0, 13, 24, 25, 48, 49):  # first, guided, boundary, plain, last (alpha_prev = 1)
        a_t, a_prev = O.ddim_scalars(acp, timesteps, step)
        score = sc if with_score else None
        got = ops.cfg_ddim_step(ec, eu, x, score, 7.5, a_t, a_prev)
        # the reference op sequence executed by ATen on the same device (motionclone_functions.py:239, :339-389)
        want_dev = O.ddim_guided_step(O.cfg_combine(ec, eu, 7.5), x, score, a_t, a_prev)
        assert torch.equal(got, want_dev), f"step {step}: differs from the eager CUDA op sequence"
        # and the oracle's explicit CPU statement of that rounding sequence
        want_cpu = O.cfg_ddim_step_fp16_sequence(ec.cpu(), eu.cpu(), x.cpu(), None if score is None else score.cpu(),
                                                 7.5, a_t, a_prev)
        assert torch.equal(got.cpu(), want_cpu), f"step {step}: differs from the CPU oracle"


def test_add_noise_bit_exact():
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(2)
    x0, nz = (torch.randn(1, 4, 16, 64, 64, generator=g).to(dev, torch.float16) for _ in range(2))
    acp = O.alphas_cumprod()
    got = ops.add_noise(x0, nz, acp[400])
    assert torch.equal(got, O.add_noise(acp, 400, x0, nz))  # eager CUDA op sequence (fp32 opmath for the 0-dim scalars)
    a = acp[400]
    h = lambda t: t.half().float()  # noqa: E731
    want = h(h(a ** 0.5 * x0.cpu().float()) + h((1 - a) ** 0.5 * nz.cpu().float())).half()
    assert torch.equal(got.cpu(), want)


# ---------------------------------------------------------------------------------------------------------------
# T1/T2: temporal attention forward, probabilities, top-1, gathered probabilities
# ---------------------------------------------------------------------------------------------------------------
SHAPES = [  # (L, heads, dh, B, P)
    (16, 8, 40, 1, 64), (16, 8, 80, 2, 16), (16, 8, 160, 1, 16), (16, 8, 8, 1, 16), (16, 8, 16, 1, 4),
    (16, 2, 32, 1, 8), (16, 8, 64, 1, 8), (16, 8, 128, 1, 4),
    (8, 8, 40, 1, 64), (8, 8, 160, 2, 4), (8, 8, 8, 1, 16), (8, 8, 16, 1, 2), (8, 8, 32, 1, 16), (8, 8, 80, 1, 6),
    (8, 8, 40, 1, 1), (8, 8, 16, 2, 3),  # odd position counts: the tail position is paired with itself
    (32, 8, 40, 1, 16), (32, 8, 160, 1, 4), (32, 8, 80, 1, 8), (32, 8, 16, 2, 4),
]


@pytest.mark.parametrize("L,H,DH,B,P", SHAPES)
@pytest.mark.parametrize("fused", [False, True])
def test_temporal_attention_forward(L, H, DH, B, P, fused):
    ops, dev = _ops(), _dev()
    C = H * DH
    q, k, v = _make_qkv(B, L, P, C, seed=L * 1000 + DH + P, fused=fused, dev=dev)
    scale = DH ** -0.5
    o, probs, top, _ = ops.temporal_attention_forward(q, k, v, H, scale, want_probs=True, want_top1=True)
    qo, ko, vo = (_to_oracle(t).contiguous() for t in (q, k, v))
    want_probs = O.temporal_probs(qo, ko, H, scale)  # eager fp16 baddbmm -> softmax on the same device
    want_o = _from_oracle(O.attention_math(qo, ko, vo, H, scale), B, P)
    # probabilities: fp32 accumulation order of QK^T may differ from cuBLAS -> at most a few fp16 ulps on a few entries
    dp = (probs.float() - want_probs.float()).abs()
    assert dp.max().item() <= 2e-3, f"probs max diff {dp.max().item()}"
    assert (dp > 0).float().mean().item() < 0.05, "too many probabilities differ from the eager fp16 path"
    # output: |o| <~ 4, one fp16 ulp at 2-4 is 1.95e-3; fp32-accumulated PV then one rounding
    do = (o.float() - want_o.float()).abs().max().item()
    assert do <= 4e-3, f"o max diff {do}"
    # top-1 on the kernel's own probabilities: bit-exact incl. the tie rule (lowest index)
    wv, wi = O.top1_lowest_index(probs)
    assert torch.equal(top[1], wi) and torch.equal(top[0], wv)
    # and identical to torch.topk wherever the probabilities agree bitwise
    tv, ti = O.top1(want_probs)
    same_row = (probs == want_probs).all(dim=-1, keepdim=True)
    assert torch.equal(top[1][same_row], ti[same_row])
    # truth check against fp64 math on the same fp16 inputs
    p64 = torch.softmax(torch.einsum("bqd,bkd->bqk", O.heads_to_batch(qo, H).double(),
                                     O.heads_to_batch(ko, H).double()) * scale, -1)
    assert (probs.double().reshape(p64.shape) - p64).abs().max().item() <= 2.5e-3


@pytest.mark.parametrize("L,H,DH,B,P", [(16, 8, 40, 1, 32), (8, 8, 80, 1, 8), (32, 8, 160, 1, 4), (16, 8, 160, 1, 8)])
def test_temporal_attention_bit_exact_on_exact_inputs(L, H, DH, B, P):
    """Tie-heavy, exactly-representable q,k: no accumulation-order freedom, so probabilities and index sets must equal
    the eager path bit for bit (north_star: bit-exact top-k index sets; tie rule = lowest index)."""
    ops, dev = _ops(), _dev()
    C = H * DH
    q, k, v = _make_qkv(B, L, P, C, seed=7, fused=False, exact=True, dev=dev)
    scale = DH ** -0.5
    o, probs, top, _ = ops.temporal_attention_forward(q, k, v, H, scale, want_probs=True, want_top1=True)
    qo, ko = (_to_oracle(t).contiguous() for t in (q, k))
    want_probs = O.temporal_probs(qo, ko, H, scale)
    assert torch.equal(probs, want_probs), "probabilities differ bitwise from the eager fp16 path on exact inputs"
    wv, wi = O.top1_lowest_index(want_probs)
    assert torch.equal(top[1], wi) and torch.equal(top[0], wv)
    ties = (want_probs == wv).sum(-1) > 1
    assert ties.float().mean().item() > 0.01, "test inputs should be tie-heavy"
    # torch.topk on the device agrees with the lowest-index rule on these inputs? recorded, not required:
    tv, ti = O.top1(want_probs)
    assert torch.equal(tv, wv)


@pytest.mark.parametrize("L,H,DH,B,P", [(16, 8, 40, 1, 16), (8, 8, 80, 1, 8), (32, 8, 16, 1, 4)])
def test_temporal_attention_gather_and_probs_only(L, H, DH, B, P):
    ops, dev = _ops(), _dev()
    C = H * DH
    q, k, v = _make_qkv(B, L, P, C, seed=11, fused=True, dev=dev)
    scale = DH ** -0.5
    g = torch.Generator().manual_seed(5)
    idx = torch.randint(0, L, (B * P, H, L, 1), generator=g).to(dev, torch.uint8)
    o, probs, _, gathered = ops.temporal_attention_forward(q, k, v, H, scale, want_probs=True, gather_idx=idx)
    assert torch.equal(gathered, torch.gather(probs, -1, idx.long()))
    _, probs2, top, _ = ops.temporal_attention_forward(q, k, None, H, scale, want_o=False, want_probs=True,
                                                       want_top1=True)
    assert torch.equal(probs, probs2)
    v2, i2 = ops.top1_rows(probs)
    assert torch.equal(v2, top[0]) and torch.equal(i2, top[1])


# ---------------------------------------------------------------------------------------------------------------
# T1 backward + T3 loss
# ---------------------------------------------------------------------------------------------------------------
def _ref_grads(q, k, v, H, scale, d_o, d_probs, gather_idx, d_gathered):
    """fp32 autograd of the math path (models/attention.py:461-490 + :564-611) on the same fp16 inputs."""
    B, F, P, C = q.shape
    qf, kf, vf = (_to_oracle(t).float().detach().requires_grad_(True) for t in (q, k, v))
    probs = O.temporal_probs(qf, kf, H, scale)
    out = O.batch_to_heads(torch.bmm(probs.reshape(-1, F, F), O.heads_to_batch(vf, H)), H)
    loss = 0.0
    if d_o is not None:
        loss = loss + (out * _to_oracle(d_o).float()).sum()
    if d_probs is not None:
        loss = loss + (probs * d_probs.float()).sum()
    if d_gathered is not None:
        loss = loss + (torch.gather(probs, -1, gather_idx.long()) * d_gathered.float()).sum()
    gq, gk, gv = torch.autograd.grad(loss, (qf, kf, vf), allow_unused=True)
    f = lambda t: None if t is None else _from_oracle(t, B, P)  # noqa: E731
    return f(gq), f(gk), f(gv)


def _close(a, b, rel=2e-2, name=""):
    scale = b.abs().max().item() + 1e-12
    err = (a.float() - b).abs().max().item()
    assert err <= rel * scale + 1e-6, f"{name}: max err {err} vs scale {scale}"


@pytest.mark.parametrize("L,H,DH,B,P", [(16, 8, 40, 1, 16), (16, 8, 160, 1, 4), (16, 8, 80, 2, 8), (8, 8, 40, 1, 8),
                                        (8, 8, 16, 1, 4), (8, 8, 40, 1, 1), (8, 8, 16, 1, 3), (32, 8, 40, 1, 4), (32, 8, 160, 1, 2), (16, 8, 8, 1, 4)])
@pytest.mark.parametrize("branches", ["o", "o+gather", "gather", "probs", "all"])
@pytest.mark.parametrize("fused", [True, False])
def test_temporal_attention_backward(L, H, DH, B, P, branches, fused):
    ops, dev = _ops(), _dev()
    C = H * DH
    q, k, v = _make_qkv(B, L, P, C, seed=3 + L + DH, fused=True, dev=dev)
    scale = DH ** -0.5
    g = torch.Generator().manual_seed(9)
    d_o = torch.randn(B, L, P, C, generator=g).to(dev, torch.float16) if branches in ("o", "o+gather", "all") else None
    idx = torch.randint(0, L, (B * P, H, L, 1), generator=g).to(dev, torch.uint8)
    d_g = (torch.randn(B * P, H, L, 1, generator=g) * 0.5).to(dev, torch.float16) \
        if branches in ("o+gather", "gather", "all") else None
    d_p = (torch.randn(B * P, H, L, L, generator=g) * 0.5).to(dev, torch.float16) if branches in ("probs", "all") else None
    if not fused:
        q, k, v = (t.contiguous() for t in (q, k, v))
    dq, dk, dv = ops.temporal_attention_backward(q, k, v, H, scale, d_o, d_p, idx if d_g is not None else None, d_g)
    gq, gk, gv = _ref_grads(q, k, v, H, scale, d_o, d_p, idx, d_g)
    # tolerance: 2 % of the gradient's max magnitude — P, dP and dS are rounded to fp16 inside the kernel exactly where
    # the eager fp16 graph rounds them (bmm/softmax backward outputs); the fp32 reference does not round at all
    _close(dq, gq, name="dq")
    _close(dk, gk, name="dk")
    if d_o is not None:
        _close(dv, gv, name="dv")
    elif fused:
        assert dv.abs().max().item() == 0  # column block of the fused gradient buffer, zero-filled
    else:
        assert dv is None


def test_temporal_attention_autograd_function():
    ops, dev = _ops(), _dev()
    L, H, DH, B, P = 16, 8, 40, 1, 16
    C = H * DH
    q, k, v = _make_qkv(B, L, P, C, seed=21, fused=False, dev=dev)
    qkv = torch.cat([q, k, v], dim=-1).requires_grad_(True)  # the fused projection output the module feeds
    idx = torch.randint(0, L, (B * P, H, L, 1)).to(dev, torch.uint8)
    ref_val = torch.rand(B * P, H, L, 1).to(dev, torch.float16)
    o, _, gathered = ops.TemporalAttention.apply(qkv, H, DH ** -0.5, False, idx)
    loss = 2000 * ops.motion_loss([gathered], [ref_val]) + (o.float() ** 2).mean().half()
    (gqkv,) = torch.autograd.grad(loss, (qkv,))
    gq, gk, gv = gqkv[..., :C], gqkv[..., C:2 * C], gqkv[..., 2 * C:]
    # reference: fp32 autograd through the oracle's formulas
    qf, kf, vf = (_to_oracle(t.detach()).float().requires_grad_(True) for t in (q, k, v))
    probs = O.temporal_probs(qf, kf, H, DH ** -0.5)
    out = O.batch_to_heads(torch.bmm(probs.reshape(-1, L, L), O.heads_to_batch(vf, H)), H)
    lref = 2000 * O.motion_loss({"m": probs}, {"m": [ref_val.float(), idx]}) + (_from_oracle(out, B, P) ** 2).mean()
    rq, rk, rv = torch.autograd.grad(lref, (qf, kf, vf))
    assert abs(loss.item() - lref.item()) <= 2e-3 * abs(lref.item()) + 1e-3
    _close(gq, _from_oracle(rq, B, P), rel=3e-2, name="dq")
    _close(gk, _from_oracle(rk, B, P), rel=3e-2, name="dk")
    _close(gv, _from_oracle(rv, B, P), rel=3e-2, name="dv")


def test_motion_loss_matches_eager_rounding():
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(4)
    cur = [torch.rand(256, 8, 16, 1, generator=g).to(dev, torch.float16).requires_grad_(True) for _ in range(6)]
    ref = [torch.rand(256, 8, 16, 1, generator=g).to(dev, torch.float16) for _ in range(6)]
    loss = ops.motion_loss(cur, ref)
    want = torch.stack([torch.nn.functional.mse_loss(c, r) for c, r in zip(cur, ref)]).sum()  # motionclone_functions.py:96-100
    # fp32 partial sums are reduced in a different order than ATen's reduce kernel: allow one fp16 ulp of the total
    assert abs(loss.item() - want.item()) <= 1e-3 * want.item() + 1e-6
    truth = sum(((c.double() - r.double()) ** 2).mean() for c, r in zip(cur, ref)).item()
    assert abs(loss.item() - truth) <= 2e-3 * truth
    grads = torch.autograd.grad(2000 * loss, cur)
    want_g = torch.autograd.grad(2000 * want, cur)
    for a, b in zip(grads, want_g):
        _close(a, b.float(), rel=5e-3, name="dcur")


# ---------------------------------------------------------------------------------------------------------------
# glue kernels of the inference passes: NHWC GroupNorm(+SiLU), LayerNorm, GEGLU
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,C,H,W", [(16, 320, 64, 64), (2, 640, 32, 32), (4, 1280, 8, 8), (3, 2560, 8, 8), (2, 1920, 16, 16),
                                     (2, 960, 32, 32), (8, 64, 4, 4), (2, 256, 2, 2), (16, 320, 1, 1)])
@pytest.mark.parametrize("silu", [False, True])
def test_groupnorm_nhwc(N, C, H, W, silu):
    """reference: InflatedGroupNorm (+ SiLU) models/resnet.py:21-29, :186-187; eps 1e-5 / 1e-6, 32 groups."""
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(C + H)
    x = (torch.randn(N, C, H, W, generator=g) * 3 + 1.5).to(dev, torch.float16).contiguous(memory_format=torch.channels_last)
    w = (1 + 0.1 * torch.randn(C, generator=g)).to(dev, torch.float16)
    b = (0.1 * torch.randn(C, generator=g)).to(dev, torch.float16)
    with torch.no_grad():
        y = ops.groupnorm_nhwc(x, w, b, 32, 1e-5, silu)
    assert y.is_contiguous(memory_format=torch.channels_last)
    ref = torch.nn.functional.group_norm(x.float(), 32, w.float(), b.float(), 1e-5)
    eager = torch.nn.functional.group_norm(x.contiguous(), 32, w, b, 1e-5)
    if silu:
        ref, eager = torch.nn.functional.silu(ref), torch.nn.functional.silu(eager)
    err = (y.float() - ref).abs().max().item()
    err_eager = (eager.float() - ref).abs().max().item()
    # one fp16 rounding of an O(5) value (+ one more before the fused SiLU, as the eager pair of kernels does)
    assert err <= max(6e-3, 1.5 * err_eager), (err, err_eager)


@pytest.mark.parametrize("rows,C", [(4096, 320), (1024, 640), (257, 1280), (64, 64), (16, 256), (8, 2048)])
def test_layernorm(rows, C):
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(C)
    x = (torch.randn(2, rows, C, generator=g) * 2 + 0.5).to(dev, torch.float16)
    w = (1 + 0.1 * torch.randn(C, generator=g)).to(dev, torch.float16)
    b = (0.1 * torch.randn(C, generator=g)).to(dev, torch.float16)
    with torch.no_grad():
        y = ops.layernorm(x, w, b, 1e-5)
    ref = torch.nn.functional.layer_norm(x.float(), (C,), w.float(), b.float(), 1e-5)
    eager = torch.nn.functional.layer_norm(x, (C,), w, b, 1e-5)
    err, err_eager = (y.float() - ref).abs().max().item(), (eager.float() - ref).abs().max().item()
    assert err <= max(4e-3, 1.5 * err_eager), (err, err_eager)


@pytest.mark.parametrize("T,I", [(4096, 1280), (1000, 2560), (64, 5120), (16, 256)])
def test_geglu(T, I):
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(I)
    x = (torch.randn(T, 2 * I, generator=g) * 2).to(dev, torch.float16)
    with torch.no_grad():
        y = ops.geglu(x)
    h, gate = x.chunk(2, dim=-1)
    eager = h * torch.nn.functional.gelu(gate)  # the eager graph of diffusers' GEGLU
    ref = h.float() * torch.nn.functional.gelu(gate.float())
    assert (y.float() - ref).abs().max().item() <= max(1.6e-2, 1.5 * (eager.float() - ref).abs().max().item())
    assert (y != eager).float().mean().item() < 1e-3  # same rounding points as the eager kernels: almost always bit-equal


def test_groupnorm_with_time_embedding_bias_and_layernorm_with_positional_add():
    """`hidden_states + temb` folded into norm2 (models/resnet.py:194-197) and `x + pe` folded into the LayerNorm that
    precedes VersatileAttention (models/motion_module.py:215, :281-282): same rounding points as the eager ops."""
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(3)
    b, f, C, H, W = 2, 16, 320, 16, 16
    x = torch.randn(b * f, C, H, W, generator=g).to(dev, torch.float16).contiguous(memory_format=torch.channels_last)
    temb = torch.randn(b, C, generator=g).to(dev, torch.float16)
    w = (1 + 0.1 * torch.randn(C, generator=g)).to(dev, torch.float16)
    bb = (0.1 * torch.randn(C, generator=g)).to(dev, torch.float16)
    with torch.no_grad():
        y = ops.groupnorm_nhwc(x, w, bb, 32, 1e-5, True, chan_bias=temb)
    xe = x + temb.repeat_interleave(f, dim=0)[:, :, None, None]
    eager = torch.nn.functional.silu(torch.nn.functional.group_norm(xe.contiguous(), 32, w, bb, 1e-5))
    ref = torch.nn.functional.silu(torch.nn.functional.group_norm(xe.float(), 32, w.float(), bb.float(), 1e-5))
    assert (y.float() - ref).abs().max().item() <= max(6e-3, 1.5 * (eager.float() - ref).abs().max().item())

    d = 64
    t = torch.randn(b * f, d, C, generator=g).to(dev, torch.float16)
    pe = torch.randn(f, C, generator=g).to(dev, torch.float16)
    with torch.no_grad():
        z = ops.layernorm(t, w, bb, 1e-5, post_add=pe, rows_per_frame=d)
    eager = (torch.nn.functional.layer_norm(t, (C,), w, bb, 1e-5).view(b, f, d, C) + pe.view(1, f, 1, C)).view(b * f, d, C)
    ref = (torch.nn.functional.layer_norm(t.float(), (C,), w.float(), bb.float(), 1e-5).view(b, f, d, C)
           + pe.float().view(1, f, 1, C)).view(b * f, d, C)
    assert (z.float() - ref).abs().max().item() <= max(6e-3, 1.5 * (eager.float() - ref).abs().max().item())
    assert (z != eager).float().mean().item() < 2e-2


@pytest.mark.parametrize("N,C,H,W,f", [(16, 320, 32, 32, 16), (4, 1280, 8, 8, 2), (2, 2560, 8, 8, 2), (8, 64, 4, 4, 8)])
@pytest.mark.parametrize("silu,with_bias", [(True, True), (True, False), (False, False)])
def test_groupnorm_nhwc_backward(N, C, H, W, f, silu, with_bias):
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(C + H)
    x = (torch.randn(N, C, H, W, generator=g) * 2 + 0.7).to(dev, torch.float16).contiguous(memory_format=torch.channels_last)
    w = (1 + 0.1 * torch.randn(C, generator=g)).to(dev, torch.float16)
    b = (0.1 * torch.randn(C, generator=g)).to(dev, torch.float16)
    cb = torch.randn(N // f, C, generator=g).to(dev, torch.float16) if with_bias else None
    dz = torch.randn(N, C, H, W, generator=g).to(dev, torch.float16).contiguous(memory_format=torch.channels_last)
    xg = x.clone().requires_grad_(True)
    y = ops.GroupNormNHWCFn.apply(xg, w, b, cb, 32, 1e-5, silu)
    (dx,) = torch.autograd.grad(y, xg, dz)
    assert dx.is_contiguous(memory_format=torch.channels_last)
    xr = x.float().clone().requires_grad_(True)
    xin = xr if cb is None else xr + cb.float().repeat_interleave(f, dim=0)[:, :, None, None]
    yr = torch.nn.functional.group_norm(xin, 32, w.float(), b.float(), 1e-5)
    if silu:
        yr = torch.nn.functional.silu(yr)
    (dr,) = torch.autograd.grad(yr, xr, dz.float())
    assert (y.float() - yr).abs().max().item() <= 8e-3
    _close(dx, dr, rel=1e-2, name="groupnorm dx")


@pytest.mark.parametrize("rows,C", [(2048, 320), (300, 640), (64, 1280), (16, 64)])
def test_layernorm_and_geglu_backward(rows, C):
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(C)
    x = (torch.randn(2, rows, C, generator=g) * 2 + 0.3).to(dev, torch.float16)
    w = (1 + 0.1 * torch.randn(C, generator=g)).to(dev, torch.float16)
    b = (0.1 * torch.randn(C, generator=g)).to(dev, torch.float16)
    dy = torch.randn(2, rows, C, generator=g).to(dev, torch.float16)
    xg = x.clone().requires_grad_(True)
    (dx,) = torch.autograd.grad(ops.LayerNormFn.apply(xg, w, b, 1e-5, None, 0), xg, dy)
    xr = x.float().clone().requires_grad_(True)
    (dr,) = torch.autograd.grad(torch.nn.functional.layer_norm(xr, (C,), w.float(), b.float(), 1e-5), xr, dy.float())
    _close(dx, dr, rel=1e-2, name="layernorm dx")

    I = C * 2
    u = (torch.randn(rows, 2 * I, generator=g) * 1.5).to(dev, torch.float16)
    du = torch.randn(rows, I, generator=g).to(dev, torch.float16)
    ug = u.clone().requires_grad_(True)
    (dg,) = torch.autograd.grad(ops.GEGLUFn.apply(ug), ug, du)
    ur = u.float().clone().requires_grad_(True)
    h, gate = ur.chunk(2, dim=-1)
    (dgr,) = torch.autograd.grad(h * torch.nn.functional.gelu(gate), ur, du.float())
    _close(dg, dgr, rel=1e-2, name="geglu din")


def test_bias_residual_add():
    """`input_tensor + (conv2(...) + bias)` of the resnet (models/resnet.py:204-211) in one pass, eager rounding points."""
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(0)
    a, b = (torch.randn(4, 320, 16, 16, generator=g).to(dev, torch.float16).contiguous(memory_format=torch.channels_last)
            for _ in range(2))
    bias = torch.randn(320, generator=g).to(dev, torch.float16)
    out = ops.bias_residual_add(a, b, bias)
    assert torch.equal(out, (a + bias[None, :, None, None]) + b)
    ag = a.clone().requires_grad_(True)
    bg = b.clone().requires_grad_(True)
    ga, gb = torch.autograd.grad(ops.BiasResidualAddFn.apply(ag, bg, bias).float().sum(), (ag, bg))
    assert torch.equal(ga, torch.ones_like(a)) and torch.equal(gb, torch.ones_like(b))


# ---------------------------------------------------------------------------------------------------------------
# S2: text cross-attention on the wgmma attention kernels
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,Nq,Nk,H,DH", [(1, 256, 77, 8, 40), (2, 1024, 77, 8, 80), (1, 384, 77, 8, 160), (1, 128, 77, 2, 16),
                                          (1, 200, 77, 8, 32), (1, 4096, 77, 8, 40), (1, 128, 64, 8, 64)])
def test_cross_attention_tcgen05(B, Nq, Nk, H, DH):
    """reference: CrossAttention attn2 through xformers.ops.memory_efficient_attention (models/attention.py:535-542):
    softmax(q k^T * dh^-0.5) v, fp32 softmax statistics, one rounding of the output."""
    ops, dev = _ops(), _dev()
    C = H * DH
    g = torch.Generator().manual_seed(Nq + DH)
    q = torch.randn(B, Nq, C, generator=g).to(dev, torch.float16)
    kv = torch.randn(B, Nk, 2 * C, generator=g).to(dev, torch.float16)
    k, v = kv[..., :C], kv[..., C:]  # strided rows (a fused K|V projection)
    scale = DH ** -0.5
    o = ops.cross_attention_forward(q, k, v, H, scale)
    qh, kh, vh = (t.float().reshape(B, -1, H, DH).transpose(1, 2) for t in (q, k, v))
    ref = (torch.softmax(qh @ kh.transpose(-1, -2) * scale, -1) @ vh).transpose(1, 2).reshape(B, Nq, C)
    lib = torch.nn.functional.scaled_dot_product_attention(
        *(t.reshape(B, -1, H, DH).transpose(1, 2) for t in (q, k.contiguous(), v.contiguous())), scale=scale
    ).transpose(1, 2).reshape(B, Nq, C)
    err, err_lib = (o.float() - ref).abs().max().item(), (lib.float() - ref).abs().max().item()
    # P is rounded to fp16 before PV (as flash kernels do) and O once: a few fp16 ulps of O(1) values
    assert err <= max(3e-3, 2.0 * err_lib), (err, err_lib)


@pytest.mark.parametrize("B,Nq,Nk,H,DH", [(1, 256, 77, 8, 40), (2, 1024, 77, 8, 80), (1, 384, 77, 8, 160), (1, 200, 77, 8, 32),
                                          (1, 4096, 77, 8, 40), (1, 128, 64, 8, 64), (1, 100, 77, 2, 16)])
def test_cross_attention_tcgen05_backward_dq(B, Nq, Nk, H, DH):
    """dQ of attn2 (the guided pass differentiates w.r.t. the latents only, utils/motionclone_functions.py:236; the text
    K / V are constants): against fp32 autograd of the math statement, next to the library flash backward's own error."""
    ops, dev = _ops(), _dev()
    C = H * DH
    g = torch.Generator().manual_seed(7 * Nq + DH)
    q = torch.randn(B, Nq, C, generator=g).to(dev, torch.float16)
    kv = torch.randn(B, Nk, 2 * C, generator=g).to(dev, torch.float16)
    k, v = kv[..., :C], kv[..., C:]
    d_o = torch.randn(B, Nq, C, generator=g).to(dev, torch.float16)
    scale = DH ** -0.5

    qf = q.float().requires_grad_(True)
    qh, kh, vh = (t.reshape(B, -1, H, DH).transpose(1, 2) for t in (qf, k.float(), v.float()))
    ref_o = (torch.softmax(qh @ kh.transpose(-1, -2) * scale, -1) @ vh).transpose(1, 2).reshape(B, Nq, C)
    (ref,) = torch.autograd.grad(ref_o, qf, d_o.float())

    qg = q.clone().requires_grad_(True)
    o = ops.CrossAttentionTC.apply(qg, k, v, H, scale)
    (dq,) = torch.autograd.grad(o, qg, d_o)

    ql = q.clone().requires_grad_(True)
    lib_o = torch.nn.functional.scaled_dot_product_attention(
        *(t.reshape(B, -1, H, DH).transpose(1, 2) for t in (ql, k.contiguous(), v.contiguous())), scale=scale)
    (lib,) = torch.autograd.grad(lib_o, ql, d_o.reshape(B, Nq, H, DH).transpose(1, 2))
    err, err_lib = (dq.float() - ref).abs().max().item(), (lib.float() - ref).abs().max().item()
    assert torch.isfinite(dq).all()
    assert err <= max(5e-3 * ref.abs().max().item(), 2.0 * err_lib), (err, err_lib, ref.abs().max().item())


def test_cross_attention_tcgen05_rejects_kv_grad():
    ops, dev = _ops(), _dev()
    q = torch.randn(1, 128, 64, device=dev, dtype=torch.float16, requires_grad=True)
    k = torch.randn(1, 77, 64, device=dev, dtype=torch.float16, requires_grad=True)
    v = torch.randn(1, 77, 64, device=dev, dtype=torch.float16)
    o = ops.CrossAttentionTC.apply(q, k, v, 2, 32 ** -0.5)
    with pytest.raises(NotImplementedError):
        o.float().sum().backward()


# ---------------------------------------------------------------------------------------------------------------
# residual adds folded into GEMM epilogues (spatial.fold_residual_biases): LayerNorm(x + pre_bias), block equivalence
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,C", [(4096, 320), (1000, 640), (77, 1280), (64, 64)])
def test_layernorm_pre_bias(rows, C):
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(rows + C)
    x = torch.randn(rows, C, generator=g).to(dev, torch.float16)
    pb = (0.1 * torch.randn(C, generator=g)).to(dev, torch.float16)
    w = (1 + 0.1 * torch.randn(C, generator=g)).to(dev, torch.float16)
    b = (0.05 * torch.randn(C, generator=g)).to(dev, torch.float16)
    y = ops.layernorm(x, w, b, 1e-5, pre_bias=pb)
    want = ops.layernorm(x + pb, w, b, 1e-5)  # the kernel adds in fp16, exactly like the separate elementwise add
    assert torch.equal(y, want)
    xg = x.clone().requires_grad_(True)
    dy = torch.randn(rows, C, generator=g).to(dev, torch.float16)
    (dx,) = torch.autograd.grad(ops.LayerNormFn.apply(xg, w, b, 1e-5, None, 0, pb), xg, dy)
    xs = (x + pb).clone().requires_grad_(True)
    (dx_ref,) = torch.autograd.grad(ops.LayerNormFn.apply(xs, w, b, 1e-5, None, 0), xs, dy)
    assert torch.equal(dx, dx_ref)


@pytest.mark.parametrize("kind", ["spatial", "temporal"])
def test_folded_residual_biases_match_unfolded_block(kind):
    """The transformer blocks with their residual adds folded into GEMM epilogues against the same modules run the plain way
    (separate bias + residual add after every projection): same algebra, fp16 rounding points differ slightly."""
    import torch.nn.functional as F
    from motionclone_b200.spatial import Transformer3DModel
    from motionclone_b200.temporal import TemporalTransformer3DModel
    from motionclone_b200.synthetic import load_synthetic_weights
    dev = _dev()
    if kind == "spatial":
        m = Transformer3DModel(8, 40, in_channels=320, num_layers=1, cross_attention_dim=768).to(dev, torch.float16)
    else:
        m = TemporalTransformer3DModel(320, 8, 40, num_layers=1, temporal_position_encoding=True,
                                       temporal_position_encoding_max_len=32).to(dev, torch.float16)
    load_synthetic_weights(m, 7)
    for p in m.parameters():
        p.requires_grad_(False)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(8, 320, 16, 16, generator=g).to(dev, torch.float16).contiguous(memory_format=torch.channels_last)
    text = torch.randn(1, 77, 768, generator=g).to(dev, torch.float16)
    with torch.no_grad():
        # the module's own forward takes the folded path (one block, proj_in has a bias)
        y = m(x, encoder_hidden_states=text, return_dict=False)[0] if kind == "spatial" else m(x, video_length=8)
        # the plain statement of the same module (attention.py:95-142 / motion_module.py:138-161), block run unfolded
        n, c, h, w = x.shape
        residual = x.permute(0, 2, 3, 1).reshape(n, h * w, c)
        t = m.norm(x).permute(0, 2, 3, 1).reshape(n, h * w, c)
        w_in = m.proj_in.weight
        t = F.linear(t, w_in.reshape(w_in.shape[0], -1), m.proj_in.bias)
        blk = m.transformer_blocks[0]
        t = blk(t, encoder_hidden_states=text) if kind == "spatial" else blk(t, video_length=8)
        w_out = m.proj_out.weight
        t = F.linear(t, w_out.reshape(w_out.shape[0], -1), m.proj_out.bias) + residual
        y_ref = t.reshape(n, h, w, c).permute(0, 3, 1, 2)
    err = (y.float() - y_ref.float()).abs().max().item()
    mag = y_ref.float().abs().max().item()
    print(kind, "folded vs unfolded block: max abs diff", err, "of max", mag)
    assert err <= 4e-3 * max(1.0, mag)
