"""Clip lengths off the 8 / 16 / 32-frame tiles (any L in 1..32, t2v_video_sample.py --L): the ragged temporal-attention
instantiations (csrc/temporal_attn.cu, RAGGED = true) and the stand-alone top-1 kernel, then the whole pipeline on the
reference fixtures ref_tiny12 (12 frames in a 16-frame tile), ref_tiny5 (odd length in an 8-frame tile) and ref_c2mini24
(SD1.5 widths, 24 frames in a 32-frame tile).

Kernel bars are those of test_kernels_gpu.py: probabilities <= 2e-3 from the eager fp16 path with < 5 % of entries
differing, O <= 4e-3, fp64 <= 2.5e-3, top-1 bit-exact against the lowest-index argmax of the kernel's own probabilities,
bitwise-equal probabilities on exactly-representable inputs, gradients within 2 % of max against fp32 autograd. On top:
rows with an exact answer (L = 1, one-hot score rows) and canary-filled output buffers that show no padded frame is ever
stored. The end-to-end tests are those of test_pipeline_gpu.py, collected here a second time with this module's `run`
fixture, so the three new fixtures are held to exactly the same bars.
"""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import mc_oracle as O  # noqa: E402
from motionclone_b200 import _lib, ops  # noqa: E402
from test_kernels_gpu import _close, _from_oracle, _make_qkv, _ref_grads, _to_oracle  # noqa: E402
from test_pipeline_gpu import _build, _load  # noqa: E402
# the end-to-end tests of test_pipeline_gpu.py; collected in this module they take the `run` fixture defined below
from test_pipeline_gpu import (test_guidance_loss_and_gradient_vs_reference, test_latents_vs_reference,  # noqa: E402,F401
                               test_latents_vs_same_device_oracle, test_motion_representation_vs_reference,
                               test_unet_forward_vs_reference)

LENGTHS = (1, 2, 3, 5, 7, 9, 12, 15, 17, 20, 24, 31)


def _dev():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    return torch.device("cuda:0")


def _positions(L):
    return 5 if L <= 8 else 4  # L <= 8 packs two positions per 16-row item: an odd count pairs the last with itself


# ---------------------------------------------------------------------------------------------------------------
# forward: probabilities, O, top-1, gathered probabilities
# ---------------------------------------------------------------------------------------------------------------
FWD_SHAPES = ([(L, 8, dh, 1, _positions(L)) for L in LENGTHS for dh in (40, 80, 160)]
              + [(5, 8, 8, 1, 7), (12, 8, 16, 2, 4), (24, 8, 32, 1, 4), (3, 2, 32, 1, 9), (20, 8, 8, 1, 4),
                 (9, 8, 16, 1, 3), (31, 8, 64, 1, 2), (15, 8, 128, 1, 2)]
              + [(5, 8, 40, 1, 63), (12, 8, 40, 1, 64), (24, 8, 40, 1, 64), (17, 8, 80, 2, 8), (7, 8, 80, 2, 3)])


@pytest.mark.parametrize("L,H,DH,B,P", FWD_SHAPES)
@pytest.mark.parametrize("fused", [False, True])
def test_ragged_forward(L, H, DH, B, P, fused):
    dev = _dev()
    C = H * DH
    q, k, v = _make_qkv(B, L, P, C, seed=L * 1000 + DH + P, fused=fused, dev=dev)
    scale = DH ** -0.5
    o, probs, top, _ = ops.temporal_attention_forward(q, k, v, H, scale, want_probs=True, want_top1=True)
    qo, ko, vo = (_to_oracle(t).contiguous() for t in (q, k, v))
    want_probs = O.temporal_probs(qo, ko, H, scale)
    want_o = _from_oracle(O.attention_math(qo, ko, vo, H, scale), B, P)
    assert probs.shape == (B * P, H, L, L)
    dp = (probs.float() - want_probs.float()).abs()
    assert dp.max().item() <= 2e-3, f"probs max diff {dp.max().item()}"
    assert (dp > 0).float().mean().item() < 0.05, "too many probabilities differ from the eager fp16 path"
    do = (o.float() - want_o.float()).abs().max().item()
    assert do <= 4e-3, f"o max diff {do}"
    wv, wi = O.top1_lowest_index(probs)
    assert torch.equal(top[1], wi) and torch.equal(top[0], wv)
    p64 = torch.softmax(torch.einsum("bqd,bkd->bqk", O.heads_to_batch(qo, H).double(),
                                     O.heads_to_batch(ko, H).double()) * scale, -1)
    assert (probs.double().reshape(p64.shape) - p64).abs().max().item() <= 2.5e-3


@pytest.mark.parametrize("L,H,DH,B,P", [(3, 8, 40, 1, 16), (5, 8, 40, 1, 9), (7, 8, 160, 1, 5), (9, 8, 160, 1, 4),
                                        (12, 8, 80, 1, 8), (15, 8, 40, 1, 8), (17, 8, 40, 1, 8), (20, 8, 80, 1, 4),
                                        (24, 8, 160, 1, 4), (31, 8, 80, 1, 4)])
def test_ragged_bit_exact_on_exact_inputs(L, H, DH, B, P):
    """Exactly-representable, tie-heavy q, k: the kernel's summation tree over the padded tile must give ATen's warp
    softmax bit for bit (the padded key columns add exact zeros), and the lowest-index top-1 must follow."""
    dev = _dev()
    q, k, v = _make_qkv(B, L, P, H * DH, seed=7, fused=False, exact=True, dev=dev)
    scale = DH ** -0.5
    _, probs, top, _ = ops.temporal_attention_forward(q, k, v, H, scale, want_probs=True, want_top1=True)
    qo, ko = (_to_oracle(t).contiguous() for t in (q, k))
    want_probs = O.temporal_probs(qo, ko, H, scale)
    assert torch.equal(probs, want_probs), "probabilities differ bitwise from the eager fp16 path on exact inputs"
    wv, wi = O.top1_lowest_index(want_probs)
    assert torch.equal(top[1], wi) and torch.equal(top[0], wv)
    assert ((want_probs == wv).sum(-1) > 1).float().mean().item() > 0.01, "test inputs should be tie-heavy"


@pytest.mark.parametrize("L", LENGTHS)
def test_ragged_gather_probs_only_and_top1_rows(L):
    dev = _dev()
    H, DH, B, P = 8, 40, 1, _positions(L) + 2
    q, k, v = _make_qkv(B, L, P, H * DH, seed=11 + L, fused=True, dev=dev)
    scale = DH ** -0.5
    g = torch.Generator().manual_seed(5)
    idx = torch.randint(0, L, (B * P, H, L, 1), generator=g).to(dev, torch.uint8)
    o, probs, top, gathered = ops.temporal_attention_forward(q, k, v, H, scale, want_probs=True, want_top1=True,
                                                             gather_idx=idx)
    assert torch.equal(gathered, torch.gather(probs, -1, idx.long()))
    o2, probs2, _, _ = ops.temporal_attention_forward(q, k, None, H, scale, want_o=False, want_probs=True)
    assert o2 is None and torch.equal(probs, probs2)
    v2, i2 = ops.top1_rows(probs)
    assert torch.equal(v2, top[0]) and torch.equal(i2, top[1])
    # the stand-alone top-1 on rows that start at every alignment, ties included: lowest index wins
    rows = torch.randint(0, 3, (37, L), generator=g).to(dev, torch.float16)
    v3, i3 = ops.top1_rows(rows)
    wv, wi = O.top1_lowest_index(rows)
    assert torch.equal(v3, wv) and torch.equal(i3, wi)


# ---------------------------------------------------------------------------------------------------------------
# backward
# ---------------------------------------------------------------------------------------------------------------
BWD_SHAPES = ([(L, 8, (40, 80, 160)[i % 3], 1, 3 if L <= 8 else 4) for i, L in enumerate(LENGTHS)]
              + [(12, 8, 16, 1, 4), (5, 8, 8, 1, 5), (24, 8, 32, 1, 2), (20, 8, 40, 2, 8)])


@pytest.mark.parametrize("L,H,DH,B,P", BWD_SHAPES)
@pytest.mark.parametrize("branches", ["o", "o+gather", "gather", "probs", "all"])
@pytest.mark.parametrize("fused", [True, False])
def test_ragged_backward(L, H, DH, B, P, branches, fused):
    dev = _dev()
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
    for name, got in (("dq", dq), ("dk", dk)) + ((("dv", dv),) if d_o is not None else ()):
        assert torch.isfinite(got).all(), name
    _close(dq, gq, name="dq")
    _close(dk, gk, name="dk")
    if d_o is not None:
        _close(dv, gv, name="dv")
    elif fused:
        assert dv.abs().max().item() == 0
    else:
        assert dv is None


# ---------------------------------------------------------------------------------------------------------------
# rows with an exact answer
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("DH", [8, 40, 80, 160])
@pytest.mark.parametrize("fused", [False, True])
def test_single_frame_is_exact(DH, fused):
    """L = 1: the softmax of one score is 1, so o = v, dV = dO, and dQ = dK = 0 exactly."""
    dev = _dev()
    H, B, P = 8, 2, 5
    C = H * DH
    q, k, v = _make_qkv(B, 1, P, C, seed=DH, fused=fused, dev=dev)
    scale = DH ** -0.5
    o, probs, top, _ = ops.temporal_attention_forward(q, k, v, H, scale, want_probs=True, want_top1=True)
    assert torch.equal(o, v.contiguous())
    assert (probs == 1).all() and (top[0] == 1).all() and (top[1] == 0).all()
    g = torch.Generator().manual_seed(1)
    d_o = torch.randn(B, 1, P, C, generator=g).to(dev, torch.float16)
    d_p = torch.randn(B * P, H, 1, 1, generator=g).to(dev, torch.float16)
    idx = torch.zeros(B * P, H, 1, 1, dtype=torch.uint8, device=dev)
    d_g = torch.randn(B * P, H, 1, 1, generator=g).to(dev, torch.float16)
    dq, dk, dv = ops.temporal_attention_backward(q, k, v, H, scale, d_o, d_p, idx, d_g)
    assert (dq == 0).all() and (dk == 0).all()
    assert torch.equal(dv, d_o)


@pytest.mark.parametrize("L", LENGTHS)
def test_one_hot_rows_copy_values(L):
    """Score rows with one key 40 nats above the rest: every other probability rounds to fp16 zero and the dominant one to
    exactly 1, so o = v[tau] bit for bit. tau runs over every key column of the tile (it depends on frame and position)."""
    dev = _dev()
    H, DH, B, P = 8, 40, 1, _positions(L)
    C = H * DH
    tau = torch.tensor([[(L - 1 - i + p) % L for p in range(P)] for i in range(L)])  # [L, P]
    q = torch.zeros(B, L, P, C)
    k = torch.zeros(B, L, P, C)
    for h in range(H):
        for i in range(L):
            k[:, i, :, h * DH + i] = 16.0
            for p in range(P):
                q[:, i, p, h * DH + int(tau[i, p])] = 16.0
    g = torch.Generator().manual_seed(L)
    v = torch.randn(B, L, P, C, generator=g)
    q, k, v = (t.to(dev, torch.float16) for t in (q, k, v))
    o, probs, top, _ = ops.temporal_attention_forward(q, k, v, H, DH ** -0.5, want_probs=True, want_top1=True)
    want_o = v[:, tau, torch.arange(P)[None, :].expand(L, P)]  # [B, L, P, C]: frame i of position p copies v[tau[i, p], p]
    assert torch.equal(o, want_o)
    want_idx = tau.t().reshape(P, 1, L, 1).expand(P, H, L, 1).to(dev, torch.uint8)
    assert torch.equal(top[1], want_idx) and (top[0] == 1).all()
    assert torch.equal(probs, torch.nn.functional.one_hot(want_idx.squeeze(-1).long(), L).to(torch.float16))


# ---------------------------------------------------------------------------------------------------------------
# bounds: outputs inside canary-filled buffers (C ABI)
# ---------------------------------------------------------------------------------------------------------------
CANARY = {torch.float16: 0x7E5B, torch.uint8: 0xA5}  # an fp16 NaN; an index no clip length reaches
BITS = {torch.float16: torch.int16, torch.uint8: torch.uint8}


class _Canary:
    """An output of shape `padded[view]` inside a buffer pre-filled with a canary bit pattern, with `guard` elements
    before and after: `t` is the typed (possibly strided) view handed to the kernel."""

    def __init__(self, padded, view, dtype, dev, guard=64):
        n = 1
        for s in padded:
            n *= s
        self.canary = CANARY[dtype]
        self.buf = torch.full((guard + n + guard,), self.canary, dtype=BITS[dtype], device=dev)
        self.inside = torch.zeros(self.buf.shape, dtype=torch.bool, device=dev)
        self.raw = self.buf[guard:guard + n].view(padded)[view]
        self.inside[guard:guard + n].view(padded)[view] = True
        self.t = self.raw.view(dtype)

    def check(self, want, what):
        assert (self.buf[~self.inside] == self.canary).all(), f"{what}: store outside the output"
        want = want.contiguous().view(self.raw.dtype).reshape(self.raw.shape)
        assert torch.equal(self.raw, want), f"{what}: wrong bits"


def _p(t):
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def _lay(t):
    return _lib.TemporalLayout(t.stride(0), t.stride(1), t.stride(2))


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _flat(n, dtype, dev):
    return _Canary((n,), (slice(0, n),), dtype, dev)


@pytest.mark.parametrize("L", [1, 3, 5, 12, 17, 24, 31])
@pytest.mark.parametrize("DH", [8, 40, 160])
@pytest.mark.parametrize("fused", [False, True])
def test_ragged_stores_stay_in_bounds(L, DH, fused):
    """mc_temporal_attn_fwd / _bwd with every output inside a canary buffer: O and the separate dQ / dK / dV as strided
    [B, F, P, C] views with a gap after every channel row, position and batch; the fused dQ | dK | dV as the column blocks
    of one [B, F, P, 3C] view with a gap frame per batch; probs, top-1, gathered with guards on both sides. The bits
    must equal the ops path's (contiguous outputs)."""
    dev = _dev()
    H, B = 8, 2
    P = 5 if L <= 8 else 4
    C = H * DH
    scale = DH ** -0.5
    q, k, v = _make_qkv(B, L, P, C, seed=L + DH, fused=fused, dev=dev)
    g = torch.Generator().manual_seed(L)
    rows = B * P * H * L
    idx = torch.randint(0, L, (B * P, H, L, 1), generator=g).to(dev, torch.uint8)
    d_o = torch.randn(B, L, P, C, generator=g).to(dev, torch.float16)
    d_p = (torch.randn(B * P, H, L, L, generator=g) * 0.5).to(dev, torch.float16)
    d_g = (torch.randn(B * P, H, L, 1, generator=g) * 0.5).to(dev, torch.float16)
    o, probs, top, gathered = ops.temporal_attention_forward(q, k, v, H, scale, want_probs=True, want_top1=True,
                                                             gather_idx=idx)
    want_grads = ops.temporal_attention_backward(q, k, v, H, scale, d_o, d_p, idx, d_g)
    lib = _lib.lib()

    co = _Canary((B, L + 1, P + 1, C + 8), (slice(None), slice(0, L), slice(0, P), slice(0, C)), torch.float16, dev)
    cp, ctv, cg = (_flat(n, torch.float16, dev) for n in (rows * L, rows, rows))
    cti = _flat(rows, torch.uint8, dev)
    st = lib.mc_temporal_attn_fwd(_p(q), _p(k), _p(v), _lay(q), _p(co.t), _lay(co.t), _p(cp.t), _p(ctv.t), _p(cti.t),
                                  _p(idx), _p(cg.t), B, P, L, H, DH, float(scale), _stream())
    _lib.check(st, "mc_temporal_attn_fwd")
    torch.cuda.synchronize()
    co.check(o, f"L={L} o")
    cp.check(probs, f"L={L} probs")
    ctv.check(top[0], f"L={L} top_val")
    cti.check(top[1], f"L={L} top_idx")
    cg.check(gathered, f"L={L} gathered")

    if fused:  # the kernel moves dQ next to dK, dV and stores [dQ | dK | dV] per (frame, position) in one copy
        cf = _Canary((B, L + 1, P, 3 * C), (slice(None), slice(0, L)), torch.float16, dev)
        outs = {"dq": cf.t[..., :C], "dk": cf.t[..., C:2 * C], "dv": cf.t[..., 2 * C:]}
    else:
        cs = {n: _Canary((B, L + 1, P + 1, C + 8), (slice(None), slice(0, L), slice(0, P), slice(0, C)), torch.float16,
                         dev) for n in ("dq", "dk", "dv")}
        outs = {n: c.t for n, c in cs.items()}
    st = lib.mc_temporal_attn_bwd(_p(q), _p(k), _p(v), _lay(q), _p(d_o), _lay(d_o), _p(d_p), _p(idx), _p(d_g),
                                  _p(outs["dq"]), _p(outs["dk"]), _p(outs["dv"]), _lay(outs["dq"]), B, P, L, H, DH,
                                  float(scale), _stream())
    _lib.check(st, "mc_temporal_attn_bwd")
    torch.cuda.synchronize()
    if fused:
        cf.check(torch.cat(want_grads, dim=-1), f"L={L} dq|dk|dv")
    else:
        for (n, c), want in zip(cs.items(), want_grads):
            c.check(want, f"L={L} {n}")


@pytest.mark.parametrize("L", [0, 33])
def test_lengths_outside_1_to_32_are_rejected(L):
    dev = _dev()
    H, DH, B, P = 8, 40, 1, 4
    q, k, v = _make_qkv(B, max(L, 1), P, H * DH, seed=0, fused=False, dev=dev)
    q, k, v = (t[:, :L] for t in (q, k, v))
    d_o = torch.zeros_like(q)
    torch.cuda.synchronize()
    before = _lib.launch_count()
    with pytest.raises(NotImplementedError, match=r"1\.\.32"):
        ops.temporal_attention_forward(q, k, v, H, DH ** -0.5, want_probs=True, want_top1=True)
    with pytest.raises(NotImplementedError, match=r"1\.\.32"):
        ops.temporal_attention_backward(q, k, v, H, DH ** -0.5, d_o, None, None, None)
    if L > 0:
        with pytest.raises(NotImplementedError, match=r"1\.\.32"):
            ops.top1_rows(torch.rand(4, L, device=dev, dtype=torch.float16))
    torch.cuda.synchronize()
    assert _lib.launch_count() == before


# ---------------------------------------------------------------------------------------------------------------
# end to end on the reference fixtures (tests of test_pipeline_gpu.py, imported above)
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=["tiny12", "tiny5", "c2mini24"])
def run(request):
    """As test_pipeline_gpu.run: one UNet forward, the package's own extraction, and the sampling loop on the
    reference's motion representation, recording every step's latents and the guided steps' losses and gradients."""
    assert torch.cuda.is_available()
    dev = torch.device("cuda:0")
    pipe, g, meta, inp, ucfg = _build(request.param, dev)
    assert meta["infer"]["video_length"] not in (8, 16, 32)
    with torch.no_grad():
        fwd = pipe.unet(inp["noisy_latents"].to(dev, torch.float16), 500,
                        encoder_hidden_states=inp["text_embeddings"][[1]].to(dev, torch.float16)).sample
    rep = pipe.obtain_motion_representation(motion_representation_path=None)
    pipe.motion_representation_dict = {str(n): [torch.from_numpy(g[f"repr_val_{i}"]).half(),
                                                torch.from_numpy(g[f"repr_idx_{i}"])]
                                       for i, n in enumerate(g["repr_names"])}
    per_step, losses, grads = [], [], {}
    step = pipe.single_step_video

    def rec(lat, i, t, extra):
        out = step(lat, i, t, extra)
        per_step.append(out)
        if i < meta["infer"]["guidance_steps"]:
            losses.append(pipe.last_loss.float().item())
            grads[i] = pipe.last_gradient
        return out

    pipe.single_step_video = rec
    final = pipe.sample_video(noisy_latents=inp["noisy_latents"].to(dev, torch.float16), return_latents=True)
    return dict(case=request.param, pipe=pipe, g=g, meta=meta, inp=inp, ucfg=ucfg, fwd=fwd, rep=rep,
                per_step=per_step, losses=losses, grads=grads, final=final, dev=dev)


def test_graph_replay_and_representation_pack_at_12_frames():
    """CUDA-graph replay of the plain and unconditional forwards, and the broadcast packing of the motion representation,
    at a ragged clip length: replay is bit-identical to eager launches, and the packed representation round-trips."""
    import motionclone_b200 as mc
    from motionclone_b200 import dist as mcdist
    from motionclone_b200.synthetic import UNET_TINY_CONFIG, synthetic_inputs
    dev = _dev()
    _, meta = _load("tiny12")
    icfg = dict(meta["infer"])
    inp = synthetic_inputs(icfg["video_length"], icfg["height"], icfg["width"], UNET_TINY_CONFIG["cross_attention_dim"],
                           meta["input_seed"])
    icfg.update(video_latents=inp["clip_latents"].half(), video_noise=inp["clip_noise"].half(), new_prompt="synthetic")
    outs = []
    for graphs in (False, True):
        pipe = mc.build_pipeline(UNET_TINY_CONFIG, icfg, device=dev, weight_seed=meta["weight_seed"], use_cuda_graphs=graphs)
        pipe.set_prompt_embeds(inp["text_embeddings"].to(dev, torch.float16))
        rep = pipe.obtain_motion_representation(motion_representation_path=None)
        buf, manifest = mcdist.pack_representation(rep)
        back = mcdist.unpack_representation(buf, manifest)
        for n in rep:
            assert rep[n][1].shape[-2] == 12
            assert torch.equal(back[n][0], rep[n][0]) and torch.equal(back[n][1], rep[n][1])
        finals = [pipe.sample_video(noisy_latents=inp["noisy_latents"].to(dev, torch.float16), return_latents=True).clone()
                  for _ in range(2)]
        assert torch.equal(finals[0], finals[1])
        outs.append(finals[1])
    assert torch.equal(outs[0], outs[1])
