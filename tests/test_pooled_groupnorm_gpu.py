"""Frame-pooled GroupNorm kernels (mc_groupnorm_nhwc_pooled / mc_groupnorm_nhwc_bwd_pooled): statistics over each run of F
consecutive frames, as torch.nn.GroupNorm on the 5-D [b, C, F, H, W] tensor (models/resnet.py:143-146, 162-165 and
models/unet.py:244-247 with use_inflated_groupnorm=False).

  * forward against fp32 F.group_norm on the 5-D view, at the bar of test_kernels_gpu.py::test_groupnorm_nhwc, on
    inputs whose per-frame means drift across the clip (the per-frame kernels fail that bar there);
  * backward against fp32 autograd at the bars of test_groupnorm_nhwc_backward;
  * exact cases: F = 1 is the per-frame entry point bit for bit; each sample of a batched call (including the plain
    step's N = 2Bf layout with samples = B) gets the bits of its single-sample call; repeated calls agree bitwise and
    leave the ticket region zero, also after a rejected call; full-size calls are deterministic;
  * rejections: F <= 0, N % F != 0 and (N / samples) % F != 0 launch nothing.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

G, EPS = 32, 1e-5
CL = torch.channels_last

# (C, h) of every resnet norm1 / norm2 and conv_norm_out of the SD1.5 UNet at 512 x 512 (latent 64) and 128 x 128
# (latent 16): down 320 / 640 / 1280 / 1280, mid 1280, up 2560 / 2560+1920 / 1920+1280+960 / 960+640+320
_LEVELS = [(320, 1), (640, 2), (320, 2), (1280, 4), (640, 4), (1280, 8), (2560, 8), (2560, 4), (1920, 4), (1920, 2),
           (1280, 2), (960, 2), (960, 1), (640, 1)]
SHAPES = sorted({(C, 64 // d) for C, d in _LEVELS} | {(C, 16 // d) for C, d in _LEVELS})


def _ops():
    from motionclone_b200 import ops
    return ops


def _lib():
    from motionclone_b200 import _lib
    return _lib


def _dev():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    return torch.device("cuda:0")


def _inputs(N, C, h, frames, seed, with_bias, drift=3.0):
    """x [N, C, h, h] channels_last fp16 whose per-frame mean drifts linearly over each clip of `frames` frames."""
    g = torch.Generator().manual_seed(seed)
    f = torch.arange(N) % frames
    ramp = drift * (f.float() / max(frames - 1, 1) - 0.5)
    x = torch.randn(N, C, h, h, generator=g) * 2 + 0.5 + ramp[:, None, None, None] \
        + 0.5 * torch.randn(1, C, 1, 1, generator=g)
    dev = _dev()
    x = x.to(dev, torch.float16).contiguous(memory_format=CL)
    w = (1 + 0.1 * torch.randn(C, generator=g)).to(dev, torch.float16)
    b = (0.1 * torch.randn(C, generator=g)).to(dev, torch.float16)
    cb = torch.randn(N // frames, C, generator=g).to(dev, torch.float16) if with_bias else None
    return x, w, b, cb


def _pooled_ref(x, w, b, cb, frames, silu, dtype):
    """torch.nn.GroupNorm on the 5-D [N / F, C, F, h, w] view (`dtype`: fp32 truth or the fp16 eager graph)."""
    N, C, H, W = x.shape
    xin = x if cb is None else x + cb.repeat_interleave(frames, dim=0)[:, :, None, None]  # the fp16 `h + temb`
    x5 = xin.to(dtype).contiguous().reshape(N // frames, frames, C, H, W).permute(0, 2, 1, 3, 4)
    y = F.group_norm(x5, G, w.to(dtype), b.to(dtype), EPS)
    if silu:
        y = F.silu(y)
    return y.permute(0, 2, 1, 3, 4).reshape(N, C, H, W)


def _fwd(x, w, b, cb, frames, silu, samples=1):
    return _ops().groupnorm_nhwc(x, w, b, G, EPS, silu, cb, want_stats=True, samples=samples, frames_per_stat=frames)


def _fwd_bwd(x, w, b, cb, frames, silu, dz, samples=1):
    xg = x.clone().requires_grad_(True)
    y = _ops().GroupNormNHWCFn.apply(xg, w, b, cb, G, EPS, silu, samples, frames)
    (dx,) = torch.autograd.grad(y, xg, dz)
    return y.detach(), dx


def _check_forward(N, C, h, frames, silu, with_bias, seed):
    x, w, b, cb = _inputs(N, C, h, frames, seed, with_bias)
    with torch.no_grad():
        y, stats = _fwd(x, w, b, cb, frames, silu)
        y_pf = _ops().groupnorm_nhwc(x, w, b, G, EPS, silu, cb)
        ref = _pooled_ref(x, w, b, cb, frames, silu, torch.float32)
        eager = _pooled_ref(x, w, b, cb, frames, silu, torch.float16)
    assert y.is_contiguous(memory_format=CL)
    err, err_eager = (y.float() - ref).abs().max().item(), (eager.float() - ref).abs().max().item()
    bar = max(6e-3, 1.5 * err_eager)
    assert err <= bar, (err, err_eager)
    assert torch.equal(stats.view(N // frames, frames, G, 2), stats[::frames, None].expand(-1, frames, -1, -1))
    if frames > 1:  # the drifting means make the two modes differ far beyond the bar
        assert (y_pf.float() - ref).abs().max().item() > 10 * bar


@pytest.mark.parametrize("C,h", SHAPES)
def test_pooled_forward_unet_shapes(C, h):
    i = SHAPES.index((C, h))
    frames = 16 if h * h * C <= 64 * 64 * 640 else 8
    _check_forward(frames * (1 + i % 2), C, h, frames, silu=i % 3 != 0, with_bias=i % 2 == 0, seed=C + h)


@pytest.mark.parametrize("frames", [1, 5, 8, 12, 16, 24, 32])
@pytest.mark.parametrize("b", [1, 2])
@pytest.mark.parametrize("silu,with_bias", [(True, True), (False, False), (True, False), (False, True)])
@pytest.mark.parametrize("C,h", [(320, 32), (1280, 8), (2560, 4)])
def test_pooled_forward_frame_sweep(frames, b, silu, with_bias, C, h):
    _check_forward(b * frames, C, h, frames, silu, with_bias, seed=frames * 7 + b + C)


@pytest.mark.parametrize("N,C,h,frames,silu,with_bias", [
    (16, 320, 64, 16, True, True), (16, 320, 32, 8, True, False), (24, 640, 32, 12, True, True),
    (16, 1280, 16, 16, False, True), (32, 1280, 8, 16, True, True), (24, 2560, 8, 24, True, False),
    (10, 1920, 16, 5, True, True), (32, 960, 32, 32, False, False), (16, 64, 16, 8, True, True)])
def test_pooled_backward(N, C, h, frames, silu, with_bias):
    x, w, b, cb = _inputs(N, C, h, frames, C + h + N, with_bias)
    dz = torch.randn(x.shape, generator=torch.Generator().manual_seed(N)).to(x.device, torch.float16) \
        .contiguous(memory_format=CL)
    y, dx = _fwd_bwd(x, w, b, cb, frames, silu, dz)
    assert dx.is_contiguous(memory_format=CL)
    xr = x.float().clone().requires_grad_(True)
    xin = xr if cb is None else xr + cb.float().repeat_interleave(frames, dim=0)[:, :, None, None]
    x5 = xin.reshape(N // frames, frames, C, h, h).permute(0, 2, 1, 3, 4)
    yr = F.group_norm(x5, G, w.float(), b.float(), EPS)
    if silu:
        yr = F.silu(yr)
    yr = yr.permute(0, 2, 1, 3, 4).reshape(N, C, h, h)
    (dr,) = torch.autograd.grad(yr, xr, dz.float())
    assert (y.float() - yr).abs().max().item() <= 8e-3
    scale = dr.abs().max().item() + 1e-12
    err = (dx.float() - dr).abs().max().item()
    assert err <= 1e-2 * scale + 1e-6, f"pooled groupnorm dx: max err {err} vs scale {scale}"


@pytest.mark.parametrize("N,C,h", [(16, 320, 64), (8, 640, 32), (12, 1280, 16), (32, 2560, 8), (3, 960, 4)])
@pytest.mark.parametrize("silu,with_bias", [(True, True), (False, False)])
def test_pooled_f1_is_per_frame_bitwise(N, C, h, silu, with_bias):
    x, w, b, cb = _inputs(N, C, h, N, C + N, with_bias)
    dz = torch.randn(x.shape, generator=torch.Generator().manual_seed(C)).to(x.device, torch.float16) \
        .contiguous(memory_format=CL)
    with torch.no_grad():
        y1, s1 = _fwd(x, w, b, cb, 1, silu)
        y0, s0 = _fwd(x, w, b, cb, None, silu)
    assert torch.equal(y1, y0) and torch.equal(s1, s0)
    _, dx1 = _fwd_bwd(x, w, b, cb, 1, silu, dz)
    _, dx0 = _fwd_bwd(x, w, b, cb, None, silu, dz)
    assert torch.equal(dx1, dx0)


@pytest.mark.parametrize("B", [2, 3])
@pytest.mark.parametrize("plain_pass", [False, True])
@pytest.mark.parametrize("frames,C,h", [(16, 320, 64), (8, 640, 32), (12, 1280, 16), (16, 2560, 8)])
def test_pooled_batched_sample_bits(B, plain_pass, frames, C, h):
    """Sample s of a batched call = its single-sample call, bitwise. plain_pass: the CFG pass of a plain step, b = 2B
    UNet rows with samples = B, so a tiling sample is 2f frames holding two pools of f."""
    unit = 2 * frames if plain_pass else frames
    x, w, b, cb = _inputs(B * unit, C, h, frames, C + B + unit, True)
    dz = torch.randn(x.shape, generator=torch.Generator().manual_seed(B)).to(x.device, torch.float16) \
        .contiguous(memory_format=CL)
    with torch.no_grad():
        y, st = _fwd(x, w, b, cb, frames, True, samples=B)
    _, dx = _fwd_bwd(x, w, b, cb, frames, True, dz, samples=B)
    per = unit // frames  # chan_bias rows (pools) per sample
    for s in range(B):
        sl = slice(s * unit, (s + 1) * unit)
        xs = x[sl].contiguous(memory_format=CL)
        cbs = cb[s * per:(s + 1) * per]
        with torch.no_grad():
            ys, sts = _fwd(xs, w, b, cbs, frames, True)
        _, dxs = _fwd_bwd(xs, w, b, cbs, frames, True, dz[sl].contiguous(memory_format=CL))
        assert torch.equal(y[sl], ys) and torch.equal(st[sl], sts) and torch.equal(dx[sl], dxs), s


def _abi_call(x, w, b, ws, y, N, HW, C, samples, frames):
    L = _lib().lib()
    ops = _ops()
    return L.mc_groupnorm_nhwc_pooled(ops._ptr(x), None, 0, ops._ptr(y), ops._ptr(w), ops._ptr(b), ops._ptr(ws),
                                      ws.numel(), N, HW, C, G, samples, frames, EPS, 1, ops._stream())


def _abi_bwd(x, dz, dx, stats, w, b, ws, N, HW, C, samples, frames):
    L = _lib().lib()
    ops = _ops()
    return L.mc_groupnorm_nhwc_bwd_pooled(ops._ptr(x), None, 0, ops._ptr(dz), ops._ptr(dx), ops._ptr(stats),
                                          ops._ptr(w), ops._ptr(b), ops._ptr(ws), ws.numel(), N, HW, C, G, samples,
                                          frames, 1, ops._stream())


def test_pooled_repeat_and_tickets_return_to_zero():
    """Alternating inputs on one workspace: every call gives the same bits as the first call on that input (stale
    statistics would show), and the 8 KB ticket region is zero after every call, including a rejected one."""
    N, C, h, frames = 16, 320, 64, 8
    xa, w, b, _ = _inputs(N, C, h, frames, 1, False)
    xb, _, _, _ = _inputs(N, C, h, frames, 2, False, drift=-5.0)
    L = _lib().lib()
    ws = torch.zeros(int(L.mc_groupnorm_workspace_bytes(N, G)), dtype=torch.uint8, device=xa.device)
    wsb = torch.zeros_like(ws)
    dz = torch.randn(xa.shape, generator=torch.Generator().manual_seed(3)).to(xa.device, torch.float16) \
        .contiguous(memory_format=CL)
    stats = torch.empty(N, G, 2, dtype=torch.float32, device=xa.device)
    first = {}
    for it in range(3):
        for name, x in (("a", xa), ("b", xb)):
            y, dx = torch.empty_like(x), torch.empty_like(x)
            assert _abi_call(x, w, b, ws, y, N, h * h, C, 1, frames) == 0
            _lib().check(L.mc_groupnorm_nhwc_stats(_ops()._ptr(ws), _ops()._ptr(stats), N, h * h, G, EPS,
                                                   _ops()._stream()), "stats")
            assert _abi_bwd(x, dz, dx, stats, w, b, wsb, N, h * h, C, 1, frames) == 0
            assert _abi_call(x, w, b, ws, y, N, h * h, C, 1, 3) != 0  # rejected: 16 % 3
            torch.cuda.synchronize()
            assert not ws[:8192].any().item() and not wsb[:8192].any().item()
            out = (y.clone(), stats.clone(), dx.clone())
            if it == 0:
                first[name] = out
                with torch.no_grad():
                    ref = _pooled_ref(x, w, b, None, frames, True, torch.float32)
                assert (y.float() - ref).abs().max().item() <= 6e-3 * 4
            else:
                assert all(torch.equal(u, v) for u, v in zip(out, first[name])), (it, name)
    assert not torch.equal(first["a"][0], first["b"][0])


@pytest.mark.parametrize("frames", [16, 32])
def test_pooled_full_size_deterministic(frames):
    x, w, b, cb = _inputs(frames, 320, 64, frames, frames, True)
    dz = torch.randn(x.shape, generator=torch.Generator().manual_seed(5)).to(x.device, torch.float16) \
        .contiguous(memory_format=CL)
    runs = [_fwd_bwd(x, w, b, cb, frames, True, dz) for _ in range(3)]
    for y, dx in runs[1:]:
        assert torch.equal(y, runs[0][0]) and torch.equal(dx, runs[0][1])


@pytest.mark.parametrize("N,samples,frames", [(16, 1, 0), (16, 1, -1), (16, 1, 3), (16, 2, 16), (24, 2, 8),
                                              (12, 4, 2 * 3)])
def test_pooled_rejections_launch_nothing(N, samples, frames):
    C, h = 320, 16
    x, w, b, _ = _inputs(N, C, h, N, 9, False)
    L = _lib().lib()
    ws = torch.zeros(int(L.mc_groupnorm_workspace_bytes(N, G)), dtype=torch.uint8, device=x.device)
    y, dx = torch.empty_like(x), torch.empty_like(x)
    stats = torch.zeros(N, G, 2, dtype=torch.float32, device=x.device)
    before = _lib().launch_count()
    assert _abi_call(x, w, b, ws, y, N, h * h, C, samples, frames) == -1
    assert "frames_per_stat" in L.mc_last_error().decode()
    assert _abi_bwd(x, x, dx, stats, w, b, ws, N, h * h, C, samples, frames) == -1
    assert "frames_per_stat" in L.mc_last_error().decode()
    assert _lib().launch_count() == before
    with pytest.raises(_lib().MotionCloneKernelError):
        _ops().groupnorm_nhwc(x, w, b, G, EPS, True, samples=samples, frames_per_stat=frames)
    assert _lib().launch_count() == before
    torch.cuda.synchronize()
    assert not ws.any().item()
