"""The small kernels around the tensor-core GEMMs, each called on its own through the C ABI and compared with a float64
reference computed from the same fp16 / fp32 values the kernel reads: conv_in (4 -> C), conv_out (C -> 3 / 4, with the
uint8 frame post-process), post_quant_conv (vae_in), the sinusoidal timestep embedding, the fp32 linear layers of the
time MLP, the row softmax of the unfused attention, and the circular padding / cropping of tiled mode.

Every output starts as NaN (or, for uint8, a fixed byte); bytes outside the view a kernel may write start as a
sentinel and must come back unchanged."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

pytestmark = pytest.mark.gpu

I64 = C.c_int64
SENT = -7.25  # sentinel value of the bytes around an output view


def _n():
    from stable_diffusion_videos_b200 import _native as n
    return n


def _p(t):
    return C.c_void_p(t.data_ptr() if t is not None else 0)


def _call(name, *args):
    n = _n()
    n.check(getattr(n.lib(), name)(*args, n.stream_ptr()))
    torch.cuda.synchronize()


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _ulp16(ref):
    """one fp16 ulp at the magnitude of `ref` (float64; 2^-24 in the subnormal range)."""
    e = torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e - 10)


def _padded(shape, view_c, c0, dtype, fill=float("nan"), sentinel=SENT):
    """a [.., width] buffer of `sentinel` with a [.., c0:c0 + view_c] view filled with `fill`."""
    buf = torch.full(shape, sentinel, dtype=dtype, device="cuda")
    view = buf[..., c0:c0 + view_c]
    view.fill_(fill)
    return buf, view


def _outside_unchanged(buf, c0, width, sentinel=SENT):
    outside = torch.cat([buf[..., :c0].flatten(), buf[..., c0 + width:].flatten()])
    return bool((outside == sentinel).all())


# ----------------------------------------------------------------------------------------------------------------------
# conv_in: 3x3 pad 1, 4 -> N
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [32, 40, 100, 320, 512])
@pytest.mark.parametrize("B,H,W", [(1, 1, 1), (2, 8, 8), (3, 7, 9), (2, 64, 64), (1, 96, 40)])
def test_conv_in_small(B, H, W, N):
    g = _gen(B * 1000 + H * 10 + N)
    w = (torch.randn(N, 4, 3, 3, generator=g) * 0.3).half().cuda()
    bias = torch.randn(N, generator=g).float().cuda()
    for ldx, with_bias in ((4, True), (8, False)):
        # the engine passes ldx = 4; with ldx = 8 the channels beyond the 4 read ones are NaN and must stay unread
        xb = torch.full((B, H, W, ldx), float("nan"), dtype=torch.float16)
        xb[..., :4] = torch.randn(B, H, W, 4, generator=g).half()
        xb = xb.cuda()
        x = xb[..., :4]
        c0, ldy = 8, N + 24
        ybuf, y = _padded((B, H, W, ldy), N, c0, torch.float16)
        b = bias if with_bias else None
        _call("sdw_conv_in_small", _p(xb), I64(ldx), B, H, W, 4, _p(w), _p(b), N, _p(y), I64(ldy))
        xd = x.double().permute(0, 3, 1, 2)
        wd = w.double()
        bd = b.double() if b is not None else None
        ref = Fn.conv2d(xd, wd, bd, padding=1).permute(0, 2, 3, 1)
        mag = Fn.conv2d(xd.abs(), wd.abs(), bd.abs() if bd is not None else None, padding=1).permute(0, 2, 3, 1)
        err = (y.double() - ref).abs()
        # one fp16 ulp of the exact value, plus the fp32 accumulation's rounding where the sum cancels to near zero
        tol = _ulp16(ref) + 2.0 ** -20 * mag
        assert bool((err <= tol).all()), (ldx, with_bias, float((err - tol).max()))
        assert _outside_unchanged(ybuf, c0, N)


# ----------------------------------------------------------------------------------------------------------------------
# conv_out: 3x3 pad 1, C -> 3 / 4, fp32 eps and / or the uint8 frame
# ----------------------------------------------------------------------------------------------------------------------
def _u8_of(v):
    """the post-process of stable_diffusion_pipeline.py:435-438 + numpy_to_pil, in the given dtype."""
    return torch.round(torch.clamp(v / 2 + 0.5, 0, 1) * 255)


@pytest.mark.parametrize("B,H,W,Cc,nout,slice_c", [
    (2, 24, 40, 128, 4, 0),    # 16 x 16 tiles, partial in W
    (1, 17, 33, 64, 3, 16),    # 16 x 16 tiles, ragged both ways; input is a channel slice (ldx > C)
    (2, 9, 13, 128, 4, 0),     # H < 16: 8 x 8 tiles
    (1, 5, 64, 64, 3, 0),      # 8 x 8 tiles, one partial tile row
    (3, 1, 1, 320, 4, 8),      # one pixel per sample, channel slice
    (2, 24, 40, 320, 3, 0),    # C = 320 (the UNet's conv_out): 8 x 8 tiles at any size
    (4, 96, 96, 320, 4, 0),    # 576 tiles: more than 2 x SM count, so each block runs the persistent tile loop
])
def test_conv_out_small(B, H, W, Cc, nout, slice_c):
    g = _gen(H * 100 + W + Cc)
    ldx = Cc + 2 * slice_c
    xb = torch.full((B, H, W, ldx), float("nan"), dtype=torch.float16)
    xb[..., slice_c:slice_c + Cc] = torch.randn(B, H, W, Cc, generator=g).half()
    xb = xb.cuda()
    x = xb[..., slice_c:slice_c + Cc]
    w = (torch.randn(nout, Cc, 3, 3, generator=g) * (0.6 / math.sqrt(9 * Cc))).half().cuda()
    bias = (torch.randn(nout, generator=g) * 0.2).float().cuda()
    P = B * H * W
    tail = 64

    def run(want_f32, want_u8):
        f32 = torch.full((P * nout + tail,), float("nan"), device="cuda") if want_f32 else None
        if f32 is not None:
            f32[P * nout:] = SENT
        u8 = torch.full((P * nout + tail,), 0xA5, dtype=torch.uint8, device="cuda") if want_u8 else None
        _call("sdw_conv_out_small", _p(x), I64(ldx), B, H, W, Cc, _p(w), _p(bias), nout, _p(f32), _p(u8))
        if f32 is not None:
            assert bool((f32[P * nout:] == SENT).all())
            f32 = f32[:P * nout].view(B, H, W, nout)
        if u8 is not None:
            assert bool((u8[P * nout:] == 0xA5).all())
            u8 = u8[:P * nout].view(B, H, W, nout)
        return f32, u8

    f32_only, _ = run(True, False)
    _, u8_only = run(False, True)
    f32, u8 = run(True, True)
    xd = x.double().permute(0, 3, 1, 2)
    wd = w.double()
    ref = Fn.conv2d(xd, wd, bias.double(), padding=1).permute(0, 2, 3, 1)
    mag = Fn.conv2d(xd.abs(), wd.abs(), bias.double().abs(), padding=1).permute(0, 2, 3, 1)
    for out in (f32_only, f32):
        err = (out.double() - ref).abs()
        assert bool((err <= 1e-5 * mag + 1e-6).all()), float((err - 1e-5 * mag).max())
    assert torch.equal(f32_only, f32)
    # the frame is exactly the fp32 post-process of the kernel's own fp32 value, and within 1 LSB of the exact one
    assert torch.equal(u8.to(torch.float32), _u8_of(f32))
    assert int((u8.double() - _u8_of(ref)).abs().max()) <= 1
    assert torch.equal(u8_only, u8)
    if P >= 1000:
        assert int(u8.min()) == 0 and int(u8.max()) == 255  # both clamps are exercised


# ----------------------------------------------------------------------------------------------------------------------
# vae_in: 1 / 0.18215 * latents, then post_quant_conv (1x1), NCHW fp32 -> NHWC fp16
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("F,Cc,H,W", [(3, 4, 7, 9), (1, 4, 33, 31), (2, 8, 13, 11), (2, 4, 64, 64)])
def test_vae_in(F, Cc, H, W):
    g = _gen(F * 7 + Cc + H)
    x = (torch.randn(F, Cc, H, W, generator=g) * 0.9).float().cuda()
    w = (torch.randn(Cc, Cc, generator=g) * 0.5).half().cuda()
    bias = torch.randn(Cc, generator=g).float().cuda()
    P = F * H * W
    z = torch.full((P * Cc + 40,), float("nan"), dtype=torch.float16, device="cuda")
    z[P * Cc:] = SENT
    inv = 1.0 / 0.18215
    _call("sdw_vae_in", _p(x), C.c_float(inv), _p(w), _p(bias), F, Cc, H, W, _p(z))
    assert bool((z[P * Cc:] == SENT).all())
    zz = z[:P * Cc].view(F, H, W, Cc).double()
    xs = x.double().permute(0, 2, 3, 1) / 0.18215
    ref = xs @ w.double().T + bias.double()
    mag = xs.abs() @ w.double().abs().T + bias.double().abs()
    err = (zz - ref).abs()
    tol = _ulp16(ref) + 2.0 ** -20 * mag
    assert bool((err <= tol).all()), float((err - tol).max())


# ----------------------------------------------------------------------------------------------------------------------
# timestep embedding and the fp32 time MLP
# ----------------------------------------------------------------------------------------------------------------------
def _timestep_tables():
    from stable_diffusion_videos_b200.schedulers import EulerDiscreteScheduler, LMSDiscreteScheduler, PNDMScheduler

    out = []
    for sch, n in ((PNDMScheduler(), 50), (LMSDiscreteScheduler(), 50), (EulerDiscreteScheduler(), 30)):
        sch.set_timesteps(n)
        out.append(np.asarray(sch.timesteps, dtype=np.float32))
    out.append(np.array([0.0, 999.0], dtype=np.float32))
    t = np.concatenate(out)
    assert (t != np.round(t)).any()  # the K-LMS / Euler tables have fractional timesteps
    return torch.from_numpy(t)


def _sinusoid64(t, dim):
    """diffusers get_timestep_embedding (flip_sin_to_cos, freq_shift 0), the formula of oracle.unet.timestep_embedding,
    in float64."""
    half = dim // 2
    freq = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float64) / half)
    a = t.double()[:, None] * freq[None, :]
    return torch.cat([torch.cos(a), torch.sin(a)], dim=-1)


@pytest.mark.parametrize("dim", [32, 320])
def test_timestep_embed(dim):
    from oracle.unet import timestep_embedding

    t = _timestep_tables()
    n = t.numel()
    td = t.cuda()
    outs = []
    for rnd in (0, 1):
        out = torch.full((n * dim + 16,), float("nan"), device="cuda")
        out[n * dim:] = SENT
        _call("sdw_timestep_embed", _p(td), n, dim, rnd, _p(out))
        assert bool((out[n * dim:] == SENT).all())
        outs.append(out[:n * dim].view(n, dim).cpu())
    ref = _sinusoid64(t, dim)
    assert float((ref - timestep_embedding(t, dim).double()).abs().max()) <= 1e-4  # the oracle states the same formula
    # the fp32 argument t * f carries ~6e-5 of rounding at t = 999
    assert float((outs[0].double() - ref).abs().max()) <= 1e-4
    assert torch.equal(outs[1], outs[0].half().float())


def _linear64(a, w, b, silu_in, silu_out):
    a = a.double()
    if silu_in:
        a = Fn.silu(a)
    y = a @ w.double().T
    mag = a.abs() @ w.double().abs().T
    if b is not None:
        y = y + b.double()
        mag = mag + b.double().abs()
    return (Fn.silu(y) if silu_out else y), mag


@pytest.mark.parametrize("K", [33, 320, 1280])
@pytest.mark.parametrize("N", [1, 320, 1280])
@pytest.mark.parametrize("M", [1, 50, 51])
def test_linear_f32(M, N, K):
    g = _gen(M * 31 + N * 7 + K)
    w = (torch.randn(N, K, generator=g) / math.sqrt(K)).half().cuda()
    bias = torch.randn(N, generator=g).float().cuda()
    a = (torch.randn(M, K, generator=g) * 2).float().cuda()
    variants = [(si, so, K, N, True) for si in (0, 1) for so in (0, 1)]
    variants.append((1, 0, K + 5, N + 3, False))  # pitched input and output, no bias
    for si, so, ldi, ldo, with_bias in variants:
        ab = torch.full((M, ldi), float("nan"), device="cuda")
        ab[:, :K] = a
        ob, o = _padded((M, ldo), N, 0, torch.float32)
        b = bias if with_bias else None
        _call("sdw_linear_f32", _p(ab), I64(ldi), _p(w), _p(b), M, N, K, si, so, _p(ob), I64(ldo))
        ref, mag = _linear64(a, w, b, si, so)
        err = (o.double() - ref).abs()
        assert bool((err <= 1e-5 * mag + 1e-6).all()), (si, so, ldi, ldo, float((err - 1e-5 * mag).max()))
        assert _outside_unchanged(ob, 0, N)


def test_time_embedding_chain_matches_oracle():
    """the chain the engine evaluates once per schedule: sinusoid -> linear_1 + SiLU -> linear_2 -> each ResBlock's
    time projection (with the SiLU on its input), against the oracle's TimestepEmbedding in float64 on the same fp16
    weights."""
    from oracle.unet import TimestepEmbedding

    c0, tc, couts = 320, 1280, (320, 640, 1280)
    torch.manual_seed(0)
    te = TimestepEmbedding(c0, tc).double()
    projs = [torch.nn.Linear(tc, c).double() for c in couts]
    with torch.no_grad():
        for m in [te] + projs:
            for p in m.parameters():
                p.copy_(p.half().double())
    t = _timestep_tables()
    n = t.numel()

    def dev(p, half):
        return p.detach().to(torch.float16 if half else torch.float32).cuda().contiguous()

    sin = torch.empty(n, c0, device="cuda")
    h1 = torch.empty(n, tc, device="cuda")
    temb = torch.empty(n, tc, device="cuda")
    _call("sdw_timestep_embed", _p(t.cuda()), n, c0, 0, _p(sin))
    w1, b1 = dev(te.linear_1.weight, True), dev(te.linear_1.bias, False)
    w2, b2 = dev(te.linear_2.weight, True), dev(te.linear_2.bias, False)
    _call("sdw_linear_f32", _p(sin), I64(c0), _p(w1), _p(b1), n, tc, c0, 0, 1, _p(h1), I64(tc))
    _call("sdw_linear_f32", _p(h1), I64(tc), _p(w2), _p(b2), n, tc, tc, 0, 0, _p(temb), I64(tc))
    with torch.no_grad():
        s64 = _sinusoid64(t, c0)
        ref_temb = te(s64)
        # worst-case propagation of the sinusoid's 1e-4 and of each layer's own fp32 rounding (1e-5 of its magnitude)
        bound = torch.full_like(s64, 1e-4)
        a1 = s64 @ te.linear_1.weight.T + te.linear_1.bias
        bound = bound @ te.linear_1.weight.abs().T + 1e-5 * (s64.abs() @ te.linear_1.weight.abs().T + te.linear_1.bias.abs())
        bound = 1.1 * bound  # SiLU is 1.1-Lipschitz
        s1 = Fn.silu(a1)
        bound = bound @ te.linear_2.weight.abs().T + 1e-5 * (s1.abs() @ te.linear_2.weight.abs().T + te.linear_2.bias.abs())
    err = (temb.cpu().double() - ref_temb).abs()
    assert bool((err <= bound + 1e-6).all()), float((err - bound).max())
    for proj in projs:
        cout = proj.out_features
        out = torch.empty(n, cout, device="cuda")
        _call("sdw_linear_f32", _p(temb), I64(tc), _p(dev(proj.weight, True)), _p(dev(proj.bias, False)), n, cout, tc,
              1, 0, _p(out), I64(cout))
        with torch.no_grad():
            st = Fn.silu(ref_temb)
            ref = proj(st)
            pb = (1.1 * bound) @ proj.weight.abs().T + 1e-5 * (st.abs() @ proj.weight.abs().T + proj.bias.abs())
        err = (out.cpu().double() - ref).abs()
        assert bool((err <= pb + 1e-6).all()), (cout, float((err - pb).max()))


# ----------------------------------------------------------------------------------------------------------------------
# row softmax (unfused attention)
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 77, 1023, 1024, 1025, 4096, 4100])
@pytest.mark.parametrize("wide", [0, 1])
def test_softmax_rows(n, wide):
    """n <= 1024 takes the warp-per-row kernel, longer rows the block-per-row one"""
    g = _gen(n * 2 + wide)
    rows = 13
    ld = n + 64 if wide else (n + 7) // 8 * 8
    x = (torch.randn(rows, n, generator=g) * 4).half()
    x[3] = torch.linspace(-60000, 60000, n).half()[torch.randperm(n, generator=g)]  # +-60000 spread
    x[7] = 1.5  # a row of equal values
    x[8] = -3000.0
    buf = torch.full((rows, ld), float("nan"), dtype=torch.float16)
    buf[:, :n] = x
    buf = buf.cuda()
    pad_before = buf[:, n:].clone()
    _call("sdw_softmax_rows", _p(buf), I64(ld), I64(rows), n)
    ref = torch.softmax(x.double(), -1)
    got = buf[:, :n].cpu().double()
    err = (got - ref).abs()
    tol = _ulp16(ref) + 2.0 ** -24
    assert bool((err <= tol).all()), float((err - tol).max())
    assert torch.equal(buf[:, n:].view(torch.int16), pad_before.view(torch.int16))  # NaN padding untouched


@pytest.mark.parametrize("N", [64, 1024, 4096])
def test_unfused_attention_vae_mid_block(N):
    """the VAE mid-block attention as the engine runs it (d = 512 is beyond the flash kernel): batched QK^T GEMM with
    alpha = d^-1/2 into a score matrix of pitch ceil8(Nk), row softmax, batched PV GEMM on V^T."""
    n = _n()
    d, heads, B = 512, 1, 1
    g = _gen(N)
    q = torch.randn(B, N, d, generator=g).half().cuda()
    k = torch.randn(B, N, d, generator=g).half().cuda()
    v = torch.randn(B, N, d, generator=g).half().cuda()
    Nkp = (N + 7) // 8 * 8
    vt = torch.full((B, heads, d, Nkp), float("nan"), dtype=torch.float16, device="cuda")
    vt[..., :N] = v.reshape(B, N, heads, d).permute(0, 2, 3, 1)
    S = torch.full((B, heads, N, Nkp), float("nan"), dtype=torch.float16, device="cuda")
    out = torch.full((B, N, d), float("nan"), dtype=torch.float16, device="cuda")
    gd = n.GemmDesc()
    gd.A, gd.C, gd.W, gd.H, gd.B = q.data_ptr(), d, N, heads, B
    gd.sW, gd.sH, gd.sB = d, d, N * d
    gd.Wt, gd.N, gd.ldb, gd.Kb = k.data_ptr(), N, d, d
    gd.b_batched, gd.sBh, gd.sBb = 1, d, N * d
    gd.out, gd.ldc = S.data_ptr(), Nkp
    gd.o_sW, gd.o_sH, gd.o_sB = Nkp, N * Nkp, heads * N * Nkp
    gd.alpha = 1.0 / math.sqrt(d)
    n.gemm(gd)
    _call("sdw_softmax_rows", _p(S), I64(Nkp), I64(B * heads * N), N)
    hd = n.GemmDesc()
    hd.A, hd.C, hd.W, hd.H, hd.B = S.data_ptr(), N, N, heads, B
    hd.sW, hd.sH, hd.sB = Nkp, N * Nkp, heads * N * Nkp
    hd.Wt, hd.N, hd.ldb, hd.Kb = vt.data_ptr(), d, Nkp, N
    hd.b_batched, hd.sBh, hd.sBb = 1, d * Nkp, heads * d * Nkp
    hd.out, hd.ldc = out.data_ptr(), d
    hd.o_sW, hd.o_sH, hd.o_sB = d, d, N * d
    hd.alpha = 1.0
    n.gemm(hd)
    torch.cuda.synchronize()
    ref = torch.softmax(q.double() @ k.double().transpose(-1, -2) * d ** -0.5, -1) @ v.double()
    assert bool(torch.isfinite(out).all())
    err = float((out.double() - ref).abs().max())
    assert err <= 2.0 ** -8 * float(ref.abs().max()) + 1e-3, err


# ----------------------------------------------------------------------------------------------------------------------
# tiled mode: circular padding and interior crop
# ----------------------------------------------------------------------------------------------------------------------
# (dtype, channels, pixel pitch in elements): 16-byte, 8-byte and 1-byte copy paths
LAYOUTS = [(torch.float16, 320, 328), (torch.float16, 8, 16), (torch.float16, 4, 8), (torch.float32, 3, 5),
           (torch.float32, 4, 8), (torch.uint8, 3, 5)]
IMAGES = [(2, 5, 7, 1), (2, 5, 7, 2), (1, 1, 1, 1), (2, 2, 2, 2), (1, 9, 13, 1)]


def _random_pixels(shape, dtype, g):
    if dtype == torch.uint8:
        return torch.randint(0, 256, shape, generator=g, dtype=torch.uint8)
    return torch.randn(shape, generator=g).to(dtype)


def _circular(x, pad):
    """torch circular padding of an NHWC image, as an index map (also valid where pad equals the image size)."""
    B, H, W, _ = x.shape
    iy = torch.arange(-pad, H + pad, device=x.device) % H
    ix = torch.arange(-pad, W + pad, device=x.device) % W
    return x[:, iy][:, :, ix]


def _bytes(t):
    return t.contiguous().view(torch.uint8)


@pytest.mark.parametrize("dtype,Cc,ld", LAYOUTS)
@pytest.mark.parametrize("B,H,W,pad", IMAGES)
def test_wrap_pad_and_crop(dtype, Cc, ld, B, H, W, pad):
    g = _gen(Cc * 100 + H * 10 + pad)
    es = torch.tensor([], dtype=dtype).element_size()
    xb = _random_pixels((B, H, W, ld), dtype, g).cuda()
    x = xb[..., :Cc]
    Hp, Wp = H + 2 * pad, W + 2 * pad
    ny = B * Hp * Wp * Cc
    ybuf = torch.full((ny * es + 32,), 0x5A, dtype=torch.uint8, device="cuda")  # byte sentinel; the tail must survive
    ybuf_t = ybuf[:ny * es].view(dtype)
    _call("sdw_wrap_pad", _p(xb), I64(ld * es), B, H, W, Cc * es, pad, _p(ybuf_t))
    y = ybuf_t.view(B, Hp, Wp, Cc)
    if dtype == torch.float32 and pad < min(H, W):
        ref_pad = Fn.pad(x.permute(0, 3, 1, 2), (pad, pad, pad, pad), mode="circular").permute(0, 2, 3, 1)
        assert torch.equal(_bytes(ref_pad), _bytes(_circular(x, pad)))
    assert torch.equal(_bytes(y), _bytes(_circular(x, pad)))
    assert bool((ybuf[ny * es:] == 0x5A).all())
    # crop back into an output of the input's (wider than a pixel) pitch, pad channels at a byte sentinel: the round trip
    # is the identity
    ob = torch.full((B * H * W * ld * es,), 0x33, dtype=torch.uint8, device="cuda")
    out = ob.view(dtype).view(B, H, W, ld)
    _call("sdw_crop_interior", _p(y), B, H, W, Cc * es, pad, C.c_void_p(0), I64(0), _p(out), I64(ld * es))
    assert torch.equal(_bytes(out[..., :Cc]), _bytes(x))
    assert bool((_bytes(out[..., Cc:]) == 0x33).all())


@pytest.mark.parametrize("Cc", [320, 8])
@pytest.mark.parametrize("B,H,W,crop", [(2, 5, 7, 1), (1, 6, 3, 2), (1, 1, 1, 1)])
def test_crop_interior_residual_add(Cc, B, H, W, crop):
    """the fp16 crop adds the residual in fp32 and rounds once, as the GEMM epilogue it replaces"""
    g = _gen(Cc + H + crop)
    Hp, Wp = H + 2 * crop, W + 2 * crop
    yp = torch.randn(B, Hp, Wp, Cc, generator=g).half().cuda()
    ldr = Cc + 8
    rb = torch.full((B, H, W, ldr), float("nan"), dtype=torch.float16)
    rb[..., :Cc] = torch.randn(B, H, W, Cc, generator=g).half()
    rb = rb.cuda()
    ldo = Cc + 16
    obuf, out = _padded((B, H, W, ldo), Cc, 8, torch.float16)
    _call("sdw_crop_interior", _p(yp), B, H, W, Cc * 2, crop, _p(rb), I64(ldr), _p(out), I64(ldo * 2))
    ref = (yp[:, crop:crop + H, crop:crop + W].float() + rb[..., :Cc].float()).half()
    assert torch.equal(out.view(torch.int16), ref.view(torch.int16))
    assert _outside_unchanged(obuf, 8, Cc)
