"""Every distinct op of the benchmarked 30-frame SD-1.4 engine (512 x 512 frames: UNet batch 60, VAE batch 30), run
alone through its own entry point and compared with a float64 reference computed on the device from the same fp16
inputs; then the ops of a 33-frame engine whose VAE tensors pass 2^31 bytes.

The op list comes from `sdw_engine_debug_ops` of a plan-only engine (tests/_engine_ops.py): no arena is allocated.
Each distinct record is replayed once on seeded random data with the recorded extents and strides and every variant
knob left automatic, so the planner picks what it picks inside the engine (asserted through `sdw_debug_plan`).
Outputs start as NaN; every other element of an output buffer (neighbouring channels of a slice, other parities of the
folded upsampler, other rows) starts as a sentinel and must come back unchanged.

GEMM bound, per element (derivation).  Let z = alpha * sum_k a_k w_k + bias + rowvec be the exact pre-activation value
of the fp16 inputs and S = |alpha| * sum_k |a_k| |w_k| (both float64).  The kernel accumulates in fp32 registers: each
of the K / 16 wgmma k-steps adds one 16-product partial sum into the accumulator.  With u32 = 2^-24 and allowing each
addition twice the round-to-nearest unit (tensor-core alignment truncates), the accumulation error is at most
    (K / 16 + 1) * 2 * 2 * u32 * S
(one term per k-step plus the in-instruction sum).  The epilogue's fp32 scale / bias / row-vector additions round at
most three more times: 4 * u32 * (|alpha acc| + |bias| + |rowvec|).  The activation multiplies that error by its
derivative (SiLU: |silu'(z)| <= 1.1; GEGLU a * gelu(g): |gelu(g)| for the error of a plus |a| |gelu'(g)| for the error
of g, |gelu'| <= 1.13) and adds its own fp32 evaluation error (SiLU with __expf: (4 + 1.2 |z|) * 2^-22 * |silu(z)|;
GEGLU's erf polynomial, Abramowitz-Stegun 7.1.26, |error| <= 1.5e-7, rounded up to 2.5e-7 for its approximate
reciprocal: |a| * 0.5 |g| * 2.5e-7 plus 2^-21 |out|).  The residual add rounds once (2 u32 |resid|) and the fp16 store
rounds once: 2^-11 |ref| + 2^-25 (half the subnormal spacing).  The sum of these terms is the bound; nothing in it is
fitted to observed errors.

GroupNorm, LayerNorm, attention, the row softmax and the edge convs keep the tolerances of tests/test_norm_gpu.py,
tests/test_attn_gpu.py and tests/test_edge_kernels_gpu.py.
"""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as Fn

from _engine_ops import PLAN_FIELDS, gemm_desc, plan_of, plan_only_ops

pytestmark = pytest.mark.gpu

F = 30
SENT = -7.25
I64 = C.c_int64
CHUNK_ELEMS = 1 << 27  # float64 elements of one reference chunk (1 GB)


def _n():
    from stable_diffusion_videos_b200 import _native as n
    return n


def _call(name, *args):
    n = _n()
    n.check(getattr(n.lib(), name)(*args, n.stream_ptr()))
    torch.cuda.synchronize()


def _p(t):
    return C.c_void_p(t.data_ptr() if t is not None else 0)


def _distinct(recs, kinds=None):
    seen = {}
    for sec, _, kind, f in recs:
        if kinds is None or kind in kinds:
            seen.setdefault((kind, tuple(sorted(f.items()))), (sec, kind, f))
    return list(seen.values())


@pytest.fixture(scope="module")
def ops30():
    recs, _, arena = plan_only_ops(F)
    trecs, _, tarena = plan_only_ops(F, tiled=True)
    print(f"\nF = {F} engine arena: {arena} bytes ({arena / 2**30:.2f} GiB); tiled: {tarena} bytes")
    return recs, trecs


class Rand:
    def __init__(self, seed):
        self.g = torch.Generator(device="cuda").manual_seed(seed)

    def f16(self, n, scale=1.0, shift=0.0):
        return (torch.randn(n, generator=self.g, device="cuda") * scale + shift).half()

    def f32(self, n, scale=1.0):
        return torch.randn(n, generator=self.g, device="cuda") * scale

    def u8(self, n):
        return torch.randint(0, 256, (n,), generator=self.g, device="cuda", dtype=torch.uint8)


def _extent(sizes, strides, last):
    return sum((s - 1) * st for s, st in zip(sizes, strides)) + last


def _ulp16(ref):
    e = torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e - 10)


def _chunks(B, per_sample, samples=None):
    """sample index lists of at most CHUNK_ELEMS / per_sample samples each (at least one)"""
    idx = list(range(B)) if samples is None else sorted(set(samples))
    step = max(1, CHUNK_ELEMS // max(1, per_sample))
    return [idx[i:i + step] for i in range(0, len(idx), step)]


def _sentinel_buffer(n, view_fn, fill=float("nan"), dtype=torch.float16, sent=SENT):
    """a flat buffer of n elements at `sent`, with the elements of view_fn(buffer) at `fill`; returns (buffer, outside
    mask)"""
    buf = torch.full((n,), sent, dtype=dtype, device="cuda")
    inside = torch.zeros(n, dtype=torch.bool, device="cuda")
    view_fn(inside).fill_(True)
    view_fn(buf).fill_(fill)
    return buf, ~inside


def _outside_ok(buf, outside):
    return bool((buf[outside] == SENT).all())


# ----------------------------------------------------------------------------------------------------------------------
# GEMM
# ----------------------------------------------------------------------------------------------------------------------
def _gemm_geometry(f):
    conv = f["conv"]
    ntaps = {0: 1, 1: 9, 2: 9, 3: 4}[conv]
    Cp = (f["C"] + 63) // 64 * 64
    Wd, Hd = (f["W"] // 2, f["H"] // 2) if conv == 2 else (f["W"], f["H"])
    os_ = 2 if conv == 3 else 1
    OW, OH = Wd * os_, Hd * os_
    ncols = f["N"] // 2 if f["mode"] == 1 else (f["vt_col0"] if f["mode"] == 2 else f["N"])
    if f["o_sW"] or f["o_sH"] or f["o_sB"]:
        osW, osH, osB = f["o_sW"], f["o_sH"], f["o_sB"]
    else:
        osW, osH, osB = f["ldc"], OW * f["ldc"], OH * OW * f["ldc"]
    ldr = f["ldr"] or f["ldc"]
    res = (ldr, OW * ldr, OH * OW * ldr)
    return ntaps, Cp, Wd, Hd, os_, OW, OH, ncols, (osW, osH, osB), res


def _tap_inputs(f, x):
    """[(tap, shifted float64 input [nb, Hd, Wd, C])] of a conv record, zero padded"""
    conv = f["conv"]
    if conv == 0:
        return [(0, x)]
    H, W = x.shape[1], x.shape[2]
    xp = Fn.pad(x, (0, 0, 1, 1, 1, 1))
    out = []
    if conv in (1, 2):
        for t in range(9):
            ky, kx = t // 3, t % 3
            if conv == 1:
                out.append((t, xp[:, ky:ky + H, kx:kx + W]))
            else:
                out.append((t, xp[:, ky:ky + H:2, kx:kx + W:2]))
    else:
        for t in range(4):
            a, b = t >> 1, t & 1
            y0, x0 = a + f["up_py"], b + f["up_px"]
            out.append((t, xp[:, y0:y0 + H, x0:x0 + W]))
    return out


def _gelu(g):
    return 0.5 * g * (1 + torch.erf(g / math.sqrt(2)))


def replay_gemm(f, rnd, samples=None):
    """run the GEMM of record `f` on random data; returns the worst (err - bound) over the checked elements (<= 0)"""
    n = _n()
    assert not f["in_alias"]
    B, H, W, Cc, N = f["B"], f["H"], f["W"], f["C"], f["N"]
    ntaps, Cp, Wd, Hd, os_, OW, OH, ncols, (osW, osH, osB), (rsW, rsH, rsB) = _gemm_geometry(f)
    a_sizes, a_strides = (B, H, W, Cc), (f["sB"], f["sH"], f["sW"], 1)
    abuf = rnd.f16(_extent(a_sizes, a_strides, 1))
    A = abuf.as_strided(a_sizes, a_strides)
    if f["b_batched"]:
        Kb, ldb = f["Kb"], f["ldb"]
        w_sizes, w_strides = (B, H, N, Kb), (f["sBb"], f["sBh"], ldb, 1)
        wbuf = rnd.f16(_extent(w_sizes, w_strides, 1))
        K = Kb
    else:
        ldb = f["ldb"] or ntaps * Cp
        assert (f["Kb"] or ntaps * Cp) == ntaps * Cp
        wbuf = rnd.f16(N * ldb, scale=(ntaps * Cc) ** -0.5)
        wv = wbuf.view(N, ldb)[:, :ntaps * Cp].view(N, ntaps, Cp)
        wv[..., Cc:] = 0  # K padding of the packed layout
        K = ntaps * Cc
    bias = rnd.f32(N, 0.5) if f["bias"] else None
    rowvec = rnd.f32(N if f["rowvec_ld"] == 0 else B * f["rowvec_ld"], 0.5) if f["rowvec"] else None
    o_sizes, o_strides = (B, Hd, Wd, ncols), (osB, osH * os_, osW * os_, 1)
    o_off = f["up_py"] * osH + f["up_px"] * osW
    o_len = _extent((B, OH, OW, ncols), (osB, osH, osW, 1), 1)

    def oview(t):
        return t.as_strided(o_sizes, o_strides, o_off)
    if f["res_alias"]:
        obuf, outside = _sentinel_buffer(o_len, oview, fill=0.0)
        oview(obuf).copy_(rnd.f16(B * Hd * Wd * ncols).view(o_sizes))
        resid = oview(obuf).clone()
        rbuf = obuf
    else:
        obuf, outside = _sentinel_buffer(o_len, oview)
        rbuf = resid = None
        if f["resid"]:
            r_sizes, r_strides = (B, Hd, Wd, ncols), (rsB, rsH * os_, rsW * os_, 1)
            rbuf = rnd.f16(_extent((B, OH, OW, ncols), (rsB, rsH, rsW, 1), 1) + o_off)
            resid = rbuf.as_strided(r_sizes, r_strides, f["up_py"] * rsH + f["up_px"] * rsW)
    vt = None
    if f["mode"] == 2:
        assert f["H"] == 1 and f["W"] == f["vt_ntok"] and f["vt_ld"] >= f["vt_ntok"]
        vt = torch.full((B, f["vt_heads"], f["vt_d"], f["vt_ld"]), float("nan"), dtype=torch.float16, device="cuda")
    d = gemm_desc(f, A=abuf.data_ptr(), Wt=wbuf.data_ptr(), out=obuf.data_ptr(),
                  bias=bias.data_ptr() if bias is not None else None,
                  rowvec=rowvec.data_ptr() if rowvec is not None else None,
                  resid=rbuf.data_ptr() if rbuf is not None else None, vt=vt.data_ptr() if vt is not None else None)
    assert plan_of(d) == tuple(f[k] for k in PLAN_FIELDS), f  # the engine's launch, exactly
    n.gemm(d)
    torch.cuda.synchronize()
    assert _outside_ok(obuf, outside), "GEMM wrote outside its output view"
    out = oview(obuf)
    gamma = (K / 16 + 1) * 4 * 2.0 ** -24
    worst = -1.0
    u = 2.0 ** -24
    # chunks over samples; single-sample token lattices (B = 1, H = 1: Linear layers) chunk over rows instead
    rows_mode = B == 1 and H == 1 and not f["b_batched"]
    per = (W if not rows_mode else 1) * H * max(Cc, N) * (6 if f["conv"] else 4)
    groups = _chunks(W, per) if rows_mode else _chunks(B, per, samples)
    for grp in groups:
        sel = (slice(None), slice(None), grp) if rows_mode else (grp,)
        x = A[:, :, grp[0]:grp[-1] + 1].double() if rows_mode else A[grp].double()
        if f["b_batched"]:
            Wb = wbuf.as_strided(w_sizes, w_strides)[grp].double()
            acc = x[..., :K] @ Wb.transpose(-1, -2)
            mag = x[..., :K].abs() @ Wb.abs().transpose(-1, -2)
        else:
            wd = wv[..., :Cc].double()
            acc = mag = 0
            for t, xs in _tap_inputs(f, x):
                acc = acc + xs @ wd[:, t].T
                mag = mag + xs.abs() @ wd[:, t].abs().T
        alpha = f["alpha"]
        z = acc * alpha
        ez = gamma * abs(alpha) * mag + 4 * u * z.abs()
        if bias is not None:
            z = z + bias.double()
            ez = ez + 4 * u * bias.double().abs()
        if rowvec is not None:
            assert f["rowvec_ld"] == 0 or not rows_mode
            rv = rowvec.double() if f["rowvec_ld"] == 0 else rowvec.view(B, -1)[grp, :N].double()[:, None, None, :]
            z = z + rv
            ez = ez + 4 * u * rv.abs()
        if f["mode"] == 1:
            zz = z.unflatten(-1, (-1, 2, 32))
            ee = ez.unflatten(-1, (-1, 2, 32))
            a, g = zz[..., 0, :], zz[..., 1, :]
            ea, eg = ee[..., 0, :], ee[..., 1, :]
            gl = _gelu(g)
            ref = (a * gl).flatten(-2)
            bound = (gl.abs() * ea + a.abs() * 1.13 * eg + a.abs() * 0.5 * g.abs() * 2.5e-7).flatten(-2)
            bound = bound + 2.0 ** -21 * ref.abs()
        else:
            ref, bound = z, ez
            if f["act"] == 1:
                ref = Fn.silu(z)
                bound = 1.1 * ez + (4 + 1.2 * z.abs()) * 2.0 ** -22 * ref.abs()
            else:
                assert f["act"] == 0
        vt_ref = None
        if f["mode"] == 2:
            c0 = f["vt_col0"]
            vt_ref, vt_bound = ref[..., c0:], bound[..., c0:]
            ref, bound = ref[..., :c0], bound[..., :c0]
        if resid is not None:
            r = resid[:, :, grp[0]:grp[-1] + 1].double() if rows_mode else resid[grp].double()
            ref = ref + r
            bound = bound + 2 * u * r.abs()
        got = out[:, :, grp[0]:grp[-1] + 1] if rows_mode else out[grp]
        assert bool(torch.isfinite(got).all()), "non-finite GEMM output"
        err = (got.double() - ref).abs() - (bound + 2.0 ** -11 * ref.abs() + 2.0 ** -25)
        worst = max(worst, float(err.max()))
        if vt_ref is not None:
            nb, hv, dv = len(grp), f["vt_heads"], f["vt_d"]
            vr = vt_ref.reshape(nb, W, hv, dv).permute(0, 2, 3, 1)
            vb = vt_bound.reshape(nb, W, hv, dv).permute(0, 2, 3, 1)
            gv = vt[grp][..., :W].double()
            assert bool(torch.isfinite(gv).all())
            worst = max(worst, float(((gv - vr).abs() - (vb + 2.0 ** -11 * vr.abs() + 2.0 ** -25)).max()))
        del x, acc, mag, z, ez, ref, bound, err
    return worst


# ----------------------------------------------------------------------------------------------------------------------
# the other kinds
# ----------------------------------------------------------------------------------------------------------------------
def replay_groupnorm(f, rnd, samples=None):
    B, P, Cc, G, ldx, ldy = f["B"], f["P"], f["C"], f["G"], f["ldx"], f["ldy"]
    x = rnd.f16(B * P * ldx, 1.5, 0.3).view(B, P, ldx)
    gamma = rnd.f32(Cc, 0.2) + 1.0
    beta = rnd.f32(Cc, 0.1)
    ybuf, outside = _sentinel_buffer(B * P * ldy, lambda t: t.view(B, P, ldy)[..., :Cc])
    y = ybuf.view(B, P, ldy)[..., :Cc]
    _n().groupnorm(x[..., :Cc], B, P, Cc, G, gamma, beta, f["eps"], f["silu"], y)
    torch.cuda.synchronize()
    assert _outside_ok(ybuf, outside)
    err = refmax = 0.0
    for grp in _chunks(B, P * Cc * 4, samples):
        xd = x[grp][..., :Cc].double()
        ref = Fn.group_norm(xd.transpose(1, 2), G, gamma.double(), beta.double(), f["eps"]).transpose(1, 2)
        if f["silu"]:
            ref = Fn.silu(ref)
        got = y[grp].double()
        assert bool(torch.isfinite(got).all())
        err = max(err, float((got - ref).abs().max()))
        refmax = max(refmax, float(ref.abs().max()))
    return err - (2 ** -9 * refmax + 1e-3)


def replay_layernorm(f, rnd):
    rows, Cc, ldx, ldy = f["rows"], f["C"], f["ldx"], f["ldy"]
    x = rnd.f16(rows * ldx, 2.0, -0.5).view(rows, ldx)
    gamma = rnd.f32(Cc, 0.2) + 1.0
    beta = rnd.f32(Cc, 0.1)
    ybuf, outside = _sentinel_buffer(rows * ldy, lambda t: t.view(rows, ldy)[:, :Cc])
    y = ybuf.view(rows, ldy)[:, :Cc]
    _n().layernorm(x[:, :Cc], rows, Cc, gamma, beta, f["eps"], y)
    torch.cuda.synchronize()
    assert _outside_ok(ybuf, outside)
    err = refmax = 0.0
    step = max(1, CHUNK_ELEMS // (4 * Cc))
    for r0 in range(0, rows, step):
        ref = Fn.layer_norm(x[r0:r0 + step, :Cc].double(), (Cc,), gamma.double(), beta.double(), f["eps"])
        got = y[r0:r0 + step].double()
        assert bool(torch.isfinite(got).all())
        err = max(err, float((got - ref).abs().max()))
        refmax = max(refmax, float(ref.abs().max()))
    return err - (2 ** -9 * refmax + 1e-3)


def replay_attention(f, rnd):
    B, Nq, Nk, h, d = f["B"], f["Nq"], f["Nk"], f["heads"], f["d"]
    q = rnd.f16(B * Nq * f["q_ld"]).view(B, Nq, f["q_ld"])
    k = rnd.f16(B * Nk * f["k_ld"]).view(B, Nk, f["k_ld"])
    vt = rnd.f16(B * h * d * f["vt_ld"]).view(B, h, d, f["vt_ld"])
    ol = f["out_ld"]
    obuf, outside = _sentinel_buffer(B * Nq * ol, lambda t: t.view(B, Nq, ol)[..., :h * d])
    _call("sdw_attention", _p(q), I64(f["q_ld"]), _p(k), I64(f["k_ld"]), _p(vt), I64(f["vt_ld"]), B, Nq, Nk, h, d,
          _p(obuf), I64(ol))
    assert _outside_ok(obuf, outside)
    out = obuf.view(B, Nq, ol)[..., :h * d]
    err = refmax = 0.0
    for grp in _chunks(B, h * Nq * Nk * 3):
        qq = q[grp][..., :h * d].double().unflatten(-1, (h, d)).transpose(1, 2)
        kk = k[grp][..., :h * d].double().unflatten(-1, (h, d)).transpose(1, 2)
        vv = vt[grp][..., :Nk].double().transpose(-1, -2)
        ref = (torch.softmax(qq @ kk.transpose(-1, -2) / math.sqrt(d), -1) @ vv).transpose(1, 2).flatten(-2)
        got = out[grp].double()
        assert bool(torch.isfinite(got).all())
        err = max(err, float((got - ref).abs().max()))
        refmax = max(refmax, float(ref.abs().max()))
    return err - (2.0 ** -8 * refmax + 1e-3)


def replay_softmax(f, rnd):
    ld, rows, nn = f["ld"], f["rows"], f["n"]
    buf = torch.full((rows, ld), float("nan"), dtype=torch.float16, device="cuda")
    buf[:, :nn] = rnd.f16(rows * nn, 3.0).view(rows, nn)
    x = buf[:, :nn].clone()
    pad = buf[:, nn:].clone()
    _call("sdw_softmax_rows", _p(buf), I64(ld), I64(rows), nn)
    assert torch.equal(buf[:, nn:].view(torch.int16), pad.view(torch.int16))
    worst = -1.0
    step = max(1, CHUNK_ELEMS // (3 * nn))
    for r0 in range(0, rows, step):
        ref = torch.softmax(x[r0:r0 + step].double(), -1)
        err = (buf[r0:r0 + step, :nn].double() - ref).abs() - (_ulp16(ref) + 2.0 ** -24)
        worst = max(worst, float(err.max()))
    return worst


def _conv3x3_64(x, w, bias):
    """float64 3x3 pad-1 conv of an NHWC fp16 view x with OIHW weights (tap by tap); returns (ref, |.| magnitude)"""
    xd = Fn.pad(x.double(), (0, 0, 1, 1, 1, 1))
    H, W = x.shape[1], x.shape[2]
    wd = w.double()
    ref = bias.double().clone() if bias is not None else 0
    mag = bias.double().abs() if bias is not None else 0
    for ky in range(3):
        for kx in range(3):
            xs = xd[:, ky:ky + H, kx:kx + W]
            ref = ref + xs @ wd[:, :, ky, kx].T
            mag = mag + xs.abs() @ wd[:, :, ky, kx].abs().T
    return ref, mag


def replay_conv_in(f, rnd):
    B, H, W, Ci, N, ldx, ldy = f["B"], f["H"], f["W"], f["Cin"], f["N"], f["ldx"], f["ldy"]
    x = rnd.f16(B * H * W * ldx).view(B, H, W, ldx)
    w = rnd.f16(N * Ci * 9, 0.3).view(N, Ci, 3, 3)
    bias = rnd.f32(N)
    ybuf, outside = _sentinel_buffer(B * H * W * ldy, lambda t: t.view(B, H, W, ldy)[..., :N])
    _call("sdw_conv_in_small", _p(x), I64(ldx), B, H, W, Ci, _p(w), _p(bias), N, _p(ybuf), I64(ldy))
    assert _outside_ok(ybuf, outside)
    y = ybuf.view(B, H, W, ldy)[..., :N]
    worst = -1.0
    for grp in _chunks(B, H * W * N * 4):
        ref, mag = _conv3x3_64(x[grp][..., :Ci], w, bias)
        got = y[grp].double()
        assert bool(torch.isfinite(got).all())
        worst = max(worst, float(((got - ref).abs() - (_ulp16(ref) + 2.0 ** -20 * mag)).max()))
    return worst


def _u8_of(v):
    return torch.round(torch.clamp(v / 2 + 0.5, 0, 1) * 255)


def replay_conv_out(f, rnd, samples=None):
    B, H, W, Cc, no, ldx = f["B"], f["H"], f["W"], f["C"], f["nout"], f["ldx"]
    x = rnd.f16(B * H * W * ldx).view(B, H, W, ldx)
    w = rnd.f16(no * Cc * 9, 0.6 / math.sqrt(9 * Cc)).view(no, Cc, 3, 3)
    bias = rnd.f32(no, 0.2)
    P = B * H * W
    f32 = torch.full((P * no + 64,), float("nan"), device="cuda") if f["f32"] else None
    u8 = torch.full((P * no + 64,), 0xA5, dtype=torch.uint8, device="cuda") if f["u8"] else None
    if f32 is not None:
        f32[P * no:] = SENT
    _call("sdw_conv_out_small", _p(x), I64(ldx), B, H, W, Cc, _p(w), _p(bias), no, _p(f32), _p(u8))
    if f32 is not None:
        assert bool((f32[P * no:] == SENT).all())
        f32 = f32[:P * no].view(B, H, W, no)
    if u8 is not None:
        assert bool((u8[P * no:] == 0xA5).all())
        u8 = u8[:P * no].view(B, H, W, no)
    worst = -1.0
    for grp in _chunks(B, H * W * Cc * 3, samples):
        ref, mag = _conv3x3_64(x[grp][..., :Cc], w, bias)
        if f32 is not None:
            worst = max(worst, float(((f32[grp].double() - ref).abs() - (1e-5 * mag + 1e-6)).max()))
        if u8 is not None:
            assert int((u8[grp].double() - _u8_of(ref)).abs().max()) <= 1
            if f32 is not None:
                assert torch.equal(u8[grp].float(), _u8_of(f32[grp]))
    return worst


def replay_vae_in(f, rnd):
    Fr, Cc, H, W = f["F"], f["C"], f["H"], f["W"]
    x = rnd.f32(Fr * Cc * H * W, 0.9).view(Fr, Cc, H, W)
    w = rnd.f16(Cc * Cc, 0.5).view(Cc, Cc)
    bias = rnd.f32(Cc)
    P = Fr * H * W
    z = torch.full((P * Cc + 40,), float("nan"), dtype=torch.float16, device="cuda")
    z[P * Cc:] = SENT
    _call("sdw_vae_in", _p(x), C.c_float(f["inv_scale"]), _p(w), _p(bias), Fr, Cc, H, W, _p(z))
    assert bool((z[P * Cc:] == SENT).all())
    xs = x.double().permute(0, 2, 3, 1) * C.c_float(f["inv_scale"]).value
    ref = xs @ w.double().T + bias.double()
    mag = xs.abs() @ w.double().abs().T + bias.double().abs()
    return float(((z[:P * Cc].view(Fr, H, W, Cc).double() - ref).abs() - (_ulp16(ref) + 2.0 ** -20 * mag)).max())


def replay_wrap_pad(f, rnd, samples=None):
    B, H, W, pb, pad, ld = f["B"], f["H"], f["W"], f["pix_bytes"], f["pad"], f["ld_bytes"]
    x = rnd.u8(B * H * W * ld).view(B, H, W, ld)
    Hp, Wp = H + 2 * pad, W + 2 * pad
    ny = B * Hp * Wp * pb
    y = torch.full((ny + 32,), 0x5A, dtype=torch.uint8, device="cuda")
    _call("sdw_wrap_pad", _p(x), I64(ld), B, H, W, pb, pad, _p(y))
    assert bool((y[ny:] == 0x5A).all())
    yv = y[:ny].view(B, Hp, Wp, pb)
    iy = torch.arange(-pad, H + pad, device="cuda") % H
    ix = torch.arange(-pad, W + pad, device="cuda") % W
    for grp in _chunks(B, Hp * Wp * pb // 4, samples):
        assert torch.equal(yv[grp], x[grp][:, iy][:, :, ix][..., :pb])
    return -1.0


def replay_crop(f, rnd, samples=None):
    B, H, W, pb, c, ldo = f["B"], f["H"], f["W"], f["pix_bytes"], f["crop"], f["ldo_bytes"]
    Hp, Wp = H + 2 * c, W + 2 * c
    yp = rnd.u8(B * Hp * Wp * pb).view(B, Hp, Wp, pb)
    resid = None
    if f["resid"]:
        assert pb % 2 == 0
        yp = rnd.f16(B * Hp * Wp * pb // 2).view(torch.uint8).view(B, Hp, Wp, pb)
        resid = rnd.f16(B * H * W * f["ldr"]).view(B, H, W, f["ldr"])
    ob, outside = _sentinel_buffer(B * H * W * ldo, lambda t: t.view(B, H, W, ldo)[..., :pb], fill=0x33,
                                   dtype=torch.uint8, sent=0x5A)
    _call("sdw_crop_interior", _p(yp), B, H, W, pb, c, _p(resid), I64(f["ldr"]), _p(ob), I64(ldo))
    assert bool((ob[outside] == 0x5A).all())
    out = ob.view(B, H, W, ldo)[..., :pb]
    for grp in _chunks(B, H * W * pb // 2, samples):
        inner = yp[grp][:, c:c + H, c:c + W]
        if resid is None:
            assert torch.equal(out[grp], inner)
        else:
            ref = (inner.contiguous().view(torch.float16).float() + resid[grp][..., :pb // 2].float()).half()
            assert torch.equal(out[grp].contiguous().view(torch.int16), ref.view(torch.int16))
    return -1.0


REPLAY = {"gemm": replay_gemm, "groupnorm": replay_groupnorm, "layernorm": replay_layernorm,
          "attention": replay_attention, "softmax_rows": replay_softmax, "conv_in_small": replay_conv_in,
          "conv_out_small": replay_conv_out, "vae_in": replay_vae_in, "wrap_pad": replay_wrap_pad, "crop": replay_crop}


def _replay_all(recs, kinds, seed):
    bad = []
    for i, (sec, kind, f) in enumerate(_distinct(recs, kinds)):
        worst = REPLAY[kind](f, Rand(seed + i))
        if worst > 0:
            bad.append((sec, kind, worst, f))
        torch.cuda.empty_cache()
    return bad


def test_every_gemm_of_the_30_frame_engine(ops30):
    recs, _ = ops30
    gemms = _distinct(recs, {"gemm"})
    plans = {tuple(f[k] for k in ("conv", "mode", "b_batched") + PLAN_FIELDS) for _, _, f in gemms}
    print(f"\n{len(gemms)} distinct GEMM records, {len(plans)} (conv, mode, batched, plan) combinations: {sorted(plans)}")
    assert not _replay_all(recs, {"gemm"}, 1000)


def test_every_other_op_of_the_30_frame_engine(ops30):
    recs, trecs = ops30
    kinds = {"groupnorm", "layernorm", "attention", "softmax_rows", "conv_in_small", "conv_out_small", "vae_in"}
    assert not _replay_all(recs, kinds, 2000)
    # circular padding and cropping of tiled mode, up to the 4 GB activations of the 512 x 512 level
    assert not _replay_all(trecs, {"wrap_pad", "crop"}, 3000)


def _operand_bytes(kind, f):
    """the largest byte extent among a record's operands"""
    if kind == "gemm":
        ntaps, Cp, Wd, Hd, os_, OW, OH, ncols, (osW, osH, osB), _ = _gemm_geometry(f)
        a = _extent((f["B"], f["H"], f["W"], f["C"]), (f["sB"], f["sH"], f["sW"], 1), 1)
        o = _extent((f["B"], OH, OW, ncols), (osB, osH, osW, 1), 1)
        return 2 * max(a, o)
    if kind == "groupnorm":
        return 2 * f["B"] * f["P"] * max(f["ldx"], f["ldy"])
    if kind == "conv_out_small":
        return 2 * f["B"] * f["H"] * f["W"] * f["ldx"]
    if kind == "wrap_pad":
        return f["B"] * (f["H"] + 2 * f["pad"]) * (f["W"] + 2 * f["pad"]) * max(f["pix_bytes"], f["ld_bytes"])
    if kind == "crop":
        return f["B"] * (f["H"] + 2 * f["crop"]) * (f["W"] + 2 * f["crop"]) * f["pix_bytes"]
    return 0


def test_vae_ops_past_2_to_the_31():
    """SD-1.4 at 512 x 512 with 33 frames: the VAE's 512 x 512 x 256 activations hold 2.2e9 fp16 elements (4.4 GB).  Every
    op with an operand past 2^31 bytes (so past any 32-bit byte or element offset) is replayed at that batch and checked
    on the first and the last two samples, where a wrapped offset would land.  Tiled mode adds the circular padding and
    cropping around those tensors."""
    recs, _, _ = plan_only_ops(33)
    trecs, _, _ = plan_only_ops(33, tiled=True)
    big = [r for r in recs if r[0] == "vae" and _operand_bytes(r[2], r[3]) > 2 ** 31]
    tbig = [r for r in trecs if r[0] == "vae" and r[2] in ("wrap_pad", "crop") and _operand_bytes(r[2], r[3]) > 2 ** 31]
    kinds = {k for _, _, k, _ in big}
    assert {"gemm", "groupnorm", "conv_out_small"} <= kinds and tbig
    assert any(f["conv"] == 3 for _, _, k, f in big if k == "gemm") and any(f["conv"] == 1 for _, _, k, f in big if k == "gemm")
    assert any(f["B"] * f["P"] * f["C"] > 2 ** 31 for _, _, k, f in big if k == "groupnorm")
    samples = [0, 31, 32]
    bad = []
    for i, (sec, kind, f) in enumerate(_distinct(big + tbig)):
        worst = REPLAY[kind](f, Rand(4000 + i), samples=samples)
        if worst > 0:
            bad.append((kind, worst, f))
        torch.cuda.empty_cache()
    print(f"\npeak device memory {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")
    assert not bad
