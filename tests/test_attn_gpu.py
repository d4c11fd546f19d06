"""GPU parity of the fused wgmma attention kernel (sdw_attention) against a float64 reference on the same fp16 inputs.
Tolerance: P is rounded to fp16 before the PV product and the output is rounded to fp16:
|err| <= 2^-8 * max|ref| + 1e-3 (calibrated in DESIGN.md §Parity).

Besides separate Q / K buffers of pitch heads * d, the cases cover the layouts the engine passes: self-attention with Q
and K as the two halves of one [B, N, 2C] buffer, cross-attention with K of pitch C and 77 tokens, V^T rows whose pad
columns hold NaN, and outputs written into a channel slice of a wider buffer."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

SENT = -7.25


def _ceil8(n):
    return (n + 7) // 8 * 8


def _ref64(q, k, v, heads, d):
    """softmax(Q K^T d^-1/2) V per (batch, head) in float64; q [B, Nq, >= heads*d] etc., head h at columns h*d."""
    B, Nq, Nk = q.shape[0], q.shape[1], k.shape[1]
    qd = q[..., :heads * d].double().reshape(B, Nq, heads, d).transpose(1, 2)
    kd = k[..., :heads * d].double().reshape(B, Nk, heads, d).transpose(1, 2)
    vd = v.double().reshape(B, Nk, heads, d).transpose(1, 2)
    return (torch.softmax(qd @ kd.transpose(-1, -2) * d ** -0.5, -1) @ vd).transpose(1, 2).reshape(B, Nq, heads * d)


def _vt(v, heads, d, vt_ld, pad=float("nan")):
    """V^T [B][heads][d][vt_ld] as the QKV GEMM epilogue writes it; columns >= Nk hold `pad`."""
    B, Nk = v.shape[0], v.shape[1]
    vt = torch.full((B, heads, d, vt_ld), pad, dtype=torch.float16, device="cuda")
    vt[..., :Nk] = v.reshape(B, Nk, heads, d).permute(0, 2, 3, 1)
    return vt


def _attend(q, k, vt, B, Nq, Nk, heads, d, out):
    """q, k, out: [B, N, pitch] views (the pitch is stride(1)); vt: [B, heads, d, vt_ld]."""
    from stable_diffusion_videos_b200 import _native as n

    n.check(n.lib().sdw_attention(n.ptr(q), C.c_int64(q.stride(1)), n.ptr(k), C.c_int64(k.stride(1)), n.ptr(vt),
                                  C.c_int64(vt.shape[-1]), B, Nq, Nk, heads, d, n.ptr(out), C.c_int64(out.stride(1)),
                                  n.stream_ptr()))
    torch.cuda.synchronize()


def _check(out, ref, rel=2.0 ** -8, absol=1e-3):
    assert bool(torch.isfinite(out).all())
    err = float((out.double() - ref).abs().max())
    assert err <= rel * float(ref.abs().max()) + absol, (err, float(ref.abs().max()))


def _run(B, heads, Nq, Nk, d, seed=0, scale=1.0, k_ramp=None):
    g = torch.Generator().manual_seed(seed)
    Cc = heads * d
    q = (torch.randn(B, Nq, Cc, generator=g) * scale).half().cuda()
    k = torch.randn(B, Nk, Cc, generator=g) * scale
    if k_ramp is not None:
        k = k * torch.linspace(k_ramp[0], k_ramp[1], Nk)[None, :, None]
    k = k.half().cuda()
    v = torch.randn(B, Nk, Cc, generator=g).half().cuda()
    vt = _vt(v, heads, d, _ceil8(Nk))
    out = torch.full((B, Nq, Cc), float("nan"), dtype=torch.float16, device="cuda")
    _attend(q, k, vt, B, Nq, Nk, heads, d, out)
    return out, _ref64(q, k, v, heads, d)


@pytest.mark.parametrize("B,heads,Nq,Nk,d", [
    (2, 8, 256, 256, 40),     # SD-1.4 64x64-level head dim (padded to 48 in the MMA)
    (1, 8, 4096, 4096, 40),   # full 64x64 self-attention: 32 KV tiles, online softmax
    (2, 8, 1024, 77, 40),     # cross attention: one ragged KV tile
    (2, 8, 1024, 1024, 80),
    (2, 8, 256, 256, 160),    # BKV = 64 variant
    (2, 8, 64, 64, 160),      # 8x8 level: half-empty query tile
    (2, 4, 64, 64, 8),
    (2, 4, 64, 77, 16),
    (1, 5, 300, 300, 64),     # SD-2.1 head dim, ragged both ways
    (3, 2, 129, 200, 32),
])
def test_flash_attention_matches_sdpa(B, heads, Nq, Nk, d):
    _check(*_run(B, heads, Nq, Nk, d))


def test_flash_attention_peaky_scores():
    """large logits: running-max rescale path must engage and stay finite."""
    out, ref = _run(1, 4, 512, 512, 40, seed=3, scale=4.0)
    _check(out, ref, 2.0 ** -7, 2e-3)


@pytest.mark.parametrize("B,heads,Nq,Nk,d", [
    (1, 4, 300, 700, 40),     # ragged last query tile (44 of 128 rows) and ragged last KV tile
    (1, 2, 128, 1000, 32),    # exactly one query tile, eight KV tiles (the last one ragged)
    (2, 3, 576, 576, 64),     # SD-2.1 at 24x24: 4.5 query tiles and 4.5 KV tiles
    (1, 2, 2048, 2048, 16),
    (3, 8, 1024, 1024, 40),   # 192 CTAs: more than one wave on the GPU
])
def test_flash_attention_rising_max_and_ragged(B, heads, Nq, Nk, d):
    """keys scaled so that the row max keeps rising along the KV loop (the running-max rescale engages on every tile)."""
    _check(*_run(B, heads, Nq, Nk, d, seed=5, k_ramp=(0.2, 3.0)))


@pytest.mark.parametrize("d", list(range(8, 161, 8)))
def test_flash_attention_every_head_dim(d):
    """every head dim the planner accepts: all six variants and every d between their boundaries (partly or entirely
    empty 16-column k-steps and 64-column chunks, V^T boxes with rows beyond d)"""
    _check(*_run(2, 3, 130, 200, d, seed=d))


# (heads, d, self-attention tokens): SD-1.4 levels (8 heads, d = 40 / 80 / 160), SD-2.1 (d = 64 with 5 / 10 / 20
# heads) and the mid-size test VAE (one head, d = 128)
ENGINE_SHAPES = [(8, 40, 1024), (8, 80, 256), (8, 160, 64), (5, 64, 1024), (10, 64, 256), (20, 64, 64), (1, 128, 256)]


@pytest.mark.parametrize("heads,d,N", ENGINE_SHAPES)
def test_flash_attention_engine_self_layout(heads, d, N):
    """self-attention as the transformer block runs it: Q|K in one [B, N, 2C] buffer (q_ld = k_ld = 2C, k = q + C),
    V^T of pitch ceil8(N) with NaN in the pad columns, which must never be read"""
    B, Cc = 2, heads * d
    g = torch.Generator().manual_seed(heads * 1000 + d)
    qk = torch.randn(B, N, 2 * Cc, generator=g).half().cuda()
    v = torch.randn(B, N, Cc, generator=g).half().cuda()
    vt = _vt(v, heads, d, _ceil8(N))
    out = torch.full((B, N, Cc), float("nan"), dtype=torch.float16, device="cuda")
    q, k = qk[..., :Cc], qk[..., Cc:]
    _attend(q, k, vt, B, N, N, heads, d, out)
    _check(out, _ref64(q, k, v, heads, d))


@pytest.mark.parametrize("heads,d,N", ENGINE_SHAPES)
def test_flash_attention_engine_cross_layout(heads, d, N):
    """cross-attention as the engine runs it: Q of pitch C, 77 context tokens with K of pitch C, V^T of pitch 80 whose
    three pad columns hold NaN"""
    B, Cc, T = 2, heads * d, 77
    g = torch.Generator().manual_seed(heads * 1000 + d + 1)
    q = torch.randn(B, N, Cc, generator=g).half().cuda()
    k = torch.randn(B, T, Cc, generator=g).half().cuda()
    v = torch.randn(B, T, Cc, generator=g).half().cuda()
    vt = _vt(v, heads, d, 80)
    out = torch.full((B, N, Cc), float("nan"), dtype=torch.float16, device="cuda")
    _attend(q, k, vt, B, N, T, heads, d, out)
    _check(out, _ref64(q, k, v, heads, d))


@pytest.mark.parametrize("d", [40, 160])
@pytest.mark.parametrize("c0,extra", [(8, 24), (3, 8)])
def test_flash_attention_output_pitch(d, c0, extra):
    """output into columns [c0, c0 + heads*d) of a wider buffer whose other columns must keep their sentinel; an odd
    pitch (c0 = 3: heads*d + 11 columns) takes the scalar-store path"""
    B, heads, Nq, Nk = 2, 3, 200, 150
    Cc = heads * d
    g = torch.Generator().manual_seed(d + c0)
    q = torch.randn(B, Nq, Cc, generator=g).half().cuda()
    k = torch.randn(B, Nk, Cc, generator=g).half().cuda()
    v = torch.randn(B, Nk, Cc, generator=g).half().cuda()
    vt = _vt(v, heads, d, _ceil8(Nk))
    ld = Cc + c0 + extra
    buf = torch.full((B, Nq, ld), SENT, dtype=torch.float16, device="cuda")
    out = buf[..., c0:c0 + Cc]
    out.fill_(float("nan"))
    _attend(q, k, vt, B, Nq, Nk, heads, d, out)
    assert bool((buf[..., :c0] == SENT).all()) and bool((buf[..., c0 + Cc:] == SENT).all())
    _check(out, _ref64(q, k, v, heads, d))


@pytest.mark.parametrize("d", [40, 160])  # BKV = 128 and 64
@pytest.mark.parametrize("Nq", [1, 127, 128, 129])
@pytest.mark.parametrize("Nk", [1, 63, 64, 65, 127, 128, 129])
def test_flash_attention_edge_lengths(Nk, Nq, d):
    _check(*_run(1, 2, Nq, Nk, d, seed=Nq * 1000 + Nk))


def test_flash_attention_fresh_process():
    """a fresh process (first launch of the kernels, no cached attributes) computes the same attention"""
    import os
    import subprocess
    import sys
    code = ("import torch, ctypes as C\n"
            "from stable_diffusion_videos_b200 import _native as n\n"
            "torch.manual_seed(0)\n"
            "for (B,h,Nq,Nk,d) in [(2,8,1024,1024,40),(1,2,256,700,64)]:\n"
            "    Cc=h*d; q=torch.randn(B,Nq,Cc,device='cuda').half(); k=torch.randn(B,Nk,Cc,device='cuda').half()\n"
            "    v=torch.randn(B,Nk,Cc,device='cuda').half(); ld=(Nk+7)//8*8\n"
            "    vt=torch.zeros(B,h,d,ld,device='cuda',dtype=torch.float16); vt[...,:Nk]=v.reshape(B,Nk,h,d).permute(0,2,3,1)\n"
            "    out=torch.empty(B,Nq,Cc,device='cuda',dtype=torch.float16)\n"
            "    n.check(n.lib().sdw_attention(n.ptr(q),C.c_int64(Cc),n.ptr(k),C.c_int64(Cc),n.ptr(vt),C.c_int64(ld),B,Nq,Nk,h,d,n.ptr(out),C.c_int64(Cc),n.stream_ptr()))\n"
            "    torch.cuda.synchronize()\n"
            "    qf=q.double().reshape(B,Nq,h,d).permute(0,2,1,3); kf=k.double().reshape(B,Nk,h,d).permute(0,2,1,3); vf=v.double().reshape(B,Nk,h,d).permute(0,2,1,3)\n"
            "    ref=(torch.softmax(qf@kf.transpose(-1,-2)*d**-0.5,-1)@vf).permute(0,2,1,3).reshape(B,Nq,Cc)\n"
            "    err=(out.double()-ref).abs().max().item(); assert err <= 2**-8*ref.abs().max().item()+1e-3, (err, B,h,Nq,Nk,d)\n"
            "print('ok')\n")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ)
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=root, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "ok" in r.stdout, (r.stdout[-500:], r.stderr[-2000:])
