"""GPU checks of the pipelined fused attention kernel (sdw_attention) that the parity suite in test_attn_gpu.py does not
cover: the prologue / drain of the software pipeline at BKV = 64 (d = 80: one, two and three KV tiles, with one or both
consumer warpgroups holding rows beyond Nq), and bit reproducibility of the ping-pong between the two consumer
warpgroups at the engine's 64x64 self-attention shape.  Reference: float64 on the same fp16 inputs, tolerance
2^-8 * max|ref| + 1e-3 as in test_attn_gpu.py."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref64(q, k, v, heads, d):
    B, Nq, Nk = q.shape[0], q.shape[1], k.shape[1]
    qd = q[..., :heads * d].double().reshape(B, Nq, heads, d).transpose(1, 2)
    kd = k[..., :heads * d].double().reshape(B, Nk, heads, d).transpose(1, 2)
    vd = v.double().reshape(B, Nk, heads, d).transpose(1, 2)
    return (torch.softmax(qd @ kd.transpose(-1, -2) * d ** -0.5, -1) @ vd).transpose(1, 2).reshape(B, Nq, heads * d)


def _vt(v, heads, d, vt_ld):
    """V^T [B][heads][d][vt_ld] with NaN in the pad columns, which must never be read"""
    B, Nk = v.shape[0], v.shape[1]
    vt = torch.full((B, heads, d, vt_ld), float("nan"), dtype=torch.float16, device="cuda")
    vt[..., :Nk] = v.reshape(B, Nk, heads, d).permute(0, 2, 3, 1)
    return vt


def _attend(q, k, vt, B, Nq, Nk, heads, d, out):
    from stable_diffusion_videos_b200 import _native as n

    n.check(n.lib().sdw_attention(n.ptr(q), C.c_int64(q.stride(1)), n.ptr(k), C.c_int64(k.stride(1)), n.ptr(vt),
                                  C.c_int64(vt.shape[-1]), B, Nq, Nk, heads, d, n.ptr(out), C.c_int64(out.stride(1)),
                                  n.stream_ptr()))


@pytest.mark.parametrize("Nq", [64, 65, 128])
@pytest.mark.parametrize("Nk", [40, 64, 100, 128, 150, 192])
def test_attention_d80_pipeline_prologue_and_drain(Nk, Nq):
    """d = 80 runs 64-key tiles: Nk = 40 / 64 is one tile (prologue straight into the drain), 100 / 128 two, 150 / 192
    three, ragged or full.  Nq = 64 leaves the second consumer warpgroup with no valid row, 65 with one.  The keys
    are ramped so the running max rises from tile to tile and every rescale of O is exercised."""
    B, heads, d = 2, 3, 80
    Cc = heads * d
    g = torch.Generator().manual_seed(Nq * 1000 + Nk)
    q = torch.randn(B, Nq, Cc, generator=g).half().cuda()
    k = (torch.randn(B, Nk, Cc, generator=g) * torch.linspace(0.2, 3.0, Nk)[None, :, None]).half().cuda()
    v = torch.randn(B, Nk, Cc, generator=g).half().cuda()
    vt = _vt(v, heads, d, (Nk + 7) // 8 * 8)
    out = torch.full((B, Nq, Cc), float("nan"), dtype=torch.float16, device="cuda")
    _attend(q, k, vt, B, Nq, Nk, heads, d, out)
    torch.cuda.synchronize()
    ref = _ref64(q, k, v, heads, d)
    assert bool(torch.isfinite(out).all())
    err = float((out.double() - ref).abs().max())
    assert err <= 2.0 ** -8 * float(ref.abs().max()) + 1e-3, err


def test_attention_engine_shape_bit_reproducible():
    """the 64x64-level self-attention as the engine runs it (Q|K in one buffer, 8 heads x 40, 4096 tokens), launched
    twice on the same inputs with other work in between: the output bytes must be identical, so the timing of the
    two consumer warpgroups' ping-pong never reaches the arithmetic"""
    B, heads, d, N = 4, 8, 40, 4096
    Cc = heads * d
    g = torch.Generator().manual_seed(11)
    qk = torch.randn(B, N, 2 * Cc, generator=g).half().cuda()
    v = torch.randn(B, N, Cc, generator=g).half().cuda()
    vt = _vt(v, heads, d, N)
    q, k = qk[..., :Cc], qk[..., Cc:]
    outs = []
    for i in range(2):
        out = torch.full((B, N, Cc), float("nan"), dtype=torch.float16, device="cuda")
        _attend(q, k, vt, B, N, N, heads, d, out)
        if i == 0:
            # a different attention in between, so the second launch starts from other cache and scheduling state
            other = torch.empty(2, N, Cc, dtype=torch.float16, device="cuda")
            _attend(qk[:2, :, Cc:], qk[:2, :, :Cc], vt[:2], 2, N, N, heads, d, other)
        outs.append(out)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(outs[0]).all())
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16))
    ref = _ref64(q[:1], k[:1], v[:1], heads, d)
    err = float((outs[0][:1].double() - ref).abs().max())
    assert err <= 2.0 ** -8 * float(ref.abs().max()) + 1e-3, err
