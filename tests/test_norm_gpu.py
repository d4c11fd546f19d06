"""GroupNorm / LayerNorm kernels vs torch fp32 on the same fp16 inputs (reference layers: diffusers ResnetBlock2D /
Transformer2D norms inside `self.unet(...)`, stable_diffusion_pipeline.py:418; VAE decoder norms, :433)."""
import pytest
import torch
import torch.nn.functional as Fn

pytestmark = pytest.mark.gpu


def _native():
    from stable_diffusion_videos_b200 import _native as n
    return n


def _rand(*shape, seed=0, scale=1.0, shift=0.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale + shift).to(torch.float16).cuda()


@pytest.mark.parametrize("B,H,W,Cc,G,silu", [(4, 64, 64, 320, 32, 1), (2, 32, 32, 640, 32, 0), (3, 8, 8, 1280, 32, 1),
                                            (2, 16, 16, 2560, 32, 1), (1, 128, 128, 128, 32, 1), (5, 3, 5, 64, 32, 0),
                                            (40, 16, 16, 320, 32, 1), (2, 64, 64, 960, 32, 1)])
def test_groupnorm(B, H, W, Cc, G, silu):
    n = _native()
    x = _rand(B, H, W, Cc, seed=1, scale=1.5, shift=0.3)
    gamma = _rand(Cc, seed=2).float() * 0.2 + 1.0
    beta = _rand(Cc, seed=3).float() * 0.1
    y = torch.full_like(x, float("nan"))
    n.groupnorm(x, B, H * W, Cc, G, gamma, beta, 1e-5, silu, y)
    torch.cuda.synchronize()
    ref = Fn.group_norm(x.float().permute(0, 3, 1, 2), G, gamma, beta, 1e-5)
    if silu:
        ref = Fn.silu(ref)
    ref = ref.permute(0, 2, 3, 1)
    assert torch.isfinite(y.float()).all()
    assert (y.float() - ref).abs().max().item() <= 2 ** -9 * ref.abs().max().item() + 1e-3


def test_groupnorm_strided_views_and_determinism():
    """input / output are channel slices of wider buffers (skip concat); two runs are bit-identical"""
    n = _native()
    big = _rand(2, 32, 32, 1024, seed=4)
    x = big[..., 128:768]
    gamma = torch.ones(640, device="cuda")
    beta = torch.zeros(640, device="cuda")
    outs = []
    for _ in range(2):
        ybuf = torch.zeros(2, 32, 32, 896, dtype=torch.float16, device="cuda")
        y = ybuf[..., 64:704]
        n.groupnorm(x, 2, 32 * 32, 640, 32, gamma, beta, 1e-6, 0, y)
        torch.cuda.synchronize()
        assert (ybuf[..., :64] == 0).all() and (ybuf[..., 704:] == 0).all()
        outs.append(y.clone())
    assert torch.equal(outs[0], outs[1])
    ref = Fn.group_norm(x.float().permute(0, 3, 1, 2), 32, eps=1e-6).permute(0, 2, 3, 1)
    assert (outs[0].float() - ref).abs().max().item() <= 2 ** -9 * ref.abs().max().item() + 1e-3


@pytest.mark.parametrize("rows,Cc", [(4096, 320), (1000, 640), (77, 1280), (5, 512), (4099, 320), (3, 320), (1, 640), (129, 768)] +
                         # the CLIP widths: OpenCLIP-H (1024, five vectors per lane) and the 8-vector kernel (1288, 2048)
                         [(r, c) for c in (1024, 1288, 2048) for r in (77, 154, 616)])
def test_layernorm(rows, Cc):
    n = _native()
    x = _rand(rows, Cc, seed=5, scale=2.0, shift=-0.5)
    gamma = _rand(Cc, seed=6).float() * 0.2 + 1.0
    beta = _rand(Cc, seed=7).float() * 0.1
    y = torch.full_like(x, float("nan"))
    n.layernorm(x, rows, Cc, gamma, beta, 1e-5, y)
    torch.cuda.synchronize()
    ref = Fn.layer_norm(x.double(), (Cc,), gamma.double(), beta.double(), 1e-5)
    assert (y.double() - ref).abs().max().item() <= 2 ** -9 * ref.abs().max().item() + 1e-3


@pytest.mark.parametrize("Cc", [320, 640, 1280])
def test_layernorm_strided_rows(Cc):
    """input / output rows are slices of wider buffers (pitch != C): the lane-group kernel must honour both pitches"""
    n = _native()
    rows = 531
    big = _rand(rows, Cc + 64, seed=8, scale=1.5, shift=0.25)
    x = big[:, 32:32 + Cc]
    gamma = _rand(Cc, seed=9).float() * 0.2 + 1.0
    beta = _rand(Cc, seed=10).float() * 0.1
    ybuf = torch.zeros(rows, Cc + 128, dtype=torch.float16, device="cuda")
    y = ybuf[:, 64:64 + Cc]
    n.layernorm(x, rows, Cc, gamma, beta, 1e-5, y)
    torch.cuda.synchronize()
    assert (ybuf[:, :64] == 0).all() and (ybuf[:, 64 + Cc:] == 0).all()
    ref = Fn.layer_norm(x.float(), (Cc,), gamma, beta, 1e-5)
    assert (y.float() - ref).abs().max().item() <= 2 ** -9 * ref.abs().max().item() + 1e-3


def _gn_ref64(x, G, gamma, beta, eps, silu):
    ref = Fn.group_norm(x.double().permute(0, 3, 1, 2), G, gamma.double(), beta.double(), eps)
    return (Fn.silu(ref) if silu else ref).permute(0, 2, 3, 1)


@pytest.mark.parametrize("Cc", [320, 640])
@pytest.mark.parametrize("offset", [0, 64, 256, 512])
def test_groupnorm_large_mean(offset, Cc):
    """groups whose mean is large against their spread (std 1): the statistics must not cancel"""
    n = _native()
    B, H, W, G = 2, 32, 32, 32
    x = _rand(B, H, W, Cc, seed=12, shift=float(offset))
    gamma = _rand(Cc, seed=13).float() * 0.2 + 1.0
    beta = _rand(Cc, seed=14).float() * 0.1
    y = torch.full_like(x, float("nan"))
    n.groupnorm(x, B, H * W, Cc, G, gamma, beta, 1e-5, 0, y)
    torch.cuda.synchronize()
    ref = _gn_ref64(x, G, gamma, beta, 1e-5, 0)
    err = (y.double() - ref).abs().max().item()
    assert err <= 2 ** -9 * ref.abs().max().item() + 1e-3, err


@pytest.mark.parametrize("B,H,W,Cc,G,silu", [
    (2, 16, 16, 320, 8, 1), (2, 16, 16, 320, 16, 0), (2, 16, 16, 640, 64, 1),
    (2, 8, 8, 64, 64, 0),     # one channel per group
    (2, 8, 8, 32, 8, 1),      # the tiny test configuration's first level
    (3, 1, 1, 320, 32, 1),    # P < 16: a single statistics chunk
    (2, 3, 3, 640, 32, 0),
    (2, 1, 1, 64, 64, 0),     # one value per group: variance 0
])
def test_groupnorm_group_counts_and_tiny_images(B, H, W, Cc, G, silu):
    n = _native()
    x = _rand(B, H, W, Cc, seed=15, scale=1.5, shift=0.3)
    gamma = _rand(Cc, seed=16).float() * 0.2 + 1.0
    beta = _rand(Cc, seed=17).float() * 0.1
    y = torch.full_like(x, float("nan"))
    n.groupnorm(x, B, H * W, Cc, G, gamma, beta, 1e-5, silu, y)
    torch.cuda.synchronize()
    ref = _gn_ref64(x, G, gamma, beta, 1e-5, silu)
    assert torch.isfinite(y.float()).all()
    assert (y.double() - ref).abs().max().item() <= 2 ** -9 * ref.abs().max().item() + 1e-3


@pytest.mark.parametrize("Cc", [320, 768, 1024, 1288, 2048])
@pytest.mark.parametrize("offset", [0, 64, 256, 512])
def test_layernorm_large_mean(offset, Cc):
    """the same offset sweep for LayerNorm (two-pass statistics)"""
    n = _native()
    rows = 1000
    x = _rand(rows, Cc, seed=18, shift=float(offset))
    gamma = _rand(Cc, seed=19).float() * 0.2 + 1.0
    beta = _rand(Cc, seed=20).float() * 0.1
    y = torch.full_like(x, float("nan"))
    n.layernorm(x, rows, Cc, gamma, beta, 1e-5, y)
    torch.cuda.synchronize()
    ref = Fn.layer_norm(x.double(), (Cc,), gamma.double(), beta.double(), 1e-5)
    err = (y.double() - ref).abs().max().item()
    assert err <= 2 ** -9 * ref.abs().max().item() + 1e-3, err
