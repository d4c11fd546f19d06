"""Real-ESRGAN x4 on the GPU: the new GEMM capabilities (BLOCK_N 32, LeakyReLU, dense-block reads of C = 96 / 160 from a
192-channel buffer, 32-channel slice outputs), the two edge convs, the whole network against the CPU oracle with a
calibrated tolerance, graph / eager reproducibility, and the walk with `upsample=True`."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from PIL import Image

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
SENTINEL = 1234.0


def _fp64_conv(x_nhwc, w, b, act=0):
    y = F.conv2d(x_nhwc.double().permute(0, 3, 1, 2), w.double(), None if b is None else b.double(), padding=1)
    if act == 2:
        y = F.leaky_relu(y, 0.2)
    mag = F.conv2d(x_nhwc.double().abs().permute(0, 3, 1, 2), w.double().abs(), None, padding=1)
    return y.permute(0, 2, 3, 1), mag.permute(0, 2, 3, 1)


def _check(got, ref, mag):
    err = (got.double().cpu() - ref.cpu()).abs()
    tol = 2.0 ** -10 * ref.cpu().abs() + 2.0 ** -20 * mag.cpu() + 1e-6
    assert torch.isfinite(got).all()
    assert (err <= tol).all(), float((err - tol).max())


def _gemm_desc(A, Cin, lda, Bn, H, W, wp, N, bias, out, ldc, **kw):
    from stable_diffusion_videos_b200._native import GemmDesc

    d = GemmDesc()
    d.A, d.C, d.W, d.H, d.B = A.data_ptr(), Cin, W, H, Bn
    d.sW, d.sH, d.sB = lda, W * lda, H * W * lda
    d.conv = 1
    d.Wt, d.N = wp.data_ptr(), N
    d.bias = bias.data_ptr() if bias is not None else None
    d.out, d.ldc = out.data_ptr(), ldc
    d.alpha = 1.0
    for k, v in kw.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("et", [1, 2])
@pytest.mark.parametrize("shape", [(1, 16, 16, 64), (2, 13, 21, 128), (1, 40, 24, 64)])
def test_block_n_32_leaky_relu(et, shape):
    from stable_diffusion_videos_b200 import _native

    torch.manual_seed(0)
    Bn, H, W, Cin = shape
    N = 32
    x = torch.randn(Bn, H, W, Cin, device="cuda").half()
    w = (torch.randn(N, Cin, 3, 3, device="cuda") * 0.05).half()
    b = torch.randn(N, device="cuda") * 0.1
    out = torch.full((Bn, H, W, N), float("nan"), device="cuda").half()
    wp = _native.pack_weight(w)
    d = _gemm_desc(x, Cin, Cin, Bn, H, W, wp, N, b, out, N, bn=32, ver=1, act=2, et=et)
    _native.gemm(d)
    torch.cuda.synchronize()
    ref, mag = _fp64_conv(x.cpu(), w.cpu(), b.cpu(), act=2)
    _check(out, ref, mag)


@pytest.mark.parametrize("et", [1, 2])
@pytest.mark.parametrize("cin,off", [(64, 64), (96, 96), (128, 128), (160, 160), (96, 64), (160, 128)])
def test_dense_block_reads_and_slice_writes(cin, off, et):
    """3x3 conv reading C channels of a 192-pitch buffer whose other channels and trailing rows are NaN, writing a
    32-channel slice of another 192-pitch buffer whose other bytes are a sentinel that must survive."""
    from stable_diffusion_videos_b200 import _native

    torch.manual_seed(1)
    Bn, H, W = 2, 19, 24
    buf = torch.full((Bn * H * W + 3 * W, 192), float("nan"), device="cuda").half()
    x = torch.randn(Bn, H, W, cin).half()
    buf[: Bn * H * W, :cin] = x.reshape(-1, cin).cuda()
    w = (torch.randn(32, cin, 3, 3) * 0.05).half()
    b = torch.randn(32) * 0.1
    out = torch.full((Bn * H * W + W, 192), SENTINEL, device="cuda").half()
    wp, bd = _native.pack_weight(w.cuda()), b.cuda()
    d = _gemm_desc(buf, cin, 192, Bn, H, W, wp, 32, bd, out[:, off:], 192, bn=32, ver=1, act=2, et=et)
    _native.gemm(d)
    torch.cuda.synchronize()
    o = out.cpu()
    ref, mag = _fp64_conv(x, w, b, act=2)
    _check(o[: Bn * H * W, off:off + 32].reshape(Bn, H, W, 32), ref, mag)
    keep = torch.ones_like(o, dtype=torch.bool)
    keep[: Bn * H * W, off:off + 32] = False
    assert (o[keep] == SENTINEL).all()


@pytest.mark.parametrize("et", [0, 1])
def test_rrdb_tail_epilogue(et):
    """The rdb1 / rdb2 tail, 0.2 (acc + b) + x, into a 192-pitch slice on both epilogue paths (the rdb3 tail's scaled
    second residual is internal to the engine and covered by the end-to-end tests)."""
    from stable_diffusion_videos_b200 import _native

    torch.manual_seed(2)
    Bn, H, W = 1, 16, 32
    buf = torch.randn(Bn * H * W, 192).half()
    w = (torch.randn(64, 192, 3, 3) * 0.03).half()
    b = torch.randn(64) * 0.1
    bc = buf.cuda()
    out = torch.full((Bn * H * W, 192), SENTINEL, device="cuda").half()
    wp, bd = _native.pack_weight(w.cuda()), (b * 0.2).cuda()
    d = _gemm_desc(bc, 192, 192, Bn, H, W, wp, 64, bd, out, 192, alpha=0.2, resid=bc.data_ptr(), ldr=192, et=et)
    _native.gemm(d)
    torch.cuda.synchronize()
    ref, mag = _fp64_conv(buf.reshape(Bn, H, W, 192), w, b)
    ref = 0.2 * ref + buf[:, :64].double().reshape(Bn, H, W, 64)
    _check(out.cpu()[:, :64].reshape(Bn, H, W, 64), ref, 0.2 * mag + buf[:, :64].double().abs().reshape(Bn, H, W, 64))
    assert (out.cpu()[:, 64:] == SENTINEL).all()


# ---- edge kernels ------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(1, 7, 9), (2, 16, 16), (3, 33, 5)])
def test_conv_first_u8(shape):
    from stable_diffusion_videos_b200 import _native

    lib = _native.lib()
    Bn, H, W = shape
    g = torch.Generator().manual_seed(3)
    x = torch.randint(0, 256, (Bn, H, W, 3), generator=g, dtype=torch.uint8)
    w = (torch.randn(64, 3, 3, 3, generator=g) * 0.2).half()
    b = torch.randn(64, generator=g) * 0.1
    y = torch.full((Bn * H * W, 192), SENTINEL, device="cuda").half()
    xd, wd, bd = x.cuda(), w.cuda(), b.cuda()
    _native.check(lib.sdw_conv_first_u8(_native.ptr(xd), Bn, H, W, _native.ptr(wd), _native.ptr(bd), 64, _native.ptr(y),
                                        C.c_int64(192), _native.stream_ptr()))
    torch.cuda.synchronize()
    xf = (x.float() / 255.0).half()
    ref, mag = _fp64_conv(xf, w, b)
    _check(y.cpu()[:, :64].reshape(Bn, H, W, 64), ref, mag)
    assert (y.cpu()[:, 64:] == SENTINEL).all()


@pytest.mark.parametrize("shape", [(1, 8, 8), (2, 32, 48), (1, 37, 21)])
def test_conv_last_u8_is_the_rounding_of_its_own_fp32_output(shape):
    from stable_diffusion_videos_b200 import _native

    lib = _native.lib()
    Bn, H, W = shape
    g = torch.Generator().manual_seed(4)
    x = torch.randn(Bn, H, W, 64, generator=g).half()
    w = (torch.randn(3, 64, 3, 3, generator=g) * 0.05).half()
    b = torch.tensor([0.5, 0.4, 0.6])
    f32 = torch.full((Bn, H, W, 3), float("nan"), device="cuda")
    u8 = torch.zeros((Bn, H, W, 3), dtype=torch.uint8, device="cuda")
    xd, wd, bd = x.cuda(), w.cuda(), b.cuda()
    _native.check(lib.sdw_conv_last_u8(_native.ptr(xd), C.c_int64(64), Bn, H, W, 64, _native.ptr(wd), _native.ptr(bd),
                                       _native.ptr(f32), _native.ptr(u8), _native.stream_ptr()))
    # the VAE form on the same input: (v / 2 + 0.5) before the clamp
    u8v = torch.zeros_like(u8)
    _native.check(lib.sdw_conv_out_small(_native.ptr(xd), C.c_int64(64), Bn, H, W, 64, _native.ptr(wd), _native.ptr(bd),
                                         3, None, _native.ptr(u8v), _native.stream_ptr()))
    torch.cuda.synchronize()
    v = f32.cpu()
    ref, mag = _fp64_conv(x, w, b)
    assert ((v.double() - ref).abs() <= 1e-5 * mag + 1e-6).all()
    assert ((v < 0).any() and (v > 1).any())  # the clamp is exercised
    assert torch.equal(u8.cpu(), (v.clamp(0, 1) * 255).round().to(torch.uint8))
    assert torch.equal(u8v.cpu(), ((v * 0.5 + 0.5).clamp(0, 1) * 255).round().to(torch.uint8))


# ---- end to end against the oracle -------------------------------------------------------------
def _model(num_block, seed, calib_frames):
    """random fp16-rounded weights with non-zero biases everywhere; conv_last rescaled so the fp32 oracle's pre-clamp
    output spans about [-0.2, 1.2] on `calib_frames` (otherwise the clamp hides errors)."""
    from oracle.esrgan import upsample_u8
    from stable_diffusion_videos_b200.upsampling import RealESRGANModel

    m = RealESRGANModel.from_random(seed, num_block=num_block)
    g = torch.Generator().manual_seed(seed + 100)
    sd = {k: v.float() for k, v in m.state.items()}
    for k in sd:
        if k.startswith("body.") and k.endswith(".bias"):
            sd[k] = torch.randn(sd[k].shape, generator=g) * 0.02
    sd = {k: v.half().float() for k, v in sd.items()}
    _, y = upsample_u8(calib_frames, sd, num_block)
    lo, hi = np.percentile(y, 0.5), np.percentile(y, 99.5)
    a = 1.4 / max(hi - lo, 1e-6)
    sd["conv_last.weight"] = (sd["conv_last.weight"] * a).half().float()
    sd["conv_last.bias"] = (sd["conv_last.bias"] * a + (-0.2 - a * lo)).half().float()
    return RealESRGANModel(state_dict=sd), sd


def _frames(n, h, w, seed):
    """smooth-ish synthetic frames (gradients + noise), uint8 RGB"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([xx / max(w - 1, 1), yy / max(h - 1, 1), (xx + yy) / max(h + w - 2, 1)], -1)
    f = base[None] * 200 + rng.normal(0, 25, (n, h, w, 3)) + 20
    return np.clip(f, 0, 255).round().astype(np.uint8)


def _compare(model, sd, num_block, frames, frames_per_call):
    from oracle.esrgan import upsample_u8

    x = torch.from_numpy(frames).cuda()
    eng = model.engine(frames.shape[1], frames.shape[2], frames_per_call)
    B = frames.shape[0]
    u8 = torch.empty((B, 4 * frames.shape[1], 4 * frames.shape[2], 3), dtype=torch.uint8, device="cuda")
    pre = torch.empty(u8.shape, dtype=torch.float32, device="cuda")
    for i0 in range(0, B, frames_per_call):
        eng.run(x[i0:i0 + frames_per_call], u8[i0:i0 + frames_per_call], pre[i0:i0 + frames_per_call])
    torch.cuda.synchronize()
    u_ref, y_ref = upsample_u8(frames, sd, num_block)
    u_16, y_16 = upsample_u8(frames, sd, num_block, fp16_storage=True)
    got_u, got_y = u8.cpu().numpy(), pre.cpu().numpy()
    assert np.isfinite(got_y).all()
    assert torch.equal(u8.cpu(), (pre.cpu().clamp(0, 1) * 255).round().to(torch.uint8))

    def stats(u, y):
        d = np.abs(u.astype(np.int32) - u_ref.astype(np.int32))
        return (float(np.linalg.norm(y - y_ref) / np.linalg.norm(y_ref)), float(d.mean()), float(np.percentile(d, 99.9)))

    nat, spread = stats(got_u, got_y), stats(u_16, y_16)
    # calibrated: at most 1.25x the fp16-storage oracle's own distance from the fp32 oracle (p99.9 of integer levels
    # gets a floor of one level)
    assert nat[0] <= 1.25 * spread[0] + 1e-6, (nat, spread)
    assert nat[1] <= 1.25 * spread[1] + 1e-3 and nat[1] <= 1.0, (nat, spread)
    assert nat[2] <= max(1.25 * spread[2], 1.0), (nat, spread)
    return u8


@pytest.mark.parametrize("num_block", [1, 2])
@pytest.mark.parametrize("hw", [(8, 8), (24, 40), (37, 53)])
@pytest.mark.parametrize("fpc", [1, 3])
def test_network_matches_oracle(num_block, hw, fpc):
    frames = _frames(3, *hw, seed=hw[0] + num_block)
    model, sd = _model(num_block, 7 + num_block, frames)
    _compare(model, sd, num_block, frames, fpc)


def test_forward_matches_oracle_and_returns_bgr():
    from oracle.esrgan import upsample_u8

    frames = _frames(1, 37, 53, seed=5)
    model, sd = _model(2, 11, frames)
    img = frames[0].astype(np.float32) / 255.0  # the float frame the reference hands over
    bgr = model(img, convert_to_pil=False)
    pil = model(img)
    u_16, _ = upsample_u8(frames, sd, 2, fp16_storage=True)
    assert bgr.shape == (148, 212, 3) and np.array_equal(np.asarray(pil), bgr[:, :, ::-1])
    assert np.abs(bgr[:, :, ::-1].astype(int) - u_16[0].astype(int)).mean() <= 1.0


def test_full_x4plus_network_at_64x64():
    frames = _frames(1, 64, 64, seed=9)
    model, sd = _model(23, 1, frames)
    _compare(model, sd, 23, frames, 1)


def test_graph_replay_equals_eager_and_is_reproducible():
    from stable_diffusion_videos_b200.upsampling import RealESRGANModel

    model = RealESRGANModel.from_random(2, num_block=2).to("cuda")
    x = torch.from_numpy(_frames(2, 24, 40, seed=1)).cuda()
    eng = model.engine(24, 40, 2)
    outs = []
    for use_graph in (False, True, True, False):
        o = torch.zeros((2, 96, 160, 3), dtype=torch.uint8, device="cuda")
        p = torch.zeros(o.shape, dtype=torch.float32, device="cuda")
        eng.run(x, o, p, use_graph=use_graph)
        outs.append((o.cpu(), p.cpu()))
    for o, p in outs[1:]:
        assert torch.equal(o, outs[0][0]) and torch.equal(p, outs[0][1])
    # the device path (own stream, two frames per call) gives the same bytes
    assert torch.equal(model.upsample_frames(x).cpu(), outs[0][0])
    assert torch.equal(model.upsample_frames(x, frames_per_call=1).cpu(), outs[0][0])


def test_profile_lists_every_op(tmp_path):
    from stable_diffusion_videos_b200.upsampling import RealESRGANModel

    model = RealESRGANModel.from_random(2, num_block=2).to("cuda")
    eng = model.engine(16, 16, 1)
    eng.profile(tmp_path / "p.tsv")
    rows = [l.split("\t") for l in (tmp_path / "p.tsv").read_text().splitlines()]
    assert len(rows) == 1 + 2 * 15 + 1 + 8 + 1 + 1
    assert rows[0][3].startswith("conv_first") and rows[-1][3].startswith("conv_last")


# ---- the walk ----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pipe():
    from _helpers import TINY_UNET, TINY_VAE, make_oracle, product_cfgs
    from stable_diffusion_videos_b200.pipeline import (NativeUNet, NativeVAE, StableDiffusionWalkPipeline,
                                                       SyntheticTextEncoder, SyntheticTokenizer)
    from stable_diffusion_videos_b200.schedulers import PNDMScheduler
    from stable_diffusion_videos_b200.upsampling import RealESRGANModel

    unet, vae = make_oracle(TINY_UNET, TINY_VAE)
    ucfg, vcfg = product_cfgs(TINY_UNET, TINY_VAE)
    usd = {k: v.half() for k, v in unet.state_dict().items()}
    vsd = {k: v.half() for k, v in vae.state_dict().items()}
    p = StableDiffusionWalkPipeline(NativeVAE(vcfg, vsd), SyntheticTextEncoder(TINY_UNET.cross_attention_dim),
                                    SyntheticTokenizer(), NativeUNet(ucfg, usd), PNDMScheduler()).to("cuda")
    p.upsampler = RealESRGANModel.from_random(4, num_block=1)
    return p


def _read(root):
    files = sorted(p.relative_to(root).as_posix() for p in root.glob("**/*.png"))
    return files, [np.asarray(Image.open(root / f)) for f in files]


def test_walk_with_upsample_equals_upsampled_frames(pipe, tmp_path):
    kw = dict(seeds=[42, 1337, 2022], num_interpolation_steps=[3, 3], fps=3, num_inference_steps=3, height=64,
              width=64, batch_size=2, make_video=False, output_dir=str(tmp_path))  # 3 frames per clip: a tail batch of 1
    pipe.walk(["0", "1", "2"], name="plain", upsample=False, **kw)
    pipe.walk(["0", "1", "2"], name="up", upsample=True, **kw)
    fp, plain = _read(tmp_path / "plain")
    fu, up = _read(tmp_path / "up")
    assert [f.replace("plain", "up") for f in fp] == fu and len(fu) == 6
    assert plain[0].shape == (16, 16, 3) and up[0].shape == (64, 64, 3)
    want = pipe.upsampler.upsample_frames(torch.from_numpy(np.stack(plain)).cuda()).cpu().numpy()
    assert np.array_equal(np.stack(up), want)
    # resume: the config records upsample=True; deleted frames come back identical
    clip = tmp_path / "up" / "up_000001"
    (clip / "frame000002.png").unlink()
    (clip / "frame000001.png").unlink()
    pipe.walk(name="up", resume=True, output_dir=str(tmp_path), batch_size=2, make_video=False)
    _, again = _read(tmp_path / "up")
    assert np.array_equal(np.stack(again), want)


def test_upsample_imagefolder_and_outscale(pipe, tmp_path):
    import cv2

    model = pipe.upsampler
    src = tmp_path / "in"
    (src / "sub").mkdir(parents=True)
    frames = _frames(3, 12, 20, seed=3)
    Image.fromarray(frames[0]).save(src / "a.png")
    Image.fromarray(frames[1]).save(src / "b.jpg")
    Image.fromarray(frames[2]).save(src / "sub" / "c.png")
    (src / "notes.txt").write_text("x")
    out = tmp_path / "out"
    model.upsample_imagefolder(src, out, suffix="_x4")
    assert sorted(p.name for p in out.glob("*")) == ["a_x4.png", "b_x4.png"]
    want = model.upsample_frames(torch.from_numpy(frames[:1]).cuda())[0].cpu().numpy()
    assert np.array_equal(np.asarray(Image.open(out / "a_x4.png")), want)
    t0 = (out / "a_x4.png").stat().st_mtime_ns
    Image.fromarray(frames[2]).save(out / "b_x4.png")  # an existing output is kept unless force=True
    model.upsample_imagefolder(src, out, suffix="_x4")
    assert (out / "a_x4.png").stat().st_mtime_ns == t0 and np.asarray(Image.open(out / "b_x4.png")).shape == (12, 20, 3)
    model.upsample_imagefolder(src, out, suffix="_x4", force=True, recursive=True)
    assert np.asarray(Image.open(out / "b_x4.png")).shape == (48, 80, 3) and (out / "sub" / "c_x4.png").exists()
    # outscale != 4: LANCZOS4 resize of the x4 uint8 result (BGR out, as the reference)
    img = frames[0].astype(np.float32) / 255.0
    x4 = model(img, convert_to_pil=False)
    x2 = model(img, outscale=2, convert_to_pil=False)
    assert x2.shape == (24, 40, 3)
    assert np.array_equal(x2, cv2.resize(x4, (40, 24), interpolation=cv2.INTER_LANCZOS4))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_sharded_walk_with_upsample_equals_single_process(tmp_path):
    worker = os.path.join(HERE, "_esrgan_walk_worker.py")
    r1 = subprocess.run([sys.executable, worker, str(tmp_path), "one"], capture_output=True, text=True, timeout=600)
    assert r1.returncode == 0, r1.stderr[-3000:]
    r2 = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                         "--master-addr", "127.0.0.1", "--master-port", "29733", worker, str(tmp_path), "two"],
                        capture_output=True, text=True, timeout=600)
    assert r2.returncode == 0, r2.stderr[-3000:]
    f1, one = _read(tmp_path / "one")
    f2, two = _read(tmp_path / "two")
    assert [f.replace("one", "") for f in f1] == [f.replace("two", "") for f in f2] and len(f1) == 9
    for a, b in zip(one, two):
        assert a.shape == (64, 64, 3) and np.abs(a.astype(int) - b.astype(int)).max() <= 1
