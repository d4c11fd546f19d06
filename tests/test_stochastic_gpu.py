"""Stochastic samplers on the GPU (DDIM eta > 0, Euler ancestral): the Philox step noise of the fused step kernel
against the numpy restatement of its specification (tests/_stochastic_oracle.py), the step kernel's noise term against a
float64 restatement, the engine's frame-noise table, and whole pipelines against the CPU oracle fed the same noise.
Tolerances of the full sampler are the calibrated ones of test_engine_gpu.py (final latents rel-L2 <= 1e-2; frames
mean |d| <= 1 LSB, >= 99 % within +-2 LSB, none beyond +-8 LSB)."""
import ctypes as C
import json

import numpy as np
import pytest
import torch
from PIL import Image

import _stochastic_oracle as O
from _helpers import MID_UNET, MID_VAE, TINY_UNET, TINY_VAE, make_oracle, product_cfgs

pytestmark = pytest.mark.gpu

LAT_C = 4


def _n():
    from stable_diffusion_videos_b200 import _native as n
    return n


def _p(t):
    return C.c_void_p(t.data_ptr() if t is not None else 0)


def _dev_table(entries):
    from stable_diffusion_videos_b200 import noise

    n = _n()
    tab = (n.FrameNoise * len(entries))(*[n.FrameNoise(*e) for e in entries])
    return noise.to_device(tab, "cuda")


def _noise(entries, hw, step):
    n = _n()
    F = len(entries)
    out = torch.full((F, LAT_C) + tuple(hw), float("nan"), device="cuda")
    d = _dev_table(entries)
    n.check(n.lib().sdw_step_noise(_p(d), F, LAT_C, hw[0], hw[1], step, _p(out), n.stream_ptr()))
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _frames_close(got, ref):
    d = np.abs(got.astype(np.int32) - ref.astype(np.int32))
    assert d.mean() <= 1.0 and (d <= 2).mean() >= 0.99 and d.max() <= 8, (d.mean(), (d <= 2).mean(), d.max())


def _rel_l2(a, b):
    return float((a - b).norm() / b.norm())


# ---------------------------------------------------------------------------------------------------------------------
# the noise
# ---------------------------------------------------------------------------------------------------------------------
def test_device_philox_is_bit_exact():
    n = _n()
    rng = np.random.default_rng(0)
    rows = [list(c) + list(k) for c, k, _ in
            [((0, 0, 0, 0), (0, 0), 0), ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, 0),
             ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), 0)]]
    rows += rng.integers(0, 2 ** 32, size=(1000, 6), dtype=np.uint64).tolist()
    inp = torch.from_numpy(np.array(rows, dtype=np.uint64).astype(np.uint32).view(np.int32)).cuda()
    out = torch.zeros((len(rows), 4), dtype=torch.int32, device="cuda")
    n.check(n.lib().sdw_philox4x32_10(_p(inp), len(rows), _p(out), n.stream_ptr()))
    got = out.cpu().numpy().view(np.uint32).astype(np.uint64)
    a = np.array(rows, dtype=np.uint64)
    want = np.stack(O.philox4x32_10(a[:, :4].T, a[:, 4:].T), axis=1)
    assert np.array_equal(got, want)
    assert [int(v) for v in got[0]] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]


@pytest.mark.parametrize("hw", [(9, 13), (64, 64)])
def test_step_noise_matches_the_specification(hw):
    entries = [(2 ** 40 + 7, 3, 1.0, 0.0), (9_000_000_123, 2 ** 63 + 5, 0.6, 0.8), (5, 2 ** 33, 0.0, 1.0),
               (2 ** 64 - 1, 12, float(np.float32(np.cos(0.3))), float(np.float32(np.sin(0.3))))]
    for step in (0, 1, 7, 49):
        got = _noise(entries, hw, step)
        ref = O.batch_noise(entries, step, (LAT_C,) + hw)
        assert np.isfinite(got).all()
        err = float(np.abs(got - ref).max())
        assert err <= 1e-5, (step, err)


def test_step_noise_does_not_depend_on_batch_position_or_size():
    hw = (9, 13)
    entries = [(k * 2 ** 33 + 11, 77 + k, 0.8, 0.6) for k in range(5)]
    full = _noise(entries, hw, 4)
    perm = [3, 0, 4, 1, 2]
    permuted = _noise([entries[i] for i in perm], hw, 4)
    assert np.array_equal(permuted.view(np.int32), full[perm].view(np.int32))
    two = _noise(entries[3:], hw, 4)
    assert np.array_equal(two.view(np.int32), full[3:].view(np.int32))


def test_walk_endpoint_noise_is_the_seed_stream():
    """T = 0 of a walk frame gives Z(key_a) bit for bit (and T = 1 Z(key_b)): the noise of the image with that key"""
    from stable_diffusion_videos_b200 import noise

    hw = (16, 16)
    tab = noise.as_numpy(noise.walk_table([0.0, 1.0], 2 ** 35 + 1, 424242))
    walk = _noise([tuple(r) for r in tab.tolist()], hw, 3)
    alone = _noise([(2 ** 35 + 1, 2 ** 35 + 1, 1.0, 0.0), (424242, 424242, 1.0, 0.0)], hw, 3)
    assert np.array_equal(walk.view(np.int32), alone.view(np.int32))


@pytest.mark.parametrize("seed,t", [(1, 0.0), (2 ** 40 + 3, 0.37)])
def test_step_noise_is_standard_normal(seed, t):
    from scipy import stats

    from stable_diffusion_videos_b200 import noise

    w_a, w_b = (float(w) for w in noise.as_numpy(noise.walk_table([t], 0, 0))[0].tolist()[2:])
    entries = [(seed + 2 * f, seed + 2 * f + 1, w_a, w_b) for f in range(16)]  # 16 independent frames
    z = _noise(entries, (128, 128), 5).reshape(-1).astype(np.float64)
    assert z.size >= 1_000_000
    assert abs(z.mean()) <= 5 / np.sqrt(z.size)  # 5 standard errors
    assert abs(z.var() - 1.0) <= 5 * np.sqrt(2.0 / z.size)
    assert stats.kstest(z, "norm").pvalue > 1e-3


def test_adjacent_walk_frames_get_nearly_the_same_noise():
    from stable_diffusion_videos_b200 import noise

    tab = noise.as_numpy(noise.walk_table(np.linspace(0.0, 1.0, 60), 42, 1337))
    z = _noise([tuple(r) for r in tab.tolist()], (64, 64), 0).reshape(60, -1)
    corr = [float(np.corrcoef(z[i], z[i + 1])[0, 1]) for i in range(59)]
    assert min(corr) > 0.99, min(corr)
    assert float(np.corrcoef(z[0], z[-1])[0, 1]) < 0.05  # the endpoints are independent fields


# ---------------------------------------------------------------------------------------------------------------------
# the step kernel
# ---------------------------------------------------------------------------------------------------------------------
def _coef(plan, i, guidance):
    n = _n()
    st = plan[i]
    k = n.StepCoef()
    k.guidance, k.c_x = float(guidance), float(st["c_x"])
    for j in range(5):
        k.c_e[j] = float(st["c_e"][j])
    for j in range(4):
        k.hist_slot[j] = int(st["hist_slot"][j])
    k.use_x_base, k.save_x_base, k.push_slot = st["use_x_base"], st["save_x_base"], st["push_slot"]
    k.next_in_scale = float(plan[i + 1]["in_scale"]) if i + 1 < len(plan) else 1.0
    k.push_e, k.push_x = float(st.get("push_e", 1.0)), float(st.get("push_x", 0.0))
    k.c_z = float(st.get("c_z", 0.0))
    return k


def _plan(kind, pred, steps, eta=None):
    from stable_diffusion_videos_b200 import schedulers as S

    s = S.SCHEDULERS[kind](prediction_type=pred)
    s.set_timesteps(steps)
    return s, (s.plan(eta=eta) if eta is not None else s.plan())


@pytest.mark.parametrize("kind,pred,eta,steps,F,hw", [
    ("ddim", "epsilon", 0.5, 6, 3, (9, 13)), ("ddim", "epsilon", 1.0, 10, 2, (64, 64)),
    ("ddim", "v_prediction", 0.5, 10, 2, (64, 64)), ("ddim", "v_prediction", 1.0, 6, 3, (9, 13)),
    ("euler_a", "epsilon", None, 6, 3, (9, 13)), ("euler_a", "v_prediction", None, 10, 2, (64, 64))])
def test_step_kernel_noise_term(kind, pred, eta, steps, F, hw):
    n = _n()
    lib = n.lib()
    H, W = hw
    sch, plan = _plan(kind, pred, steps, eta)
    entries = [(2 ** 36 + 17 * f, 5 + f, 0.8, 0.6) for f in range(F)]
    table = _dev_table(entries)
    rng = np.random.default_rng(steps * 7 + F)
    x = torch.from_numpy((rng.standard_normal((F, LAT_C, H, W)) * sch.init_noise_sigma).astype(np.float32)).cuda()
    xb, hist = torch.zeros_like(x), torch.zeros((4,) + tuple(x.shape), device="cuda")
    g = 7.5
    for i in range(len(plan)):
        k = _coef(plan, i, g)
        u = rng.standard_normal((F, H, W, LAT_C))
        eps = np.concatenate([u, u + 0.2 * rng.standard_normal(u.shape)]).astype(np.float32)
        before = x.cpu().numpy().astype(np.float64)
        n.check(lib.sdw_cfg_sched_step_noise(_p(torch.from_numpy(eps).cuda()), 1, _p(x), _p(xb), _p(hist), C.byref(k), F,
                                             LAT_C, H, W, C.c_void_p(0), LAT_C, _p(table), i, n.stream_ptr()))
        torch.cuda.synchronize()
        e64 = eps.astype(np.float64).transpose(0, 3, 1, 2)
        e = e64[:F] + k.guidance * (e64[F:] - e64[:F])
        z = O.batch_noise(entries, i, (LAT_C, H, W))
        ref = k.c_x * before + k.c_e[0] * e + k.c_z * z
        scale = float(np.abs(k.c_x * before).max() + abs(k.c_e[0]) * np.abs(e).max() * 3 + abs(k.c_z) * np.abs(z).max())
        err = float(np.abs(x.cpu().numpy() - ref).max())
        assert err <= 1e-6 * scale + 1e-5 * abs(k.c_z), (i, err, scale)


def test_step_kernel_without_noise_is_the_deterministic_kernel():
    """all c_z == 0 (DDIM eta = 0): the noise entry point computes the same bits as sdw_cfg_sched_step"""
    n = _n()
    lib = n.lib()
    F, H, W = 2, 9, 13
    _, plan = _plan("ddim", "v_prediction", 5, 0.0)
    table = _dev_table([(1, 2, 0.6, 0.8)] * F)
    rng = np.random.default_rng(3)
    x0 = torch.from_numpy(rng.standard_normal((F, LAT_C, H, W)).astype(np.float32)).cuda()
    xs = [x0.clone(), x0.clone()]
    nxt = [torch.zeros((2 * F, H, W, LAT_C), dtype=torch.float16, device="cuda") for _ in range(2)]
    scratch = [(torch.zeros_like(x0), torch.zeros((4,) + tuple(x0.shape), device="cuda")) for _ in range(2)]
    for i in range(len(plan)):
        k = _coef(plan, i, 7.5)
        assert k.c_z == 0.0
        eps = torch.from_numpy(rng.standard_normal((2 * F, H, W, LAT_C)).astype(np.float32)).cuda()
        n.check(lib.sdw_cfg_sched_step(_p(eps), 1, _p(xs[0]), _p(scratch[0][0]), _p(scratch[0][1]), C.byref(k), F, LAT_C,
                                       H, W, _p(nxt[0]), LAT_C, n.stream_ptr()))
        n.check(lib.sdw_cfg_sched_step_noise(_p(eps), 1, _p(xs[1]), _p(scratch[1][0]), _p(scratch[1][1]), C.byref(k), F,
                                             LAT_C, H, W, _p(nxt[1]), LAT_C, _p(table), i, n.stream_ptr()))
        torch.cuda.synchronize()
        assert torch.equal(xs[0].view(torch.int32), xs[1].view(torch.int32)), i
        assert torch.equal(nxt[0].view(torch.int16), nxt[1].view(torch.int16)), i


def test_deterministic_entry_point_rejects_noise():
    n = _n()
    lib = n.lib()
    F, H, W = 1, 4, 4
    x = torch.ones(F, LAT_C, H, W, device="cuda")
    xb, hist = torch.zeros_like(x), torch.zeros((4,) + tuple(x.shape), device="cuda")
    eps = torch.zeros(F, H, W, LAT_C, device="cuda")
    k = n.StepCoef()
    k.guidance, k.c_x, k.push_slot, k.c_z = 1.0, 2.0, -1, 0.5
    rc = lib.sdw_cfg_sched_step(_p(eps), 0, _p(x), _p(xb), _p(hist), C.byref(k), F, LAT_C, H, W, C.c_void_p(0), LAT_C,
                                n.stream_ptr())
    torch.cuda.synchronize()
    assert rc == 1 and b"c_z" in lib.sdw_last_error()
    assert bool((x == 1).all())
    rc = lib.sdw_cfg_sched_step_noise(_p(eps), 0, _p(x), _p(xb), _p(hist), C.byref(k), F, LAT_C, H, W, C.c_void_p(0),
                                      LAT_C, C.c_void_p(0), 0, n.stream_ptr())
    assert rc == 1 and b"frame-noise table" in lib.sdw_last_error()


# ---------------------------------------------------------------------------------------------------------------------
# the engine
# ---------------------------------------------------------------------------------------------------------------------
def _engine(ocfg_u, ocfg_v, hw, frames):
    from stable_diffusion_videos_b200.engine import Engine

    unet, vae = make_oracle(ocfg_u, ocfg_v)
    ucfg, vcfg = product_cfgs(ocfg_u, ocfg_v)
    eng = Engine(ucfg, vcfg, hw, frames, max_steps=64)
    eng.load_state_dict(unet.state_dict(), vae.state_dict())
    return eng, unet, vae


def _inputs(D, F, hw, seed=7):
    from oracle.pipeline import synthetic_embedding

    g = torch.Generator().manual_seed(seed)
    lat = torch.randn(F, 4, *hw, generator=g)
    cond = torch.cat([synthetic_embedding(k, dim=D) for k in range(F)]).half().float()
    unc = synthetic_embedding("", dim=D).half().float()
    return lat, cond, unc


def _table(entries):
    n = _n()
    return (n.FrameNoise * len(entries))(*[n.FrameNoise(*e) for e in entries])


def test_engine_noise_table_graph_and_segments():
    from stable_diffusion_videos_b200 import _native
    from stable_diffusion_videos_b200.schedulers import DDIMScheduler

    F, hw = 2, (8, 8)
    eng, _, _ = _engine(TINY_UNET, TINY_VAE, hw, F)
    lat, cond, unc = _inputs(TINY_UNET.cross_attention_dim, F, hw)
    lat, cond, unc = lat.cuda(), cond.cuda(), unc.cuda()
    eng.set_scheduler(DDIMScheduler(), 5, 7.5, eta=1.0)
    assert eng.stochastic
    with pytest.raises(_native.SdwError, match="frame-noise table"):
        eng.sample(lat, cond, unc)
    with pytest.raises(_native.SdwError, match="frame-noise table"):
        eng.sample(lat, cond, unc, callback=lambda *a: None)
    eng.set_frame_noise(_table([(11, 12, 0.6, 0.8), (2 ** 40, 2 ** 40, 1.0, 0.0)]))
    a = eng.sample(lat, cond, unc, use_graph=True, return_latents=True)
    b = eng.sample(lat, cond, unc, use_graph=True, return_latents=True)  # graph replay, same table
    seg = eng.sample(lat, cond, unc, return_latents=True, callback=lambda *a: None, callback_steps=2)
    torch.cuda.synchronize()
    for other in (b, seg):
        assert torch.equal(a[0], other[0]) and torch.equal(a[1].view(torch.int32), other[1].view(torch.int32))
    eng.set_frame_noise(_table([(13, 12, 0.6, 0.8), (2 ** 40, 2 ** 40, 1.0, 0.0)]))  # new key for frame 0 only
    c = eng.sample(lat, cond, unc, use_graph=True, return_latents=True)
    torch.cuda.synchronize()
    assert not torch.equal(c[1][0], a[1][0]) and torch.equal(c[1][1].view(torch.int32), a[1][1].view(torch.int32))
    # eta = 0 on the same engine: no table needed, the deterministic sampler
    eng.set_scheduler(DDIMScheduler(), 5, 7.5, eta=0.0)
    assert not eng.stochastic
    d = eng.sample(lat, cond, unc, return_latents=True)
    torch.cuda.synchronize()
    assert not torch.equal(d[1], a[1])
    with pytest.raises(ValueError, match="entries"):
        eng.set_frame_noise(_table([(1, 1, 1.0, 0.0)]))


@pytest.mark.parametrize("kind,cfgs,hw,steps", [
    ("ddim", (TINY_UNET, TINY_VAE), (8, 8), 5), ("euler_a", (TINY_UNET, TINY_VAE), (8, 8), 6),
    ("ddim", (MID_UNET, MID_VAE), (16, 16), 10), ("euler_a", (MID_UNET, MID_VAE), (16, 16), 10)])
def test_engine_stochastic_sampler_matches_oracle(kind, cfgs, hw, steps):
    """DDIM eta = 1 and Euler ancestral through the engine (tiny, and the MID config's SD-1.4 block structure with real
    kernel widths) against the CPU oracle given the same step noise"""
    from oracle.pipeline import to_uint8
    from stable_diffusion_videos_b200.schedulers import SCHEDULERS

    F = 2
    eng, unet, vae = _engine(cfgs[0], cfgs[1], hw, F)
    lat, cond, unc = _inputs(cfgs[0].cross_attention_dim, F, hw)
    entries = [(2 ** 34 + 1, 99, 0.8, 0.6), (7, 7, 1.0, 0.0)]
    eta = 1.0 if kind == "ddim" else 0.0
    img, lat_ref = O.sample_frames(unet, vae, O.make_scheduler(kind), lat, cond, unc, steps, 7.5, eta=eta, table=entries,
                                   return_latents=True)
    eng.set_scheduler(SCHEDULERS[kind](), steps, 7.5, eta=eta)
    eng.set_frame_noise(_table(entries))
    u8, fin = eng.sample(lat.cuda(), cond.cuda(), unc.cuda(), return_latents=True)
    torch.cuda.synchronize()
    assert _rel_l2(fin.cpu(), lat_ref) <= 1e-2, _rel_l2(fin.cpu(), lat_ref)
    _frames_close(u8.cpu().numpy(), to_uint8(img))


# ---------------------------------------------------------------------------------------------------------------------
# the pipeline
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny():
    from stable_diffusion_videos_b200.pipeline import (NativeUNet, NativeVAE, StableDiffusionWalkPipeline,
                                                       SyntheticTextEncoder, SyntheticTokenizer)
    from stable_diffusion_videos_b200.schedulers import DDIMScheduler

    unet, vae = make_oracle(TINY_UNET, TINY_VAE)
    ucfg, vcfg = product_cfgs(TINY_UNET, TINY_VAE)
    usd = {k: v.half() for k, v in unet.state_dict().items()}
    vsd = {k: v.half() for k, v in vae.state_dict().items()}
    pipe = StableDiffusionWalkPipeline(NativeVAE(vcfg, vsd), SyntheticTextEncoder(TINY_UNET.cross_attention_dim),
                                       SyntheticTokenizer(), NativeUNet(ucfg, usd), DDIMScheduler()).to("cuda")
    return pipe, unet, vae


@pytest.mark.parametrize("kind", ["ddim", "euler_a"])
def test_call_matches_oracle(tiny, kind):
    from oracle.pipeline import to_uint8
    from stable_diffusion_videos_b200.schedulers import SCHEDULERS

    pipe, unet, vae = tiny
    pipe.scheduler = SCHEDULERS[kind]()
    eta = 1.0 if kind == "ddim" else 0.0
    lat = torch.randn(3, 4, 8, 8, generator=torch.Generator(device="cuda").manual_seed(1), device="cuda",
                      dtype=torch.float16)
    emb = torch.cat([pipe.embed_text(str(k)) for k in range(3)])
    seen = []
    out = pipe(text_embeddings=emb, latents=lat, height=64, width=64, num_inference_steps=5, eta=eta,
               generator=torch.Generator(device="cuda").manual_seed(11), output_type="pil",
               callback=lambda i, t, x: seen.append(x.float().cpu()))
    got = np.stack([np.asarray(im) for im in out.images])
    table = O.call_table(3, torch.Generator(device="cuda").manual_seed(11), "cuda")
    img, lat_ref = O.sample_frames(unet, vae, O.make_scheduler(kind), lat.float().cpu(), emb.float().cpu(),
                                   pipe._uncond([""]).float().cpu(), 5, 7.5, eta=eta, table=table, return_latents=True)
    assert _rel_l2(seen[-1], lat_ref) <= 1e-2
    _frames_close(got, to_uint8(img))
    # the graph path (no callback) renders the same frames; eta = 0 renders other ones
    again = pipe(text_embeddings=emb, latents=lat, height=64, width=64, num_inference_steps=5, eta=eta,
                 generator=torch.Generator(device="cuda").manual_seed(11))
    assert np.array_equal(np.stack([np.asarray(im) for im in again.images]), got)
    if kind == "ddim":
        det = pipe(text_embeddings=emb, latents=lat, height=64, width=64, num_inference_steps=5, eta=0.0)
        assert np.abs(np.stack([np.asarray(im) for im in det.images]).astype(int) - got).max() > 8


def _walk_frames(root, name):
    files = sorted(p.relative_to(root / name).as_posix() for p in (root / name).glob("**/*.png"))
    return files, np.stack([np.asarray(Image.open(root / name / f)) for f in files])


def test_walk_with_eta_matches_oracle(tiny, tmp_path):
    from stable_diffusion_videos_b200.schedulers import DDIMScheduler

    pipe, unet, vae = tiny
    pipe.scheduler = DDIMScheduler()
    seeds = [42, 2 ** 33 + 1337, 2022]
    kw = dict(output_dir=str(tmp_path), num_inference_steps=4, height=64, width=64, make_video=False,
              num_interpolation_steps=[3, 3])
    pipe.walk(["0", "1", "2"], seeds=seeds, name="eta1", eta=1.0, batch_size=2, **kw)
    assert json.loads((tmp_path / "eta1" / "prompt_config.json").read_text())["eta"] == 1.0
    files, got = _walk_frames(tmp_path, "eta1")
    assert files == [f"eta1_{i:06d}/frame{j:06d}.png" for i in range(2) for j in range(3)]
    embed = [pipe.embed_text(str(k)).float().cpu() for k in range(3)]
    init = [pipe.init_noise(s, (1, 4, 8, 8), torch.float16).float().cpu() for s in seeds]
    ref = O.walk_frames(unet, vae, "ddim", seeds, embed, pipe._uncond([""]).float().cpu(), init, 3, 4, 7.5, eta=1.0)
    _frames_close(got, ref)
    pipe.walk(["0", "1", "2"], seeds=seeds, name="eta0", eta=0.0, batch_size=2, **kw)
    assert np.abs(_walk_frames(tmp_path, "eta0")[1].astype(int) - got).max() > 8


def test_stochastic_walk_resume_and_batch_size(tiny, tmp_path):
    """the noise of a frame is a function of its seeds and T: an interrupted and resumed walk is bit-identical to an
    uninterrupted one, and batch sizes 1 and 3 agree up to the GEMM shapes"""
    from stable_diffusion_videos_b200.schedulers import EulerAncestralDiscreteScheduler

    pipe, _, _ = tiny
    pipe.scheduler = EulerAncestralDiscreteScheduler()
    kw = dict(output_dir=str(tmp_path), num_inference_steps=4, height=64, width=64, make_video=False)
    pipe.walk(["0", "1"], seeds=[5, 2 ** 40 + 6], num_interpolation_steps=5, name="full", batch_size=3, **kw)
    pipe.walk(["0", "1"], seeds=[5, 2 ** 40 + 6], num_interpolation_steps=5, name="res", batch_size=3, **kw)
    clip = tmp_path / "res" / "res_000000"
    for j in (2, 3, 4):
        (clip / f"frame{j:06d}.png").unlink()
    pipe.walk(name="res", resume=True, batch_size=3, **kw)
    pipe.walk(["0", "1"], seeds=[5, 2 ** 40 + 6], num_interpolation_steps=5, name="b1", batch_size=1, **kw)
    _, full = _walk_frames(tmp_path, "full")
    _, res = _walk_frames(tmp_path, "res")
    _, b1 = _walk_frames(tmp_path, "b1")
    assert full.shape[0] == 5 and np.array_equal(res, full)
    _frames_close(b1, full)


def test_from_random_euler_ancestral():
    from stable_diffusion_videos_b200.configs import UNetConfig, VAEConfig
    from stable_diffusion_videos_b200.pipeline import StableDiffusionWalkPipeline
    from stable_diffusion_videos_b200.schedulers import EulerAncestralDiscreteScheduler

    ucfg, vcfg = product_cfgs(TINY_UNET, TINY_VAE)
    pipe = StableDiffusionWalkPipeline.from_random(ucfg, vcfg, scheduler="euler_a")
    assert isinstance(pipe.scheduler, EulerAncestralDiscreteScheduler)
    a = pipe("0", height=64, width=64, num_inference_steps=3, generator=torch.Generator(device="cuda").manual_seed(1))
    b = pipe("0", height=64, width=64, num_inference_steps=3, generator=torch.Generator(device="cuda").manual_seed(1))
    assert np.array_equal(np.asarray(a.images[0]), np.asarray(b.images[0]))  # seeded: latents and step noise
