"""The fused classifier-free-guidance + scheduler step (sdw_cfg_sched_step) and the state initialisation
(sdw_latents_init), driven through the C ABI with the real step tables of every scheduler and compared with a float64
restatement of the update documented in include/sdwalk.h:

    e = u + g (c - u);  s = use_x_base ? x_base : x;  x' = c_x s + c_e[0] e + sum_j c_e[1+j] hist[hist_slot[j]]
    save_x_base: x_base := x (before the update);  push_slot >= 0: hist[push_slot] := push_e e + push_x s

x, x_base and the history ring stay on the device between steps, as in the engine; after every step each of them is
compared with the reference step applied to the state the kernel started from."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

LAT_C = 4  # latent channels


def _n():
    from stable_diffusion_videos_b200 import _native as n
    return n


def _p(t):
    return C.c_void_p(t.data_ptr() if t is not None else 0)


def _scheduler(name, pred):
    from stable_diffusion_videos_b200 import schedulers as S

    return S.SCHEDULERS[name](prediction_type=pred)


def _coef(plan, i, guidance):
    n = _n()
    st = plan[i]
    k = n.StepCoef()
    k.guidance = float(guidance)
    k.c_x = float(st["c_x"])
    for j in range(5):
        k.c_e[j] = float(st["c_e"][j])
    for j in range(4):
        k.hist_slot[j] = int(st["hist_slot"][j])
    k.use_x_base, k.save_x_base, k.push_slot = st["use_x_base"], st["save_x_base"], st["push_slot"]
    k.next_in_scale = float(plan[i + 1]["in_scale"]) if i + 1 < len(plan) else 1.0
    k.push_e, k.push_x = float(st.get("push_e", 1.0)), float(st.get("push_x", 0.0))
    return k


def _ref_step(k, eps_nhwc, has_uncond, F, x, x_base, hist):
    """float64 restatement of one step on host copies of the state (NCHW x / x_base, [4] + NCHW hist).  Also returns
    the magnitude of the terms summed into x' and into the pushed history entry, the scale of fp32's rounding."""
    eps = eps_nhwc.astype(np.float64).transpose(0, 3, 1, 2)  # NHWC -> NCHW
    if has_uncond:
        u, c = eps[:F], eps[F:]
        e = u + k.guidance * (c - u)
        e_mag = np.abs(u) + abs(k.guidance) * (np.abs(c) + np.abs(u))
    else:
        e = eps
        e_mag = np.abs(e)
    x, x_base, hist = x.astype(np.float64), x_base.astype(np.float64), hist.astype(np.float64)
    if k.save_x_base:
        x_base = x.copy()
    s = x_base if k.use_x_base else x
    xn = k.c_x * s + k.c_e[0] * e
    mag = np.abs(k.c_x * s) + abs(k.c_e[0]) * e_mag
    for j in range(4):
        if k.c_e[j + 1] != 0.0:  # a zero coefficient does not read its slot (it may still be unwritten)
            xn = xn + k.c_e[j + 1] * hist[k.hist_slot[j]]
            mag = mag + abs(k.c_e[j + 1]) * np.abs(hist[k.hist_slot[j]])
    push_mag = 0.0
    if k.push_slot >= 0:
        hist = hist.copy()
        hist[k.push_slot] = k.push_e * e + k.push_x * s
        push_mag = float((abs(k.push_e) * e_mag + abs(k.push_x) * np.abs(s)).max())
    return xn, x_base, hist, float(mag.max()), push_mag


def _amax(a):
    a = a[~np.isnan(a)]
    return float(np.abs(a).max()) if a.size else 0.0


def _close(got, ref, scale):
    """|d| <= 1e-6 * scale elementwise; NaN (a slot never written) must match NaN."""
    got = got.astype(np.float64)
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan)
    err = np.abs(got[~nan] - ref[~nan])
    return err.size == 0 or float(err.max()) <= 1e-6 * scale


# (scheduler, prediction, steps, F, has_uncond, (H, W), guidance, next_in channel pitch or None)
CASES = [
    ("pndm", "epsilon", 4, 1, 1, (9, 13), 7.5, 4),
    ("pndm", "epsilon", 10, 3, 1, (64, 64), 15.0, 8),
    ("ddim", "epsilon", 4, 3, 0, (9, 13), 1.0, None),
    ("ddim", "epsilon", 10, 1, 1, (64, 64), 7.5, 8),
    ("ddim", "v_prediction", 4, 1, 1, (9, 13), 15.0, 8),
    ("ddim", "v_prediction", 10, 3, 0, (64, 64), 1.0, 4),
    ("lms", "epsilon", 4, 3, 1, (64, 64), 7.5, 4),
    ("lms", "epsilon", 10, 1, 0, (9, 13), 1.0, 8),
    ("euler", "epsilon", 4, 1, 1, (64, 64), 1.0, None),
    ("euler", "epsilon", 10, 3, 1, (9, 13), 7.5, 8),
    ("dpm", "epsilon", 4, 3, 1, (9, 13), 15.0, 4),
    ("dpm", "epsilon", 10, 1, 0, (64, 64), 7.5, 8),
]


@pytest.mark.parametrize("name,pred,steps,F,has_uncond,hw,guidance,cpad", CASES)
def test_cfg_sched_step_follows_scheduler_plans(name, pred, steps, F, has_uncond, hw, guidance, cpad):
    n = _n()
    lib = n.lib()
    H, W = hw
    sch = _scheduler(name, pred)
    sch.set_timesteps(steps)
    plan = sch.plan()
    rng = np.random.default_rng(sum(map(ord, name + pred)) * 100 + steps)
    x = torch.from_numpy((rng.standard_normal((F, LAT_C, H, W)) * sch.init_noise_sigma).astype(np.float32)).cuda()
    x_base = torch.full_like(x, float("nan"))
    hist = torch.full((4,) + tuple(x.shape), float("nan"), device="cuda")  # slots are read only after being written
    Bn = 2 * F if has_uncond else F
    for i in range(len(plan)):
        k = _coef(plan, i, guidance)
        # uncond and cond predictions differ by a small fraction, as a UNet's do
        u = rng.standard_normal((F, H, W, LAT_C))
        eps = np.concatenate([u, u + 0.2 * rng.standard_normal(u.shape)]) if has_uncond else u
        eps = eps.astype(np.float32)
        last = i + 1 == len(plan)
        nxt = None
        if cpad is not None and not last:
            nxt = torch.full((Bn, H, W, cpad), -3.5, dtype=torch.float16, device="cuda")
            nxt[..., :LAT_C] = float("nan")
        before = [t.cpu().numpy() for t in (x, x_base, hist)]
        eps_d = torch.from_numpy(eps).cuda()
        n.check(lib.sdw_cfg_sched_step(_p(eps_d), has_uncond, _p(x), _p(x_base), _p(hist), C.byref(k), F, LAT_C, H, W,
                                       _p(nxt), cpad or LAT_C, n.stream_ptr()))
        torch.cuda.synchronize()
        rx, rb, rh, mag, push_mag = _ref_step(k, eps, has_uncond, F, *before)
        scale = max(mag, _amax(before[0]), _amax(rx))
        gx, gb, gh = x.cpu().numpy(), x_base.cpu().numpy(), hist.cpu().numpy()
        assert _close(gx, rx, scale), (i, "x", float(np.abs(gx - rx).max()), scale)
        assert _close(gb, rb, scale), (i, "x_base")
        for j in range(4):
            assert _close(gh[j], rh[j], max(scale, push_mag)), (i, "hist", j)
        if nxt is not None:
            want = (x * k.next_in_scale).half().permute(0, 2, 3, 1)  # fp16(x' * next_in_scale), NHWC
            got = nxt[..., :LAT_C]
            assert torch.equal(got[:F].view(torch.int16), want.view(torch.int16)), i
            if has_uncond:
                assert torch.equal(got[F:].view(torch.int16), got[:F].view(torch.int16)), i
            assert bool((nxt[..., LAT_C:] == -3.5).all())


def test_cfg_sched_step_rejects_bad_slots():
    """a history slot or push slot of 4 is refused on the host (rc 1) and nothing is launched"""
    n = _n()
    lib = n.lib()
    F, H, W = 1, 4, 4
    x = torch.ones(F, LAT_C, H, W, device="cuda")
    xb, hist = torch.zeros_like(x), torch.zeros((4,) + tuple(x.shape), device="cuda")
    eps = torch.zeros(F, H, W, LAT_C, device="cuda")
    for field in ("hist_slot", "push_slot"):
        k = n.StepCoef()
        k.guidance, k.c_x, k.push_slot = 1.0, 2.0, -1
        if field == "hist_slot":
            k.hist_slot[2] = 4
        else:
            k.push_slot = 4
        rc = lib.sdw_cfg_sched_step(_p(eps), 0, _p(x), _p(xb), _p(hist), C.byref(k), F, LAT_C, H, W, C.c_void_p(0),
                                    LAT_C, n.stream_ptr())
        torch.cuda.synchronize()
        assert rc == 1, field
        assert b"slot" in lib.sdw_last_error()
        assert bool((x == 1).all())


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("dup", [0, 1])
@pytest.mark.parametrize("cpad", [None, 4, 8])
def test_latents_init(dtype, dup, cpad):
    n = _n()
    F, H, W = 3, 9, 13
    g = torch.Generator().manual_seed(11)
    lat = torch.randn(F, LAT_C, H, W, generator=g).to(dtype).cuda()
    sigma, in_scale = 14.614642, 0.06826489  # the K-LMS init_noise_sigma and its first input scale
    x = torch.full((F, LAT_C, H, W), float("nan"), device="cuda")
    Bn = 2 * F if dup else F
    mi = None
    if cpad is not None:
        mi = torch.full((Bn, H, W, cpad), -3.5, dtype=torch.float16, device="cuda")
        mi[..., :LAT_C] = float("nan")
    n.check(n.lib().sdw_latents_init(_p(lat), int(dtype == torch.float16), C.c_float(sigma), C.c_float(in_scale), _p(x),
                                     _p(mi), cpad or LAT_C, dup, F, LAT_C, H, W, n.stream_ptr()))
    torch.cuda.synchronize()
    want = lat.float() * float(np.float32(sigma))  # one fp32 multiply
    assert torch.equal(x, want)
    if mi is not None:
        m = (x * float(np.float32(in_scale))).half().permute(0, 2, 3, 1)
        assert torch.equal(mi[:F, ..., :LAT_C].view(torch.int16), m.view(torch.int16))
        if dup:
            assert torch.equal(mi[F:, ..., :LAT_C].view(torch.int16), m.view(torch.int16))
        assert bool((mi[..., LAT_C:] == -3.5).all())
