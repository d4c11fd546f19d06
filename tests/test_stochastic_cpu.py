"""Stochastic samplers on the host: the step-noise generator's specification (Philox4x32-10 known answers, uniforms),
the DDIM (eta > 0) and Euler-ancestral coefficient plans replayed against stateful restatements of diffusers' steps,
and the per-frame key / weight tables the pipeline builds."""
import math

import numpy as np
import pytest
import torch

import _stochastic_oracle as O

RANDOM123_KAT = [  # Random123 kat_vectors, philox4x32_10
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]


@pytest.mark.parametrize("ctr,key,want", RANDOM123_KAT)
def test_philox_known_answers(ctr, key, want):
    assert tuple(int(w) for w in O.philox4x32_10(ctr, key)) == want


def test_uniforms_are_exact_in_fp32_and_strictly_inside_the_unit_interval():
    b = np.array([0, 1, 511, 512, 2 ** 31, 2 ** 32 - 512, 2 ** 32 - 1], dtype=np.uint64)
    u = O.uniform(b)
    assert (u > 0).all() and (u < 1).all()
    assert np.array_equal(u.astype(np.float32).astype(np.float64), u)  # what the kernel computes in fp32
    assert np.float32(u[-1]) < 1 and np.float32(u[0]) > 0


def _sched(kind, pred, steps):
    from stable_diffusion_videos_b200 import schedulers as S

    s = S.SCHEDULERS[kind](prediction_type=pred)
    s.set_timesteps(steps)
    return s


def _old_ddim_plan(s):
    """the deterministic DDIM coefficients of the parent implementation"""
    r = s.config.num_train_timesteps // s.num_inference_steps
    out = []
    for t in s.timesteps:
        t = int(t)
        a_t = s.alphas_cumprod[t]
        a_p = s.alphas_cumprod[t - r] if t - r >= 0 else s.final_alpha_cumprod
        if s.config.prediction_type == "epsilon":
            out.append(((a_p / a_t) ** 0.5, (1 - a_p) ** 0.5 - (a_p * (1 - a_t) / a_t) ** 0.5))
        else:
            out.append(((a_p * a_t) ** 0.5 + ((1 - a_p) * (1 - a_t)) ** 0.5,
                        ((1 - a_p) * a_t) ** 0.5 - (a_p * (1 - a_t)) ** 0.5))
    return out


@pytest.mark.parametrize("pred", ["epsilon", "v_prediction"])
@pytest.mark.parametrize("steps", [50, 7])
def test_ddim_eta0_plan_is_the_deterministic_plan(pred, steps):
    s = _sched("ddim", pred, steps)
    for plan in (s.plan(), s.plan(eta=0.0)):
        assert [(st["c_x"], st["c_e"][0]) for st in plan] == _old_ddim_plan(s)  # the same floats
        assert all(st["c_z"] == 0.0 for st in plan)


def _replay(kind, pred, steps, eta=None, seed=0, tol=1e-12):
    """x' = c_x x + c_e e + c_z z from the plan against the oracle's stateful step with the same noise (fp64)"""
    s = _sched(kind, pred, steps)
    plan = s.plan(eta=eta) if eta is not None else s.plan()
    ref = O.make_scheduler(kind, pred)
    ref.set_timesteps(steps)
    rng = np.random.default_rng(seed)
    x = torch.from_numpy(rng.standard_normal((2, 4, 3, 5)) * ref.init_noise_sigma)
    xr = x.clone()
    for i, t in enumerate(ref.timesteps):
        e = torch.from_numpy(rng.standard_normal(x.shape))
        z = torch.from_numpy(rng.standard_normal(x.shape))
        st = plan[i]
        x = st["c_x"] * x + st["c_e"][0] * e + st["c_z"] * z
        if kind == "ddim":
            xr = ref.step(e, t, xr, eta=eta, variance_noise=z)
        else:
            xr = ref.step(e, t, xr, noise=z)
        err = float((x - xr).abs().max() / max(1.0, float(xr.abs().max())))
        assert err <= tol, (i, err)
    return plan, s


@pytest.mark.parametrize("pred", ["epsilon", "v_prediction"])
@pytest.mark.parametrize("steps", [50, 7])
@pytest.mark.parametrize("eta", [0.5, 1.0])
def test_ddim_plan_replays_the_stochastic_ddim_step(pred, steps, eta):
    plan, _ = _replay("ddim", pred, steps, eta=eta, seed=steps)
    assert all(st["c_z"] > 0 for st in plan[:-1])


@pytest.mark.parametrize("steps", [50, 7])
def test_ddim_eta1_noise_is_the_ddpm_posterior_variance(steps):
    s = _sched("ddim", "epsilon", steps)
    r = 1000 // steps
    for t, st in zip(s.timesteps, s.plan(eta=1.0)):
        t = int(t)
        a_t = s.alphas_cumprod[t]
        a_p = s.alphas_cumprod[t - r] if t - r >= 0 else s.final_alpha_cumprod
        beta = 1 - a_t / a_p  # the strided schedule's beta_t
        assert math.isclose(st["c_z"] ** 2, (1 - a_p) / (1 - a_t) * beta, rel_tol=1e-12, abs_tol=1e-300)


@pytest.mark.parametrize("eta", [-0.1, 1.5])
def test_ddim_rejects_eta_outside_the_unit_interval(eta):
    from stable_diffusion_videos_b200.schedulers import check_eta

    s = _sched("ddim", "epsilon", 10)
    with pytest.raises(ValueError, match="eta"):
        s.plan(eta=eta)
    with pytest.raises(ValueError, match="eta"):
        check_eta(s, eta)
    check_eta(_sched("euler", "epsilon", 10), eta)  # the other schedulers ignore eta, as in the reference


@pytest.mark.parametrize("pred", ["epsilon", "v_prediction"])
@pytest.mark.parametrize("steps", [50, 7])
def test_euler_ancestral_plan_replays_the_ancestral_step(pred, steps):
    # the oracle's sigma table is computed in fp32 before its final rounding (oracle/schedulers.py), the plan's in
    # fp64: an ulp of fp32 between them
    plan, s = _replay("euler_a", pred, steps, seed=100 + steps, tol=1e-6)
    for i, st in enumerate(plan):
        sg, sn = float(s.sigmas[i]), float(s.sigmas[i + 1])
        s_down = st["c_e"][0] + sg if pred == "epsilon" else None
        if s_down is not None:
            assert math.isclose(st["c_z"] ** 2 + s_down ** 2, sn ** 2, rel_tol=1e-9, abs_tol=1e-12)
    assert plan[-1]["c_z"] == 0.0 and all(st["c_z"] > 0 for st in plan[:-1])
    # same timesteps, init_noise_sigma and input scaling as Euler
    e = _sched("euler", pred, steps)
    assert np.array_equal(s.timesteps, e.timesteps) and s.init_noise_sigma == e.init_noise_sigma
    assert [st["in_scale"] for st in plan] == [st["in_scale"] for st in e.plan()]


def test_walk_table_endpoints_and_keys():
    from stable_diffusion_videos_b200 import noise

    T = np.linspace(0.0, 1.0, 7)
    seed_a, seed_b = 9_000_000_123, 2 ** 63 + 5  # the reference example draws seeds up to 9e9
    tab = noise.as_numpy(noise.walk_table(T, seed_a, seed_b))
    assert (tab["key_a"] == seed_a).all() and (tab["key_b"] == seed_b).all()
    assert (tab["w_a"][0], tab["w_b"][0]) == (1.0, 0.0) and (tab["w_a"][-1], tab["w_b"][-1]) == (0.0, 1.0)
    np.testing.assert_allclose(tab["w_a"] ** 2 + tab["w_b"] ** 2, 1.0, rtol=1e-6)
    want = O.walk_table(T, seed_a, seed_b)
    assert [tuple(r) for r in tab.tolist()] == want
    assert noise.as_numpy(noise.walk_table([0.5], -1, 0))["key_a"][0] == 2 ** 64 - 1  # seed mod 2^64
    pad = noise.as_numpy(noise.pad_table(noise.walk_table(T[:2], 1, 2), 4))
    assert pad.tolist()[2] == pad.tolist()[1] == pad.tolist()[3]


class _FakeEngine:
    def __init__(self, stochastic):
        self.stochastic, self.tables = stochastic, []

    def set_frame_noise(self, table):
        self.tables.append(table)


def _cpu_pipe(stochastic):
    """a pipeline whose engine is replaced by a recorder: exercises __call__'s host logic without a GPU"""
    from stable_diffusion_videos_b200.configs import UNetConfig, VAEConfig
    from stable_diffusion_videos_b200.pipeline import (NativeUNet, NativeVAE, StableDiffusionWalkPipeline,
                                                       SyntheticTextEncoder, SyntheticTokenizer)
    from stable_diffusion_videos_b200.schedulers import DDIMScheduler

    pipe = StableDiffusionWalkPipeline(NativeVAE(VAEConfig(), {}), SyntheticTextEncoder(64), SyntheticTokenizer(),
                                       NativeUNet(UNetConfig(cross_attention_dim=64, sample_size=8), {}), DDIMScheduler())
    eng = _FakeEngine(stochastic)
    pipe._prepare = lambda *a, **k: eng
    pipe._sample_device = lambda lat, *a, **k: (torch.zeros((lat.shape[0], 8, 8, 3), dtype=torch.uint8), None)
    return pipe, eng


@pytest.mark.parametrize("stochastic", [False, True])
def test_call_draws_keys_only_for_a_stochastic_schedule(stochastic):
    from stable_diffusion_videos_b200 import noise

    pipe, eng = _cpu_pipe(stochastic)
    g = torch.Generator().manual_seed(7)
    pipe(prompt=["0", "1", "2"], height=64, width=64, num_inference_steps=2, eta=1.0 if stochastic else 0.0,
         generator=g)
    g_ref = torch.Generator().manual_seed(7)
    torch.randn((3, 4, 8, 8), generator=g_ref, dtype=torch.float16)  # the latents come first
    if stochastic:
        want = O.call_table(3, g_ref, "cpu")
        assert len(eng.tables) == 1 and [tuple(r) for r in noise.as_numpy(eng.tables[0]).tolist()] == want
    else:
        assert eng.tables == []
    assert torch.equal(g.get_state(), g_ref.get_state())  # exactly the RNG the call consumed before
    with pytest.raises(ValueError, match="eta"):
        pipe(prompt="0", height=64, width=64, eta=1.5)


def test_from_pretrained_names_the_euler_ancestral_route(tmp_path):
    import _fake_checkpoint as fc
    from stable_diffusion_videos_b200.pipeline import StableDiffusionWalkPipeline

    fc.write_checkpoint(str(tmp_path), scheduler="EulerAncestralDiscreteScheduler", with_weights=False)
    with pytest.raises(NotImplementedError, match="pipe.scheduler = EulerAncestralDiscreteScheduler"):
        StableDiffusionWalkPipeline.from_pretrained(str(tmp_path))
