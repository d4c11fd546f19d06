"""Host-side scheduler descriptors for the native sampler.

The reference drives a diffusers scheduler object through `set_timesteps`, `timesteps`, `init_noise_sigma`,
`scale_model_input` and `step` (stable_diffusion_pipeline.py:394-426).  Every scheduler it accepts that is
deterministic (PNDM/PLMS — the SD-1.4 default, DDIM with eta = 0 — the SD-2.1 default, LMS —
examples/make_music_video.py:15-17, Euler) is a LINEAR multistep rule, so here `set_timesteps` pre-computes, in fp64 on
the host, one `sdw_step_coef` per step (include/sdwalk.h); the update itself runs in one fused fp32 CUDA kernel
together with classifier-free guidance.  The stochastic members (DDIM with eta > 0, Euler ancestral) are the same rules
plus `c_z` times fresh Gaussian noise, generated inside that kernel from per-frame keys (noise.py).
`beta_schedule="scaled_linear"`, `steps_offset=1`, `set_alpha_to_one=False`, `clip_sample=False` as the reference forces
(stable_diffusion_pipeline.py:85-110).
"""
from types import SimpleNamespace

import math

import numpy as np


def _alphas_cumprod(beta_start, beta_end, n):
    # diffusers builds the table in fp32: linspace(sqrt(b0), sqrt(b1), n) ** 2, cumprod — keep its rounding
    import torch

    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, n, dtype=torch.float32) ** 2
    return torch.cumprod(1.0 - betas, dim=0).double().numpy()


class _Base:
    order = 1

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                 prediction_type="epsilon", steps_offset=1, **unused):
        if beta_schedule != "scaled_linear":
            raise ValueError("only beta_schedule='scaled_linear' (the Stable Diffusion schedule) is supported")
        self.config = SimpleNamespace(num_train_timesteps=num_train_timesteps, beta_start=beta_start,
                                      beta_end=beta_end, beta_schedule=beta_schedule,
                                      prediction_type=prediction_type, steps_offset=steps_offset,
                                      clip_sample=False, set_alpha_to_one=False)
        self.alphas_cumprod = _alphas_cumprod(beta_start, beta_end, num_train_timesteps)
        self.final_alpha_cumprod = self.alphas_cumprod[0]
        self.init_noise_sigma = 1.0
        self.timesteps = None
        self.num_inference_steps = None

    # the native plan: list of dict(c_x, c_e[5], hist_slot[4], use_x_base, save_x_base, push_slot, in_scale), plus the
    # optional push_e / push_x (history contents) and c_z (noise coefficient, 0 when absent)
    def plan(self):
        raise NotImplementedError

    def scale_model_input(self, sample, timestep=None):
        return sample

    def _eps_coeffs(self, a_t, a_p):
        """x_prev = cx * x + ce * eps for the PNDM `_get_prev_sample` transfer formula."""
        b_t, b_p = 1 - a_t, 1 - a_p
        cx = (a_p / a_t) ** 0.5
        denom = a_t * b_p ** 0.5 + (a_t * b_t * a_p) ** 0.5
        return cx, -(a_p - a_t) / denom


class PNDMScheduler(_Base):
    """PLMS (skip_prk_steps=True): N+1 UNet calls for N steps (the second timestep is visited twice)."""

    def __init__(self, skip_prk_steps=True, **kw):
        super().__init__(**kw)
        if not skip_prk_steps:
            raise ValueError("the Runge-Kutta warm-up (skip_prk_steps=False) is not implemented; SD uses PLMS")
        if self.config.prediction_type != "epsilon":
            raise ValueError("PNDM native plan supports epsilon prediction")
        self.config.skip_prk_steps = True

    def set_timesteps(self, n, device=None):
        self.num_inference_steps = n
        r = self.config.num_train_timesteps // n
        ts = (np.arange(0, n) * r).round() + self.config.steps_offset
        self.timesteps = np.concatenate([ts[:-1], ts[-2:-1], ts[-1:]])[::-1].copy().astype(np.int64)

    def plan(self):
        n = self.num_inference_steps
        r = self.config.num_train_timesteps // n
        ac = self.alphas_cumprod
        steps = []
        ring = []  # slots of stored eps, oldest first (max 4 incl. current)
        next_slot = 0
        for counter, t in enumerate(self.timesteps):
            t = int(t)
            prev = t - r
            st = dict(c_x=0.0, c_e=[0.0] * 5, hist_slot=[0, 0, 0, 0], use_x_base=0, save_x_base=0, push_slot=-1)
            if counter != 1:
                ring = ring[-3:]
                slot = next_slot
                next_slot = (next_slot + 1) % 4
                ring.append(slot)
                st["push_slot"] = slot
            else:
                prev, t = t, t + r
            a_t = ac[t]
            a_p = ac[prev] if prev >= 0 else self.final_alpha_cumprod
            cx, ce = self._eps_coeffs(a_t, a_p)
            st["c_x"] = cx
            if len(ring) == 1 and counter == 0:
                w = [1.0]
                st["save_x_base"] = 1
            elif len(ring) == 1 and counter == 1:
                # e' = (e + ets[-1]) / 2 with e the CURRENT (un-pushed) output
                st["c_e"][0] = ce * 0.5
                st["c_e"][1] = ce * 0.5
                st["hist_slot"][0] = ring[-1]
                st["use_x_base"] = 1
                steps.append(st)
                continue
            elif len(ring) == 2:
                w = [3 / 2, -1 / 2]
            elif len(ring) == 3:
                w = [23 / 12, -16 / 12, 5 / 12]
            else:
                w = [55 / 24, -59 / 24, 37 / 24, -9 / 24]
            # w[0] multiplies the current eps (just pushed), w[k] the k-th previous one
            st["c_e"][0] = ce * w[0]
            for k in range(1, len(w)):
                st["c_e"][k] = ce * w[k]
                st["hist_slot"][k - 1] = ring[-1 - k]
            steps.append(st)
        for st in steps:
            st["in_scale"] = 1.0
        return steps


class DDIMScheduler(_Base):
    def set_timesteps(self, n, device=None):
        self.num_inference_steps = n
        r = self.config.num_train_timesteps // n
        self.timesteps = ((np.arange(0, n) * r).round()[::-1].copy() + self.config.steps_offset).astype(np.int64)

    def plan(self, eta=0.0):
        """diffusers' DDIM step with use_clipped_model_output=False:
            sigma = eta sqrt((1 - a_p) / (1 - a_t) (1 - a_t / a_p)),  D = sqrt(1 - a_p - sigma^2)
            epsilon      : c_x = sqrt(a_p / a_t),                  c_e = D - sqrt(a_p (1 - a_t) / a_t)
            v_prediction : c_x = sqrt(a_p a_t) + D sqrt(1 - a_t),  c_e = D sqrt(a_t) - sqrt(a_p (1 - a_t))
        and c_z = sigma on the step noise.  D^2 stays under the square roots so that eta = 0 gives the same floats as
        the deterministic form."""
        eta = float(eta)
        if not 0.0 <= eta <= 1.0:
            raise ValueError(f"DDIM eta must lie in [0, 1], got {eta}")
        n = self.num_inference_steps
        r = self.config.num_train_timesteps // n
        ac = self.alphas_cumprod
        steps = []
        for t in self.timesteps:
            t = int(t)
            prev = t - r
            a_t = ac[t]
            a_p = ac[prev] if prev >= 0 else self.final_alpha_cumprod
            sigma = eta * ((1 - a_p) / (1 - a_t) * (1 - a_t / a_p)) ** 0.5 if eta else 0.0
            d2 = 1 - a_p - sigma * sigma
            if self.config.prediction_type == "epsilon":
                cx = (a_p / a_t) ** 0.5
                ce = d2 ** 0.5 - (a_p * (1 - a_t) / a_t) ** 0.5
            elif self.config.prediction_type == "v_prediction":
                cx = (a_p * a_t) ** 0.5 + (d2 * (1 - a_t)) ** 0.5
                ce = (d2 * a_t) ** 0.5 - (a_p * (1 - a_t)) ** 0.5
            else:
                raise ValueError(self.config.prediction_type)
            steps.append(dict(c_x=cx, c_e=[ce, 0, 0, 0, 0], hist_slot=[0, 0, 0, 0], use_x_base=0, save_x_base=0,
                              push_slot=-1, in_scale=1.0, c_z=float(sigma)))
        return steps


class LMSDiscreteScheduler(_Base):
    """K-LMS, order 4.  derivative = (x - x0) / sigma = eps for epsilon prediction, so the update is
    x' = x + sum_k coeff_k * eps_{i-k}; scale_model_input divides the UNet input by sqrt(sigma^2 + 1)."""

    def __init__(self, **kw):
        super().__init__(**kw)
        if self.config.prediction_type != "epsilon":
            raise ValueError("LMS native plan supports epsilon prediction")
        ac = self.alphas_cumprod
        sig = ((1 - ac) / ac) ** 0.5
        self.init_noise_sigma = float(np.concatenate([sig[::-1], [0.0]]).astype(np.float32).max())

    def set_timesteps(self, n, device=None):
        self.num_inference_steps = n
        nt = self.config.num_train_timesteps
        ts = np.linspace(0, nt - 1, n, dtype=float)[::-1].copy()
        ac = self.alphas_cumprod
        sig = ((1 - ac) / ac) ** 0.5
        sig = np.interp(ts, np.arange(0, len(sig)), sig)
        self.sigmas = np.concatenate([sig, [0.0]]).astype(np.float32)
        self.timesteps = ts

    def _coef(self, order, t, cur):
        from scipy import integrate

        def f(tau):
            prod = 1.0
            for k in range(order):
                if cur == k:
                    continue
                prod *= (tau - self.sigmas[t - k]) / (self.sigmas[t - cur] - self.sigmas[t - k])
            return prod

        return integrate.quad(f, self.sigmas[t], self.sigmas[t + 1], epsrel=1e-4)[0]

    def scale_model_input(self, sample, timestep=None):
        i = int(np.nonzero(self.timesteps == float(timestep))[0][0])
        return sample / ((float(self.sigmas[i]) ** 2 + 1) ** 0.5)

    def plan(self):
        steps = []
        for i in range(self.num_inference_steps):
            order = min(i + 1, 4)
            coeffs = [self._coef(order, i, k) for k in range(order)]
            st = dict(c_x=1.0, c_e=[0.0] * 5, hist_slot=[0, 0, 0, 0], use_x_base=0, save_x_base=0, push_slot=i % 4)
            st["c_e"][0] = coeffs[0]
            for k in range(1, order):
                st["c_e"][k] = coeffs[k]
                st["hist_slot"][k - 1] = (i - k) % 4
            st["in_scale"] = 1.0 / ((float(self.sigmas[i]) ** 2 + 1) ** 0.5)
            steps.append(st)
        return steps


class EulerDiscreteScheduler(_Base):
    """Euler (Karras et al. 2022, Alg. 2 with s_churn = 0 — the deterministic form the reference's scheduler union
    accepts, stable_diffusion_pipeline.py:71-78).  derivative = (x - x0) / sigma, x' = x + (sigma_next - sigma) * derivative:
      epsilon      : derivative = eps                                   -> c_x = 1,                       c_e = dt
      v_prediction : x0 = -sigma/sqrt(sigma^2+1) * v + x / (sigma^2+1)  -> c_x = 1 + dt*sigma/(sigma^2+1), c_e = dt/sqrt(sigma^2+1)
    Same sigma table / linspace timesteps / input scaling as K-LMS."""

    def __init__(self, **kw):
        super().__init__(**kw)
        if self.config.prediction_type not in ("epsilon", "v_prediction"):
            raise ValueError("Euler native plan supports epsilon and v_prediction")
        ac = self.alphas_cumprod
        sig = ((1 - ac) / ac) ** 0.5
        self.init_noise_sigma = float(np.concatenate([sig[::-1], [0.0]]).astype(np.float32).max())

    def set_timesteps(self, n, device=None):
        self.num_inference_steps = n
        nt = self.config.num_train_timesteps
        ts = np.linspace(0, nt - 1, n, dtype=float)[::-1].copy()
        ac = self.alphas_cumprod
        sig = ((1 - ac) / ac) ** 0.5
        sig = np.interp(ts, np.arange(0, len(sig)), sig)
        self.sigmas = np.concatenate([sig, [0.0]]).astype(np.float32)
        self.timesteps = ts

    def scale_model_input(self, sample, timestep=None):
        i = int(np.nonzero(self.timesteps == float(timestep))[0][0])
        return sample / ((float(self.sigmas[i]) ** 2 + 1) ** 0.5)

    def plan(self):
        steps = []
        for i in range(self.num_inference_steps):
            s, s_next = float(self.sigmas[i]), float(self.sigmas[i + 1])
            dt = s_next - s
            if self.config.prediction_type == "epsilon":
                cx, ce = 1.0, dt
            else:
                cx, ce = 1.0 + dt * s / (s * s + 1.0), dt / (s * s + 1.0) ** 0.5
            steps.append(dict(c_x=cx, c_e=[ce, 0, 0, 0, 0], hist_slot=[0, 0, 0, 0], use_x_base=0, save_x_base=0,
                              push_slot=-1, in_scale=1.0 / (s * s + 1.0) ** 0.5))
        return steps


class EulerAncestralDiscreteScheduler(EulerDiscreteScheduler):
    """Euler ancestral (Karras et al. 2022 with ancestral sampling; diffusers' EulerAncestralDiscreteScheduler): each step
    goes to sigma_down with the Euler rule, then adds fresh noise of standard deviation sigma_up,
        sigma_up = sqrt(sigma_next^2 (sigma^2 - sigma_next^2) / sigma^2),  sigma_down = sqrt(sigma_next^2 - sigma_up^2),
    so x' = c_x x + c_e e + sigma_up z with Euler's coefficients at dt = sigma_down - sigma.  Same sigma table, timesteps,
    init_noise_sigma and input scaling as Euler; sigma_up = 0 on the last step."""

    def plan(self):
        steps = []
        for i in range(self.num_inference_steps):
            s, s_next = float(self.sigmas[i]), float(self.sigmas[i + 1])
            s_up = (s_next ** 2 * (s ** 2 - s_next ** 2) / s ** 2) ** 0.5
            s_down = (s_next ** 2 - s_up ** 2) ** 0.5
            dt = s_down - s
            if self.config.prediction_type == "epsilon":
                cx, ce = 1.0, dt
            else:
                cx, ce = 1.0 + dt * s / (s * s + 1.0), dt / (s * s + 1.0) ** 0.5
            steps.append(dict(c_x=cx, c_e=[ce, 0, 0, 0, 0], hist_slot=[0, 0, 0, 0], use_x_base=0, save_x_base=0,
                              push_slot=-1, in_scale=1.0 / (s * s + 1.0) ** 0.5, c_z=s_up))
        return steps


class DPMSolverMultistepScheduler(_Base):
    """DPM-Solver++ (2M), the diffusers default configuration (algorithm_type "dpmsolver++", solver_order 2,
    solver_type "midpoint", lower_order_final=True, no thresholding): a two-step linear multistep rule on the DATA
    prediction x0 = (x - sigma_t eps) / alpha_t.  The native step keeps x0 in the history ring (push_e, push_x) and the
    update is again  x' = c_x x + c_e0 eps + c_e1 hist:
        first order :  x' = (s_p/s_t) x - a_p (e^-h - 1) x0_t
        second order:  x' = (s_p/s_t) x - a_p (e^-h - 1) [ (1 + 1/(2r)) x0_t - 1/(2r) x0_prev ],   r = h_prev / h
    with a = sqrt(abar), s = sqrt(1 - abar), lambda = ln(a/s), h = lambda_p - lambda_t (scheduler union P:71-78)."""
    order = 2

    def __init__(self, solver_order=2, lower_order_final=True, **kw):
        super().__init__(**kw)
        if solver_order not in (1, 2):
            raise ValueError("DPM-Solver++ native plan: solver_order 1 or 2")
        self.config.solver_order, self.config.lower_order_final = solver_order, lower_order_final

    def set_timesteps(self, n, device=None):
        self.num_inference_steps = n
        T = self.config.num_train_timesteps
        self.timesteps = np.linspace(0, T - 1, n + 1).round()[::-1][:-1].copy().astype(np.int64)

    def plan(self):
        ac = self.alphas_cumprod
        ts = [int(t) for t in self.timesteps]
        n = len(ts)
        lam = lambda a: 0.5 * (math.log(a) - math.log(1.0 - a))  # noqa: E731
        steps = []
        for i, t in enumerate(ts):
            prev = ts[i + 1] if i + 1 < n else 0
            a_t, a_p = float(ac[t]), float(ac[prev])
            al_t, si_t, al_p, si_p = a_t ** 0.5, (1 - a_t) ** 0.5, a_p ** 0.5, (1 - a_p) ** 0.5
            h = lam(a_p) - lam(a_t)
            g = -al_p * math.expm1(-h)  # coefficient on the (combined) data prediction
            first = (self.config.solver_order == 1 or i == 0
                     or (i == n - 1 and self.config.lower_order_final and n < 15))
            if first:
                w_cur, w_old = 1.0, 0.0
            else:
                h_prev = lam(a_t) - lam(float(ac[ts[i - 1]]))
                r = h_prev / h
                w_cur, w_old = 1.0 + 0.5 / r, -0.5 / r
            # x0_t = x / al_t - (si_t / al_t) eps
            st = dict(c_x=si_p / si_t + g * w_cur / al_t, c_e=[-g * w_cur * si_t / al_t, g * w_old, 0.0, 0.0, 0.0],
                      hist_slot=[(i - 1) & 1, 0, 0, 0], use_x_base=0, save_x_base=0, push_slot=i & 1,
                      push_e=-si_t / al_t, push_x=1.0 / al_t, in_scale=1.0)
            steps.append(st)
        return steps


SCHEDULERS = {"dpm": DPMSolverMultistepScheduler, "pndm": PNDMScheduler, "ddim": DDIMScheduler, "lms": LMSDiscreteScheduler,
              "euler": EulerDiscreteScheduler, "euler_a": EulerAncestralDiscreteScheduler}


def accepts_eta(scheduler):
    """whether the scheduler's plan takes `eta` (DDIM), as the reference asks of `scheduler.step` (P:404-410)"""
    import inspect

    return "eta" in inspect.signature(scheduler.plan).parameters


def check_eta(scheduler, eta):
    """eta is a DDIM parameter in [0, 1]; the other schedulers ignore it, as in the reference"""
    if accepts_eta(scheduler) and not 0.0 <= float(eta) <= 1.0:
        raise ValueError(f"DDIM eta must lie in [0, 1], got {eta}")
