"""ORACLE (test infrastructure only) of the stochastic samplers: an independent numpy restatement of the step noise
specified in include/sdwalk.h (sdw_frame_noise) and stateful restatements of diffusers' stochastic steps that take their
noise as an argument.

  Philox4x32-10 (Salmon et al., SC'11) in uint64 arithmetic, uniforms ((b >> 9) + 1/2) 2^-23, Box-Muller in float64;
  frame mixing w_a Z(key_a) + w_b Z(key_b) with the fp32 weights the device table holds;
  walk weights (cos(pi T / 2), sin(pi T / 2)), exact at T = 0 / 1; __call__ keys: one non-negative int64 per image;
  DDIMScheduler.step(..., eta, variance_noise) and EulerAncestralDiscreteScheduler.step(..., noise) restated from
  diffusers' published code (DDIM: use_clipped_model_output=False; Euler ancestral: sigma_up / sigma_down).
"""
import math

import numpy as np
import torch

from oracle import schedulers as _S
from oracle.pipeline import to_uint8

M32 = np.uint64(0xFFFFFFFF)
TAG = 0x5344574E


def philox4x32_10(ctr, key):
    """ctr: four uint32 arrays (or scalars), key: two; returns the four output words as uint64 arrays"""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & M32 for c in ctr)
    k0, k1 = (np.asarray(k, dtype=np.uint64) & M32 for k in key)
    for r in range(10):
        if r:
            k0 = (k0 + np.uint64(0x9E3779B9)) & M32
            k1 = (k1 + np.uint64(0xBB67AE85)) & M32
        p0 = c0 * np.uint64(0xD2511F53)  # 32 x 32 -> 64 bits, exact in uint64
        p1 = c2 * np.uint64(0xCD9E8D57)
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & M32
    return c0, c1, c2, c3


def uniform(b):
    return ((np.asarray(b, dtype=np.uint64) >> np.uint64(9)).astype(np.float64) + 0.5) * 2.0 ** -23


def normal_field(key, step, n):
    """Z(key, step, i) for i < n (n a multiple of 4), float64"""
    key = int(key) & ((1 << 64) - 1)
    g = np.arange(n // 4, dtype=np.uint64)
    x = philox4x32_10((g, step, TAG, 0), (key & 0xFFFFFFFF, key >> 32))
    u = [uniform(w) for w in x]
    z = np.empty((n // 4, 4))
    for j in (0, 2):
        r = np.sqrt(-2.0 * np.log(u[j]))
        z[:, j] = r * np.cos(2 * np.pi * u[j + 1])
        z[:, j + 1] = r * np.sin(2 * np.pi * u[j + 1])
    return z.reshape(-1)


def frame_noise(entry, step, shape):
    """noise of one frame: entry = (key_a, key_b, w_a, w_b), shape = (C, H, W)"""
    ka, kb, wa, wb = entry
    n = int(np.prod(shape))
    z = np.zeros(n)
    if wa != 0:
        z += float(np.float32(wa)) * normal_field(ka, step, n)
    if wb != 0:
        z += float(np.float32(wb)) * normal_field(kb, step, n)
    return z.reshape(shape)


def batch_noise(table, step, shape):
    return np.stack([frame_noise(e, step, shape) for e in table])


def walk_table(T, seed_a, seed_b):
    out = []
    for t in T:
        t = float(t)
        wa, wb = (1.0, 0.0) if t == 0 else (0.0, 1.0) if t == 1 else (math.cos(math.pi * t / 2), math.sin(math.pi * t / 2))
        out.append((int(seed_a) % 2 ** 64, int(seed_b) % 2 ** 64, float(np.float32(wa)), float(np.float32(wb))))
    return out


def call_table(n, generator, device):
    keys = torch.randint(0, 2 ** 63 - 1, (n,), generator=generator, device=device, dtype=torch.int64).tolist()
    return [(k, k, 1.0, 0.0) for k in keys]


class DDIMScheduler(_S.DDIMScheduler):
    def step(self, model_output, timestep, sample, eta=0.0, variance_noise=None):
        timestep = int(timestep)
        prev = timestep - self.n_train // self.num_inference_steps
        a_t = float(self.alphas_cumprod[timestep])
        a_p = float(self.alphas_cumprod[prev] if prev >= 0 else self.final_alpha_cumprod)
        b_t = 1 - a_t
        if self.prediction_type == "epsilon":
            x0, e = (sample - b_t ** 0.5 * model_output) / a_t ** 0.5, model_output
        else:
            x0 = a_t ** 0.5 * sample - b_t ** 0.5 * model_output
            e = a_t ** 0.5 * model_output + b_t ** 0.5 * sample
        variance = ((1 - a_p) / b_t) * (1 - a_t / a_p)
        std = eta * variance ** 0.5
        prev_sample = a_p ** 0.5 * x0 + (1 - a_p - std ** 2) ** 0.5 * e
        if eta > 0:
            prev_sample = prev_sample + std * variance_noise
        return prev_sample


class EulerAncestralDiscreteScheduler(_S.EulerDiscreteScheduler):
    def step(self, model_output, timestep, sample, noise=None):
        i = self._index(timestep)
        s, s_to = float(self.sigmas[i]), float(self.sigmas[i + 1])
        if self.prediction_type == "epsilon":
            x0 = sample - s * model_output
        else:
            x0 = model_output * (-s / (s ** 2 + 1) ** 0.5) + (sample / (s ** 2 + 1))
        s_up = (s_to ** 2 * (s ** 2 - s_to ** 2) / s ** 2) ** 0.5
        s_down = (s_to ** 2 - s_up ** 2) ** 0.5
        derivative = (sample - x0) / s
        return sample + derivative * (s_down - s) + noise * s_up


def make_scheduler(kind, prediction_type="epsilon"):
    if kind == "ddim":
        return DDIMScheduler(prediction_type=prediction_type)
    if kind == "euler_a":
        return EulerAncestralDiscreteScheduler(prediction_type=prediction_type)
    return _S.make_scheduler(kind, prediction_type)


@torch.no_grad()
def sample_frames(unet, vae, scheduler, latents, text_embeddings, uncond_embeddings, num_inference_steps, guidance_scale,
                  eta=0.0, table=None, return_latents=False):
    """oracle.pipeline.sample_frames with each step's noise drawn from `table` (one entry per frame)"""
    B = text_embeddings.shape[0]
    do_cfg = guidance_scale > 1.0
    if do_cfg:
        text_embeddings = torch.cat([uncond_embeddings.repeat(B, 1, 1), text_embeddings])
    scheduler.set_timesteps(num_inference_steps)
    latents = latents * scheduler.init_noise_sigma
    shape = tuple(latents.shape[1:])
    for i, t in enumerate(scheduler.timesteps):
        x = torch.cat([latents] * 2) if do_cfg else latents
        noise_pred = unet(scheduler.scale_model_input(x, t), t, text_embeddings)
        if do_cfg:
            u, c = noise_pred.chunk(2)
            noise_pred = u + guidance_scale * (c - u)
        z = torch.from_numpy(batch_noise(table, i, shape)).to(latents.dtype) if table is not None else None
        if isinstance(scheduler, DDIMScheduler):
            latents = scheduler.step(noise_pred, t, latents, eta=eta, variance_noise=z)
        elif isinstance(scheduler, EulerAncestralDiscreteScheduler):
            latents = scheduler.step(noise_pred, t, latents, noise=z)
        else:
            latents = scheduler.step(noise_pred, t, latents)
    image = (vae.decode(1 / 0.18215 * latents) / 2 + 0.5).clamp(0, 1).cpu().permute(0, 2, 3, 1).float().numpy()
    return (image, latents) if return_latents else image


def walk_frames(unet, vae, kind, keyframes, embed, uncond, init_latents, num_interpolation_steps, num_inference_steps,
                guidance_scale, eta=0.0, prediction_type="epsilon"):
    """the frames of walk(prompts, seeds) (every clip, every frame) given the keyframe embeddings `embed[k]` and init
    latents `init_latents[k]` ([1, C, h, w] each, float32): uint8 [n, H, W, 3]"""
    from oracle.pipeline import generate_inputs

    out = []
    for k in range(len(keyframes) - 1):
        T = np.linspace(0.0, 1.0, num_interpolation_steps)
        table = walk_table(T, keyframes[k], keyframes[k + 1])
        for b, e, z in generate_inputs(embed[k], embed[k + 1], init_latents[k], init_latents[k + 1], T, len(T)):
            img = sample_frames(unet, vae, make_scheduler(kind, prediction_type), z, e, uncond, num_inference_steps,
                                guidance_scale, eta=eta, table=table)
            out.append(to_uint8(img))
    return np.concatenate(out)
