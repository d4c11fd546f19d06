"""Python handle of the native sampler engine (sdw_engine_* in include/sdwalk.h).

Owns the arena (one torch.uint8 CUDA tensor), loads fp16 state dicts by diffusers key name, installs a scheduler
plan and runs `sample` for `frames` frames per call.  No CPU fallback: everything here needs the CUDA library.
"""
import ctypes as C

import numpy as np
import torch

from . import _native as N
from .configs import VAE_KEY_ALIASES, UNetConfig, VAEConfig, unet_param_shapes, vae_param_shapes


class EngineConfig(C.Structure):
    _fields_ = [
        ("in_channels", C.c_int32), ("out_channels", C.c_int32), ("num_levels", C.c_int32),
        ("block_out_channels", C.c_int32 * 4), ("layers_per_block", C.c_int32), ("attention_heads", C.c_int32 * 4),
        ("cross_attention_dim", C.c_int32), ("ctx_tokens", C.c_int32), ("norm_num_groups", C.c_int32),
        ("norm_eps", C.c_float),
        ("vae_num_levels", C.c_int32), ("vae_block_out_channels", C.c_int32 * 4), ("vae_layers_per_block", C.c_int32),
        ("vae_norm_num_groups", C.c_int32), ("vae_out_channels", C.c_int32), ("vae_scale", C.c_int32),
        ("vae_scaling_factor", C.c_float),
        ("latent_h", C.c_int32), ("latent_w", C.c_int32), ("frames", C.c_int32), ("guidance", C.c_int32),
        ("max_steps", C.c_int32), ("tiled", C.c_int32),
    ]


class Engine:
    def __init__(self, unet_cfg: UNetConfig, vae_cfg: VAEConfig, latent_hw, frames, guidance=True, ctx_tokens=77,
                 max_steps=128, device=None, tiled=False):
        if not torch.cuda.is_available():
            raise N.SdwError("the native engine needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device(device or f"cuda:{torch.cuda.current_device()}")
        self.unet_cfg, self.vae_cfg = unet_cfg, vae_cfg
        self.frames, self.guidance = int(frames), bool(guidance)
        self.latent_hw = (int(latent_hw[0]), int(latent_hw[1]))
        self.ctx_tokens = ctx_tokens
        c = EngineConfig()
        c.in_channels, c.out_channels = unet_cfg.in_channels, unet_cfg.out_channels
        ch = unet_cfg.block_out_channels
        c.num_levels = len(ch)
        for i, v in enumerate(ch):
            c.block_out_channels[i] = v
            c.attention_heads[i] = unet_cfg.heads(i)
        c.layers_per_block = unet_cfg.layers_per_block
        c.cross_attention_dim, c.ctx_tokens = unet_cfg.cross_attention_dim, ctx_tokens
        c.norm_num_groups, c.norm_eps = unet_cfg.norm_num_groups, unet_cfg.norm_eps
        vch = vae_cfg.block_out_channels
        c.vae_num_levels = len(vch)
        for i, v in enumerate(vch):
            c.vae_block_out_channels[i] = v
        c.vae_layers_per_block = vae_cfg.layers_per_block
        c.vae_norm_num_groups = vae_cfg.norm_num_groups
        c.vae_out_channels = vae_cfg.out_channels
        c.vae_scale = 2 ** (len(vch) - 1)
        c.vae_scaling_factor = vae_cfg.scaling_factor
        c.latent_h, c.latent_w = self.latent_hw
        c.frames, c.guidance, c.max_steps = self.frames, int(self.guidance), max_steps
        c.tiled = int(bool(tiled))  # circular convolution padding (reference from_pretrained(tiled=True), P:841-858)
        self.cfg = c
        self.vae_scale = c.vae_scale
        self._model = N.NativeModel("engine", c, 1024, self.device, "UNet / VAE")
        self._h = self._model.h
        self.n_steps = 0
        self._plan_key = None
        # graph capture is illegal on the legacy default stream: the engine runs on its own stream, fenced both ways
        self._stream = torch.cuda.Stream(device=self.device)

    # ------------------------------------------------------------------------------------------
    def param_names(self):
        return self._model.param_names()

    def load_state_dict(self, unet_sd, vae_sd, strict=True):
        """unet_sd: diffusers UNet keys; vae_sd: AutoencoderKL keys (post_quant_conv.*, decoder.*; encoder ignored)."""
        shapes = dict(unet_param_shapes(self.unet_cfg))
        shapes.update({"vae." + k: v for k, v in vae_param_shapes(self.vae_cfg).items()})
        items = dict(unet_sd)
        for k, v in vae_sd.items():
            if k.startswith("encoder.") or k.startswith("quant_conv."):
                continue
            parts = k.split(".")
            parts = [VAE_KEY_ALIASES.get(p, p) for p in parts]
            items["vae." + ".".join(parts)] = v
        for name, t in items.items():
            if name not in shapes:
                continue  # the engine's table is the same key set: load() rejects or skips it
            want, got = tuple(shapes[name]), tuple(t.shape)
            # the only accepted alias: a 1x1 conv stored as a Linear weight or the reverse, (c_out, c_in) <->
            # (c_out, c_in, 1, 1) (old VAE attention checkpoints, use_linear_projection models)
            if got != want and got + (1, 1) != want and got != want + (1, 1):
                raise N.SdwError(f"shape mismatch for {name}: {got} vs {want}")
        self._model.load(items, strict)

    def set_scheduler(self, scheduler, num_inference_steps, guidance_scale):
        scheduler.set_timesteps(num_inference_steps)
        plan = scheduler.plan()
        n = len(plan)
        ts = np.asarray(scheduler.timesteps, dtype=np.float32)
        assert ts.shape[0] == n
        coefs = (N.StepCoef * n)()
        for i, st in enumerate(plan):
            k = coefs[i]
            k.guidance = float(guidance_scale)
            k.c_x = float(st["c_x"])
            for j in range(5):
                k.c_e[j] = float(st["c_e"][j])
            for j in range(4):
                k.hist_slot[j] = int(st["hist_slot"][j])
            k.use_x_base, k.save_x_base, k.push_slot = st["use_x_base"], st["save_x_base"], st["push_slot"]
            k.next_in_scale = float(plan[i + 1]["in_scale"]) if i + 1 < n else 1.0
            k.push_e, k.push_x = float(st.get("push_e", 1.0)), float(st.get("push_x", 0.0))
        with torch.cuda.device(self.device):
            N.check(N.lib().sdw_engine_set_schedule(
                self._h, n, ts.ctypes.data_as(C.POINTER(C.c_float)), coefs, C.c_float(scheduler.init_noise_sigma),
                C.c_float(plan[0]["in_scale"]), N.stream_ptr()))
            torch.cuda.current_stream().synchronize()
        self.n_steps = n
        self._timesteps = [torch.tensor(t) for t in np.asarray(scheduler.timesteps).tolist()]

    def launches(self):
        a, b, c = C.c_int(), C.c_int(), C.c_int()
        N.check(N.lib().sdw_engine_launches(self._h, C.byref(a), C.byref(b), C.byref(c)))
        return a.value, b.value, c.value

    # ------------------------------------------------------------------------------------------
    def sample(self, latents, cond, uncond=None, use_graph=True, return_latents=False, return_raw=False, callback=None,
               callback_steps=1):
        """latents [F,4,h,w] (any float dtype), cond [F,tokens,D], uncond [1,tokens,D] -> uint8 [F,8h,8w,3] (CUDA).

        `callback(i, t, latents)` (reference P:429-430) is called every `callback_steps` denoise steps with the current
        fp32 latents; the sampler then runs as eager per-step segments instead of one CUDA graph."""
        F = self.frames
        h, w = self.latent_hw
        N.require_cuda(latents, cond, uncond)
        if tuple(latents.shape) != (F, self.unet_cfg.in_channels, h, w):
            raise ValueError(f"Unexpected latents shape, got {tuple(latents.shape)}, expected "
                             f"{(F, self.unet_cfg.in_channels, h, w)}")
        D = self.unet_cfg.cross_attention_dim
        if tuple(cond.shape) != (F, self.ctx_tokens, D):
            raise ValueError(f"Unexpected text_embeddings shape, got {tuple(cond.shape)}, expected "
                             f"{(F, self.ctx_tokens, D)}")
        if self.guidance and (uncond is None or tuple(uncond.shape) not in ((1, self.ctx_tokens, D), (F, self.ctx_tokens, D))):
            raise ValueError(f"Unexpected unconditional embedding shape, got "
                             f"{None if uncond is None else tuple(uncond.shape)}, expected {(1, self.ctx_tokens, D)} "
                             f"(shared) or {(F, self.ctx_tokens, D)} (one per sample)")
        if self.guidance:
            N.check(N.lib().sdw_engine_set_uncond_batch(self._h, int(uncond.shape[0])))
        lat = latents.to(torch.float32).contiguous()
        cnd = cond.to(torch.float16).contiguous()
        unc = uncond.to(torch.float16).contiguous() if uncond is not None else None
        out = torch.empty((F, h * self.vae_scale, w * self.vae_scale, self.vae_cfg.out_channels), dtype=torch.uint8,
                          device=self.device)
        fin = torch.empty_like(lat) if return_latents else None
        raw = torch.empty(out.shape, dtype=torch.float32, device=self.device) if return_raw else None
        with torch.cuda.device(self.device):
            cur = torch.cuda.current_stream()
            self._stream.wait_stream(cur)
            with torch.cuda.stream(self._stream):
                if callback is None:
                    N.check(N.lib().sdw_engine_sample(self._h, N.ptr(lat), N.ptr(cnd), N.ptr(unc), N.ptr(out), N.ptr(fin),
                                                      N.ptr(raw), int(use_graph), N.stream_ptr()))
                else:
                    lib = N.lib()
                    N.check(lib.sdw_engine_sample_begin(self._h, N.ptr(lat), N.ptr(cnd), N.ptr(unc), N.stream_ptr()))
                    step_lat = torch.empty_like(lat)
                    for i in range(self.n_steps):
                        report = i % callback_steps == 0
                        N.check(lib.sdw_engine_sample_steps(self._h, i, i + 1, N.ptr(step_lat) if report else None,
                                                            N.stream_ptr()))
                        if report:
                            self._stream.synchronize()
                            callback(i, self._timesteps[i], step_lat.clone())
                    N.check(lib.sdw_engine_sample_end(self._h, N.ptr(out), N.ptr(fin), N.ptr(raw), N.stream_ptr()))
            cur.wait_stream(self._stream)
        if return_raw:
            return out, raw
        return (out, fin) if return_latents else out

    def debug_unet(self, x_nchw, step, ctx):
        """one UNet forward on an explicit [Bn] batch -> eps [Bn,4,h,w] fp32 (parity hook)."""
        Bn = self.frames * (2 if self.guidance else 1)
        h, w = self.latent_hw
        x = x_nchw.to(torch.float32).contiguous()
        c = ctx.to(torch.float16).contiguous()
        assert x.shape[0] == Bn and c.shape[0] == Bn
        out = torch.empty((Bn, h, w, self.unet_cfg.out_channels), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            N.check(N.lib().sdw_engine_debug_unet(self._h, N.ptr(x), int(step), N.ptr(c), N.ptr(out), N.stream_ptr()))
        return out.permute(0, 3, 1, 2).contiguous()

    def debug_profile(self, path):
        """Tooling: per-op CUDA-event times of one UNet forward + the VAE decode, written as TSV (section, idx, us, tag)."""
        with torch.cuda.device(self.device):
            N.check(N.lib().sdw_engine_debug_profile(self._h, str(path).encode(), N.stream_ptr()))
            torch.cuda.synchronize()

    def debug_vae(self, latents):
        """VAE decode of [F,4,h,w] latents (pre-division by 0.18215 happens inside) -> (uint8 NHWC, fp32 NHWC raw)."""
        F = self.frames
        h, w = self.latent_hw
        lat = latents.to(torch.float32).contiguous()
        shp = (F, h * self.vae_scale, w * self.vae_scale, self.vae_cfg.out_channels)
        out = torch.empty(shp, dtype=torch.uint8, device=self.device)
        raw = torch.empty(shp, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            N.check(N.lib().sdw_engine_debug_vae(self._h, N.ptr(lat), N.ptr(out), N.ptr(raw), N.stream_ptr()))
        return out, raw
