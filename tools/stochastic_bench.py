"""Cost of the step noise of the stochastic samplers on one GPU.

  python tools/stochastic_bench.py [--frames 30] [--steps 50] [--reps 3] [--out result.json]

Times the SD-1.4 random-weight sampler (classifier-free guidance, 64x64 latents, CUDA graph) at `--frames` frames per
call for DDIM eta = 0 against eta = 1 and Euler against Euler ancestral, the two members of each pair alternating call by
call, with CUDA events; then the fused CFG + step kernel alone (sdw_cfg_sched_step_noise) at the same F with c_z = 0
(the deterministic arithmetic) and c_z != 0 (Philox noise of two keys per frame, the walk case).  Prints one JSON line
with the card's name and power limit.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def sampler_bench(a):
    from stable_diffusion_videos_b200 import noise
    from stable_diffusion_videos_b200.configs import (UNetConfig, VAEConfig, random_state_dict, unet_param_shapes,
                                                      vae_param_shapes)
    from stable_diffusion_videos_b200.engine import Engine
    from stable_diffusion_videos_b200.schedulers import SCHEDULERS

    dev = torch.device("cuda", 0)
    F, h = a.frames, 64
    ucfg, vcfg = UNetConfig.sd14(), VAEConfig()
    eng = Engine(ucfg, vcfg, (h, h), F)
    eng.load_state_dict({k: v.to(dev) for k, v in random_state_dict(unet_param_shapes(ucfg), 0).items()},
                        {k: v.to(dev) for k, v in random_state_dict(vae_param_shapes(vcfg), 1).items()})
    g = torch.Generator(device=dev).manual_seed(0)
    lat = torch.randn(F, 4, h, h, generator=g, device=dev)
    cond = torch.randn(F, 77, 768, generator=g, device=dev).half()
    unc = torch.randn(1, 77, 768, generator=g, device=dev).half()
    table = noise.walk_table(np.linspace(0.0, 1.0, F), 42, 1337)
    legs = {"ddim_eta0": ("ddim", 0.0), "ddim_eta1": ("ddim", 1.0), "euler": ("euler", 0.0), "euler_a": ("euler_a", 0.0)}
    times = {k: [] for k in legs}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for pair in (("ddim_eta0", "ddim_eta1"), ("euler", "euler_a")):
        for r in range(a.reps + 1):  # rep 0 warms up (graph capture)
            for leg in pair:
                kind, eta = legs[leg]
                eng.set_scheduler(SCHEDULERS[kind](), a.steps, 7.5, eta=eta)  # a new plan re-captures the graph
                if eng.stochastic:
                    eng.set_frame_noise(table)
                eng.sample(lat, cond, unc)  # capture
                torch.cuda.synchronize()
                ev0.record(eng._stream)
                for _ in range(a.calls):
                    eng.sample(lat, cond, unc)
                ev1.record(eng._stream)
                torch.cuda.synchronize()
                if r:
                    times[leg].append(ev0.elapsed_time(ev1) / a.calls)
    return {k: {"ms_per_call": float(np.median(v)), "all_ms": [round(x, 2) for x in v],
                "frames_per_s": F / (float(np.median(v)) / 1000)} for k, v in times.items()}


def kernel_bench(a):
    from stable_diffusion_videos_b200 import _native as n
    from stable_diffusion_videos_b200 import noise

    F, H, W = a.frames, 64, 64
    lib = n.lib()
    x = torch.randn(F, 4, H, W, device="cuda")
    xb, hist = torch.zeros_like(x), torch.zeros((4,) + tuple(x.shape), device="cuda")
    eps = torch.randn(2 * F, H, W, 4, device="cuda")
    nxt = torch.zeros((2 * F, H, W, 4), dtype=torch.float16, device="cuda")
    tab = noise.to_device(noise.walk_table(np.linspace(0.0, 1.0, F), 42, 1337), "cuda")
    out = {}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for name, cz in (("c_z=0", 0.0), ("c_z=0.5", 0.5)) * (a.reps + 1):
        k = n.StepCoef()
        k.guidance, k.c_x, k.c_e[0], k.push_slot, k.next_in_scale, k.c_z = 7.5, 0.99, -0.05, -1, 1.0, cz
        ptrs = [C.c_void_p(t.data_ptr()) for t in (eps, x, xb, hist)]
        ev0.record()
        for s in range(a.kernel_iters):
            n.check(lib.sdw_cfg_sched_step_noise(ptrs[0], 1, ptrs[1], ptrs[2], ptrs[3], C.byref(k), F, 4, H, W,
                                                 C.c_void_p(nxt.data_ptr()), 4, C.c_void_p(tab.data_ptr()), s % 50,
                                                 n.stream_ptr()))
        ev1.record()
        torch.cuda.synchronize()
        out.setdefault(name, []).append(ev0.elapsed_time(ev1) * 1000 / a.kernel_iters)
    return {k: {"us": float(np.median(v[1:])), "all_us": [round(x, 2) for x in v[1:]]} for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--calls", type=int, default=2)
    ap.add_argument("--kernel-iters", type=int, default=2000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("stochastic_bench needs a GPU")
    res = {"card": card(), "frames": a.frames, "steps": a.steps, "kernel": kernel_bench(a), "sampler": sampler_bench(a)}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
