"""Real-ESRGAN x4plus (23 RRDB blocks) on 512x512 frames: ms per frame, TFLOP/s against the network's 9.40 TFLOP per
frame, the per-op profile, and walk() frames/s with and without upsample=True.  Random weights (the cost does not depend
on them).  Writes only to a temporary directory.
Usage: python tools/esrgan_bench.py [--iters 5] [--walk-frames 4] [--walk-steps 10] [--no-walk]"""
import argparse
import collections
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from stable_diffusion_videos_b200.upsampling import RealESRGANModel  # noqa: E402

TFLOP_PER_FRAME = 9.40  # 8.67 in the 512^2 trunk + 0.71 in the 1024^2 / 2048^2 head (unfolded 3x3 convs)
PEAK = 989.4            # H100 SXM dense fp16 tensor TFLOP/s


def gpu_state():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[torch.cuda.current_device()]
    except Exception as e:  # the numbers still stand; the card description is then missing
        return f"unavailable ({e})"


def time_upsampler(model, F, iters):
    x = torch.randint(0, 256, (F, 512, 512, 3), dtype=torch.uint8, device="cuda")
    for _ in range(2):
        model.upsample_frames(x, frames_per_call=F)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(iters):
        model.upsample_frames(x, frames_per_call=F)
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / iters / F


def profile(model, F):
    eng = model.engine(512, 512, F)
    path = os.path.join(tempfile.mkdtemp(), "esrgan_profile.tsv")
    eng.profile(path)
    agg = collections.OrderedDict()
    for line in open(path):
        _, _, us, tag = line.rstrip("\n").split("\t")
        key = re.sub(r"^body\.\d+\.", "body.*.", tag)
        a = agg.setdefault(key, [0, 0.0])
        a[0] += 1
        a[1] += float(us)
    return agg


def walk_fps(upsampler, frames, steps, batch):
    from stable_diffusion_videos_b200 import StableDiffusionWalkPipeline

    pipe = StableDiffusionWalkPipeline.from_random(device="cuda")
    pipe.upsampler = upsampler
    out = {}
    with tempfile.TemporaryDirectory() as d:
        for up in (False, True):
            kw = dict(seeds=[1, 2], num_interpolation_steps=frames, output_dir=d, num_inference_steps=steps,
                      batch_size=batch, upsample=up, make_video=False)
            pipe.walk(["a", "b"], name=f"warm{int(up)}", **kw)
            torch.cuda.synchronize()
            t = time.perf_counter()
            pipe.walk(["a", "b"], name=f"run{int(up)}", **kw)
            torch.cuda.synchronize()
            out["upsample" if up else "plain"] = frames / (time.perf_counter() - t)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--walk-frames", type=int, default=4)
    ap.add_argument("--walk-steps", type=int, default=10)
    ap.add_argument("--walk-batch", type=int, default=2)
    ap.add_argument("--no-walk", action="store_true")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    model = RealESRGANModel.from_random(0, num_block=23).to("cuda")
    res = {"gpu": gpu_state()}
    for F in (1, 2):
        ms = time_upsampler(model, F, a.iters)
        res[f"ms_per_frame_F{F}"] = round(ms, 3)
        res[f"tflops_F{F}"] = round(TFLOP_PER_FRAME / ms * 1e3, 1)
        res[f"frac_of_peak_F{F}"] = round(TFLOP_PER_FRAME / ms * 1e3 / PEAK, 3)
    agg = profile(model, 2)
    tot = sum(v[1] for v in agg.values())
    print(f"== per-op profile, 2 frames of 512x512: {tot / 1e3:.2f} ms over {sum(v[0] for v in agg.values())} ops")
    for k, (n, us) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f"{us / 1e3:8.3f} ms {100 * us / tot:5.1f}%  x{n:3d}  {us / n:8.1f} us  {k}")
    if not a.no_walk:
        fps = walk_fps(model, a.walk_frames, a.walk_steps, a.walk_batch)
        res.update({f"walk_fps_{k}": round(v, 3) for k, v in fps.items()})
        res["walk"] = f"SD-1.4 random weights, 512x512, {a.walk_frames} frames, {a.walk_steps} PNDM steps, batch {a.walk_batch}"
    res["gpu_after"] = gpu_state()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
