"""The native safety checker (SD-1.x: ViT-L/14 image tower, 17 + 3 concepts) on uint8 frames: ms per check call at
B in {1, 8, 16} for 512^2 and 768^2 frames, and the per-op profile of one B = 8 call.  Random weights (the cost does not
depend on them).  Writes only to a temporary directory.
Usage: python tools/safety_bench.py [--iters 20]"""
import argparse
import collections
import json
import os
import re
import subprocess
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from stable_diffusion_videos_b200 import _native  # noqa: E402
from stable_diffusion_videos_b200.safety import NativeSafetyChecker  # noqa: E402


def gpu_state():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[torch.cuda.current_device()]
    except Exception as e:  # the numbers still stand; the card description is then missing
        return f"unavailable ({e})"


def random_checker(max_batch=8):
    chk = NativeSafetyChecker(max_batch=max_batch, device="cuda")
    g = torch.Generator().manual_seed(0)
    sd = {}
    for name, numel in chk.param_names().items():
        if name.endswith("weights"):
            sd[name] = torch.full((numel,), 0.2)
        else:
            sd[name] = torch.randn(numel, generator=g) * 0.02
    chk.load_state_dict(sd)
    return chk


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    chk = random_checker()
    res = {"gpu": gpu_state(), "ms_per_call": {}}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for hw in (512, 768):
        for B in (1, 8, 16):
            x = torch.randint(0, 256, (B, hw, hw, 3), dtype=torch.uint8, device="cuda")
            for _ in range(3):
                chk.check_frames(x, blackout=False)
            torch.cuda.synchronize()
            ev[0].record()
            for _ in range(args.iters):
                chk.check_frames(x, blackout=False)
            ev[1].record()
            torch.cuda.synchronize()
            ms = ev[0].elapsed_time(ev[1]) / args.iters
            res["ms_per_call"][f"{hw}x{hw} B={B}"] = round(ms, 3)
            print(f"{hw}x{hw} B={B:2d}: {ms:8.3f} ms per call, {ms / B:7.3f} ms per frame", flush=True)
    x = torch.randint(0, 256, (8, 512, 512, 3), dtype=torch.uint8, device="cuda")
    path = os.path.join(tempfile.mkdtemp(), "safety_profile.tsv")
    _native.check(_native.lib().sdw_safety_debug_profile(chk._h, _native.ptr(x), 8, 512, 512, path.encode(),
                                                           _native.stream_ptr()))
    agg = collections.OrderedDict()
    for line in open(path):
        _, _, us, tag = line.rstrip("\n").split("\t")
        key = re.sub(r"^layer \d+ ", "layer * ", tag)
        a = agg.setdefault(key, [0, 0.0])
        a[0] += 1
        a[1] += float(us)
    print("per-op profile, B = 8 at 512x512 (CUDA events, microseconds summed over the 24 layers):")
    for k, (n, us) in agg.items():
        print(f"  {us:9.1f} us  x{n:<3d} {k}")
    res["profile_us_B8_512"] = {k: round(us, 1) for k, (n, us) in agg.items()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
