"""Per-op time of one UNet forward (batch 2F) and one VAE decode (F frames) of the SD-1.4 engine, grouped by op kind/shape.
Usage: F=16 python tools/op_profile.py [out.tsv]"""
import collections
import os
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from stable_diffusion_videos_b200 import StableDiffusionWalkPipeline  # noqa: E402

F = int(os.environ.get("F", "16"))
out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(tempfile.gettempdir(), "sdw_op_profile.tsv")
pipe = StableDiffusionWalkPipeline.from_random(device="cuda")
emb = pipe.embed_text(["a", "b"])
cond = emb[:1].expand(F, -1, -1).contiguous()
noise = torch.randn(F, 4, 64, 64, device="cuda")
pipe(text_embeddings=cond, latents=noise, num_inference_steps=2, guidance_scale=7.5, output_type="np")
eng = next(iter(pipe._engines.values()))
eng.debug_profile(out)
rows = [l.rstrip("\n").split("\t") for l in open(out)]
for sec in ("unet", "vae"):
    agg = collections.OrderedDict()
    tot = 0.0
    for s, i, us, tag in rows:
        if s != sec:
            continue
        k = tag
        a = agg.setdefault(k, [0, 0.0])
        a[0] += 1
        a[1] += float(us)
        tot += float(us)
    print(f"== {sec}: {tot/1e3:.2f} ms over {sum(a[0] for a in agg.values())} ops")
    for k, (n, us) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f"{us/1e3:8.3f} ms {100*us/tot:5.1f}%  x{n:3d}  {us/n:8.1f} us  {k}")
