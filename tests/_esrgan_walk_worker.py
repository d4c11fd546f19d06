"""Worker of tests/test_esrgan_gpu.py's sharded test: renders a tiny walk with upsample=True, under torchrun (one rank
per GPU) or alone."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

from _helpers import TINY_UNET, TINY_VAE, make_oracle, product_cfgs  # noqa: E402


def main(out_dir, name):
    from stable_diffusion_videos_b200 import parallel
    from stable_diffusion_videos_b200.pipeline import (NativeUNet, NativeVAE, StableDiffusionWalkPipeline,
                                                       SyntheticTextEncoder, SyntheticTokenizer)
    from stable_diffusion_videos_b200.schedulers import PNDMScheduler
    from stable_diffusion_videos_b200.upsampling import RealESRGANModel

    rank, world, local = parallel.init_distributed()
    torch.cuda.set_device(local)
    unet, vae = make_oracle(TINY_UNET, TINY_VAE)
    ucfg, vcfg = product_cfgs(TINY_UNET, TINY_VAE)
    usd = {k: v.half() for k, v in unet.state_dict().items()}
    vsd = {k: v.half() for k, v in vae.state_dict().items()}
    pipe = StableDiffusionWalkPipeline(NativeVAE(vcfg, vsd), SyntheticTextEncoder(TINY_UNET.cross_attention_dim),
                                       SyntheticTokenizer(), NativeUNet(ucfg, usd), PNDMScheduler()).to(f"cuda:{local}")
    pipe.upsampler = RealESRGANModel.from_random(4, num_block=1)
    pipe.walk(["0", "1", "2"], seeds=[42, 1337, 2022], num_interpolation_steps=[5, 4], output_dir=out_dir, name=name,
              fps=3, num_inference_steps=3, height=64, width=64, batch_size=2, upsample=True, make_video=False)
    if world > 1:
        import torch.distributed as dist

        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
