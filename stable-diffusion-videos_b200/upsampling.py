"""Real-ESRGAN x4 upsampling (reference upsampling.py `RealESRGANModel`) on the native sm_90a engine
(sdw_upsampler_* in include/sdwalk.h).

`RealESRGANModel` has the reference's signatures: `RealESRGANModel(model_path)`, `from_pretrained(...)`,
`model(image, outscale=4, convert_to_pil=True)` and `upsample_imagefolder(...)`.  What the reference delegates to
basicsr's RRDBNet and realesrgan's `RealESRGANer.enhance` (half precision, no tiling) runs natively here:
`u8 = round(img * 255)`, `x = fp16(u8 / 255)`, `y = RRDBNet(x)`, `out = round(clamp(y, 0, 1) * 255)`, and for
`outscale != 4` a LANCZOS4 resize of the uint8 result on the host.  `upsample_frames` is the device path the walk uses.
There is no CPU fallback and no cuDNN path: without the CUDA library this class raises.
"""
import ctypes as C
import logging
import math
from pathlib import Path

import numpy as np
import torch

from . import _native as N
from .configs import esrgan_param_shapes

logger = logging.getLogger(__name__)

HUB_FILENAME = "RealESRGAN_x4plus.pth"


class UpsamplerConfig(C.Structure):
    _fields_ = [("num_feat", C.c_int32), ("num_block", C.c_int32), ("num_grow_ch", C.c_int32), ("in_h", C.c_int32),
                ("in_w", C.c_int32), ("frames", C.c_int32)]


def load_pth(path):
    """State dict of a Real-ESRGAN `.pth` file: the `params_ema` weights when present, else `params`, else the file's
    top level (what RealESRGANer loads)."""
    sd = torch.load(str(path), map_location="cpu", weights_only=True)
    if "params_ema" in sd:
        sd = sd["params_ema"]
    elif "params" in sd:
        sd = sd["params"]
    return sd


def check_state_dict(sd):
    """Strict key and shape check against basicsr's RRDBNet x4; returns the number of RRDB blocks."""
    num_block = 0
    while f"body.{num_block}.rdb1.conv1.weight" in sd:
        num_block += 1
    if num_block == 0:
        raise KeyError("not an RRDBNet state dict: body.0.rdb1.conv1.weight is missing")
    want = esrgan_param_shapes(num_block)
    missing = [k for k in want if k not in sd]
    unexpected = [k for k in sd if k not in want]
    if missing or unexpected:
        raise KeyError(f"RRDBNet x4 ({num_block} blocks) state dict mismatch: missing {missing[:5]}"
                       f"{' ...' if len(missing) > 5 else ''}, unexpected {unexpected[:5]}"
                       f"{' ...' if len(unexpected) > 5 else ''}")
    for k, s in want.items():
        if tuple(sd[k].shape) != s:
            raise ValueError(f"shape mismatch for {k}: {tuple(sd[k].shape)}, expected {s}")
    return num_block


class UpsamplerEngine:
    """One bound native upsampler for a fixed (frames, H, W) on one device, with its own packed weights."""

    def __init__(self, state_dict, num_block, h, w, frames, device):
        self.device = torch.device(device)
        self.h, self.w, self.frames = int(h), int(w), int(frames)
        self.cfg = UpsamplerConfig(64, int(num_block), 32, self.h, self.w, self.frames)
        self._model = N.NativeModel("upsampler", self.cfg, 256, self.device, "upsampler")
        self._h = self._model.h
        self.stream = torch.cuda.Stream(device=self.device)
        self._model.load(state_dict)

    def run(self, u8_in, u8_out, preclamp=None, use_graph=True):
        """u8_in [frames, H, W, 3] -> u8_out [frames, 4H, 4W, 3] (and the fp32 pre-clamp output), ordered after the
        caller's stream's work and before its later work."""
        N.require_cuda(u8_in, u8_out, preclamp)
        assert u8_in.is_contiguous() and u8_out.is_contiguous() and u8_in.dtype == u8_out.dtype == torch.uint8
        assert tuple(u8_in.shape) == (self.frames, self.h, self.w, 3)
        assert tuple(u8_out.shape) == (self.frames, 4 * self.h, 4 * self.w, 3)
        if preclamp is not None:
            assert preclamp.is_contiguous() and preclamp.dtype == torch.float32 and preclamp.shape == u8_out.shape
        # the engine's own stream (graph capture needs a real stream), fenced both ways against the caller's
        cur = torch.cuda.current_stream(self.device)
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            N.check(N.lib().sdw_upsampler_run(self._h, N.ptr(u8_in), N.ptr(u8_out), N.ptr(preclamp),
                                              int(bool(use_graph)), N.stream_ptr()))
        cur.wait_stream(self.stream)

    def profile(self, path):
        N.check(N.lib().sdw_upsampler_debug_profile(self._h, str(path).encode(), N.stream_ptr()))


class RealESRGANModel:
    """Real-ESRGAN x4 upsampler (RRDBNet, 64 features, 32 growth channels) with the reference's interface."""

    def __init__(self, model_path=None, tile=0, tile_pad=10, pre_pad=0, fp32=False, state_dict=None):
        if tile != 0:
            raise NotImplementedError("tiled Real-ESRGAN processing is not implemented (tile must be 0)")
        if pre_pad != 0:
            raise NotImplementedError("pre_pad is not implemented (it must be 0)")
        if fp32:
            raise NotImplementedError("the native upsampler runs in half precision only (fp32=False)")
        if state_dict is None:
            if model_path is None:
                raise ValueError("RealESRGANModel needs a model_path or a state_dict")
            state_dict = load_pth(model_path)
        self.num_block = check_state_dict(state_dict)
        self.state = {k: v.detach().to("cpu", torch.float16).contiguous() for k, v in state_dict.items()}
        self.tile, self.tile_pad, self.pre_pad, self.fp32 = tile, tile_pad, pre_pad, fp32
        self.device = None
        self._engines = {}

    # ------------------------------------------------------------------------------------------
    @classmethod
    def from_pretrained(cls, model_name_or_path="nateraw/real-esrgan"):
        """A `.pth` file, a directory holding RealESRGAN_x4plus.pth, or a Hugging Face repo id (as the reference)."""
        p = Path(model_name_or_path)
        if p.is_dir():
            file = p / HUB_FILENAME
        elif p.exists():
            file = p
        else:
            from huggingface_hub import hf_hub_download

            file = hf_hub_download(model_name_or_path, HUB_FILENAME)
        return cls(file)

    @classmethod
    def from_random(cls, seed=0, num_block=23):
        """basicsr-style initialisation: the dense-block convs kaiming-normal x 0.1 with zero bias, the other convs
        PyTorch's default Conv2d initialisation."""
        g = torch.Generator().manual_seed(int(seed))
        shapes = esrgan_param_shapes(num_block)
        sd = {}
        for k, s in shapes.items():
            fan_in = shapes[k.rsplit(".", 1)[0] + ".weight"][1] * 9
            if k.startswith("body."):
                if k.endswith(".weight"):
                    sd[k] = torch.randn(s, generator=g) * math.sqrt(2.0 / fan_in) * 0.1
                else:
                    sd[k] = torch.zeros(s)
            else:
                sd[k] = (torch.rand(s, generator=g) * 2 - 1) / math.sqrt(fan_in)
        return cls(state_dict=sd)

    def to(self, device):
        device = torch.device(device)
        if device.type != "cuda":
            raise N.SdwError("the native upsampler runs on CUDA devices only (no CPU fallback)")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        if device != self.device:
            self._engines = {}
        self.device = device
        return self

    def eval(self):
        return self

    def _dev(self):
        if self.device is None:
            if not torch.cuda.is_available():
                raise N.SdwError("the native upsampler needs a CUDA device (sm_90a); there is no CPU fallback")
            self.to("cuda")
        return self.device

    def engine(self, h, w, frames):
        """The engine for (H, W, frames), built on first use; the two most recent shapes stay resident."""
        key = (int(h), int(w), int(frames))
        eng = self._engines.pop(key, None)
        if eng is None:
            if len(self._engines) >= 2:
                self._engines.pop(next(iter(self._engines)))
            eng = UpsamplerEngine(self.state, self.num_block, h, w, frames, self._dev())
        self._engines[key] = eng  # most recent last
        return eng

    # ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def upsample_frames(self, frames_u8, frames_per_call=2, use_graph=True):
        """uint8 RGB frames [B, H, W, 3] on the device -> [B, 4H, 4W, 3], `frames_per_call` frames per engine call.
        Each call runs on the engine's own stream, which waits for the caller's stream first and which the caller's
        stream waits for afterwards."""
        dev = self._dev()
        N.require_cuda(frames_u8)
        if frames_u8.dtype != torch.uint8 or frames_u8.dim() != 4 or frames_u8.shape[-1] != 3:
            raise ValueError(f"expected uint8 frames [B, H, W, 3], got {frames_u8.dtype} {tuple(frames_u8.shape)}")
        B, H, W, _ = frames_u8.shape
        with torch.cuda.device(dev):
            out = torch.empty((B, 4 * H, 4 * W, 3), dtype=torch.uint8, device=dev)
            src = frames_u8.contiguous()
            for i0 in range(0, B, frames_per_call):
                n = min(frames_per_call, B - i0)
                self.engine(H, W, n).run(src[i0:i0 + n], out[i0:i0 + n], use_graph=use_graph)
        return out

    def _enhance_rgb(self, rgb_u8, outscale):
        """uint8 RGB [H, W, 3] on the host -> uint8 RGB [4H, 4W, 3] (resized to outscale x with LANCZOS4)."""
        dev = self._dev()
        x = torch.from_numpy(np.ascontiguousarray(rgb_u8)).to(dev)[None]
        out = self.upsample_frames(x, frames_per_call=1)[0].cpu().numpy()
        if outscale is not None and outscale != 4:
            import cv2

            h, w = rgb_u8.shape[:2]
            out = cv2.resize(out, (int(w * outscale), int(h * outscale)), interpolation=cv2.INTER_LANCZOS4)
        return out

    def forward(self, image, outscale=4, convert_to_pil=True):
        """Upsample a float RGB array in [0, 1] (HWC) or an image path.  Returns a PIL image, or with
        `convert_to_pil=False` a BGR uint8 array, as the reference does."""
        if isinstance(image, (str, Path)):
            import cv2

            img = cv2.imread(str(image), cv2.IMREAD_UNCHANGED)
            if img is None:
                raise FileNotFoundError(f"cannot read image {image}")
            if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
                raise NotImplementedError("the native upsampler takes 8-bit 3-channel images (no grayscale, alpha or "
                                          f"16-bit input); {image} is {img.dtype} {img.shape}")
            rgb = img[:, :, ::-1]
        else:
            rgb = (np.asarray(image) * 255).round().astype("uint8")
            if rgb.ndim != 3 or rgb.shape[2] != 3:
                raise NotImplementedError(f"expected an RGB image [H, W, 3], got shape {rgb.shape}")
        out = self._enhance_rgb(rgb, outscale)
        if convert_to_pil:
            from PIL import Image

            return Image.fromarray(out)
        return np.ascontiguousarray(out[:, :, ::-1])

    __call__ = forward

    def upsample_imagefolder(self, in_dir, out_dir, suffix="out", outfile_ext=".png", recursive=False, force=False):
        in_dir, out_dir = Path(in_dir), Path(out_dir)
        if not in_dir.exists():
            raise FileNotFoundError(f"Provided input directory {in_dir} does not exist")
        out_dir.mkdir(exist_ok=True, parents=True)
        generator = in_dir.rglob("*") if recursive else in_dir.glob("*")
        image_paths = [x for x in generator if x.suffix.lower() in [".png", ".jpg", ".jpeg"]]
        n_img = len(image_paths)
        for i, image in enumerate(image_paths):
            out_filepath = out_dir / (str(image.relative_to(in_dir).with_suffix("")) + suffix + outfile_ext)
            if not force and out_filepath.exists():
                logger.info(f"[{i}/{n_img}] {out_filepath} already exists, skipping. To avoid skipping, pass force=True.")
                continue
            logger.info(f"[{i}/{n_img}] upscaling {image}")
            im = self(str(image))
            out_filepath.parent.mkdir(parents=True, exist_ok=True)
            im.save(out_filepath)
