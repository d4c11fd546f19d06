"""Native Stable Diffusion safety checker (sdw_safety_* in include/sdwalk.h): what `__call__` runs after the VAE decode
when the pipeline has a checker (stable_diffusion_pipeline.py:440-447).

`NativeSafetyChecker` restates diffusers' `StableDiffusionSafetyChecker` fed by a `CLIPFeatureExtractor`: the uint8
frames are resized with Pillow's bicubic filter so that the shortest edge is 224, centre-cropped to 224 x 224 and
normalised; a CLIP ViT image tower and the visual projection give the image embedding; its cosine similarity to
3 "special care" and 17 concept embeddings is scored as diffusers does, and a frame with any concept score above 0 is
flagged (and, with `blackout=True`, replaced by a black frame on the device).  Everything runs on the GPU.  Only the
first call for a frame size waits: it allocates the resize buffer and uploads Pillow's coefficient tables; later calls
at that size, such as every batch of a walk, only enqueue work.  The checker lives on the device it was built on.
Weights come from a diffusers-layout checkpoint's `safety_checker/` folder
(`from_pretrained`) or a state dict (`from_state_dict`).
"""
import ctypes as C
import json
import math
from pathlib import Path

import torch

from . import _native as N

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
_VISION_DEFAULTS = dict(hidden_size=768, intermediate_size=3072, num_hidden_layers=12, num_attention_heads=12,
                        image_size=224, patch_size=32, hidden_act="quick_gelu", layer_norm_eps=1e-5)


class SafetyConfig(C.Structure):
    _fields_ = [("hidden", C.c_int32), ("layers", C.c_int32), ("heads", C.c_int32), ("intermediate", C.c_int32),
                ("image_size", C.c_int32), ("patch", C.c_int32), ("proj_dim", C.c_int32), ("n_concepts", C.c_int32),
                ("n_special", C.c_int32), ("eps", C.c_float), ("max_batch", C.c_int32), ("act", C.c_int32),
                ("mean", C.c_float * 3), ("std", C.c_float * 3)]


def _size_224(v, field, allowed):
    """a preprocessor size field: the int 224 or a dict with exactly the keys `allowed`, each 224"""
    if isinstance(v, dict):
        if set(v) != set(allowed) or set(v.values()) != {224}:
            raise NotImplementedError(f"preprocessor_config.json: {field} {v!r} is not supported "
                                      f"(224 or {dict.fromkeys(allowed, 224)} only)")
    elif v != 224:
        raise NotImplementedError(f"preprocessor_config.json: {field} {v!r} is not supported (224 only)")


def check_preprocessor_config(pc):
    """(mean, std) of a CLIPFeatureExtractor / CLIPImageProcessor config; anything the native preprocessing does not do
    (another resample filter, no resize or crop, another crop size, non-RGB statistics) raises NotImplementedError
    naming the field."""
    if pc.get("resample", 3) != 3:
        raise NotImplementedError(f"preprocessor_config.json: resample {pc['resample']!r} is not supported "
                                  "(3, PIL bicubic, only)")
    for field in ("do_resize", "do_center_crop"):
        if not pc.get(field, True):
            raise NotImplementedError(f"preprocessor_config.json: {field}=False is not supported")
    for field in ("do_normalize", "do_rescale", "do_convert_rgb"):
        if pc.get(field, True) is False:
            raise NotImplementedError(f"preprocessor_config.json: {field}=False is not supported")
    if not math.isclose(pc.get("rescale_factor", 1 / 255), 1 / 255, rel_tol=1e-9):
        raise NotImplementedError(f"preprocessor_config.json: rescale_factor {pc['rescale_factor']!r} is not supported")
    # size {"height": 224, "width": 224} resizes to 224 x 224 without keeping the aspect ratio: not what runs here
    _size_224(pc.get("size", 224), "size", ("shortest_edge",))
    _size_224(pc.get("crop_size", 224), "crop_size", ("height", "width"))
    mean, std = pc.get("image_mean", CLIP_MEAN), pc.get("image_std", CLIP_STD)
    if len(mean) != 3 or len(std) != 3:
        raise NotImplementedError("preprocessor_config.json: image_mean / image_std must have 3 (RGB) entries")
    return tuple(float(m) for m in mean), tuple(float(s) for s in std)


def vision_config(cfg):
    """the vision tower fields of a safety_checker/config.json (CLIPConfig), with CLIPVisionConfig's defaults"""
    v = dict(_VISION_DEFAULTS)
    v.update(cfg.get("vision_config_dict") or {})
    v.update(cfg.get("vision_config") or {})
    if v["hidden_act"] not in ("quick_gelu", "gelu"):
        raise NotImplementedError(f"safety_checker/config.json: hidden_act {v['hidden_act']!r} is not supported")
    if v["image_size"] != 224:
        raise NotImplementedError(f"safety_checker/config.json: image_size {v['image_size']} is not supported (224)")
    return v


class NativeSafetyChecker:
    def __init__(self, hidden_size=1024, intermediate_size=4096, num_hidden_layers=24, num_attention_heads=16,
                 image_size=224, patch_size=14, hidden_act="quick_gelu", layer_norm_eps=1e-5, projection_dim=768,
                 n_concepts=17, n_special=3, image_mean=CLIP_MEAN, image_std=CLIP_STD, max_batch=8, device=None):
        if not torch.cuda.is_available():
            raise N.SdwError("the native safety checker needs a CUDA device (sm_90a); there is no CPU fallback")
        if hidden_act not in ("quick_gelu", "gelu"):
            raise ValueError(f"hidden_act {hidden_act!r}: quick_gelu or gelu only")
        self.device = torch.device(device or "cuda")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        c = SafetyConfig(hidden_size, num_hidden_layers, num_attention_heads, intermediate_size, image_size, patch_size,
                         projection_dim, n_concepts, n_special, layer_norm_eps, max_batch, int(hidden_act == "gelu"),
                         (C.c_float * 3)(*image_mean), (C.c_float * 3)(*image_std))
        self.cfg = c
        self.n_scores = n_special + n_concepts
        self._model = N.NativeModel("safety", c, 256, self.device, "safety checker")
        self._h = self._model.h
        self._stream = torch.cuda.Stream(device=self.device)  # graph replay needs a stream other than the legacy one

    # ------------------------------------------------------------------------------------------
    @classmethod
    def from_state_dict(cls, sd, vision, projection_dim=None, image_mean=CLIP_MEAN, image_std=CLIP_STD, max_batch=8,
                        device=None):
        """`sd`: a StableDiffusionSafetyChecker state dict; `vision`: its CLIPVisionConfig fields (dict or object)."""
        get = (lambda k: vision[k]) if isinstance(vision, dict) else (lambda k: getattr(vision, k))
        proj = projection_dim or sd["visual_projection.weight"].shape[0]
        chk = cls(get("hidden_size"), get("intermediate_size"), get("num_hidden_layers"), get("num_attention_heads"),
                  get("image_size"), get("patch_size"), get("hidden_act"), get("layer_norm_eps"), proj,
                  sd["concept_embeds"].shape[0], sd["special_care_embeds"].shape[0], image_mean, image_std,
                  max_batch=max_batch, device=device)
        chk.load_state_dict(sd)
        return chk

    @classmethod
    def from_pretrained(cls, root, max_batch=8, device=None):
        """Load `root/safety_checker/` (config.json + model.safetensors, model.fp16.safetensors or pytorch_model.bin)
        and `root/feature_extractor/preprocessor_config.json` of a local diffusers-layout checkpoint."""
        root = Path(root)
        sc_dir, fe = root / "safety_checker", root / "feature_extractor" / "preprocessor_config.json"
        if not (sc_dir / "config.json").is_file():
            raise FileNotFoundError(f"{sc_dir / 'config.json'}: the checkpoint has no safety checker")
        if not fe.is_file():
            raise FileNotFoundError(f"{fe}: the checkpoint has no feature extractor for its safety checker")
        mean, std = check_preprocessor_config(json.loads(fe.read_text()))
        cfg = json.loads((sc_dir / "config.json").read_text())
        vision = vision_config(cfg)
        sd = None
        for fn in ("model.safetensors", "model.fp16.safetensors"):
            if (sc_dir / fn).is_file():
                from safetensors.torch import load_file

                sd = load_file(str(sc_dir / fn))
                break
        if sd is None and (sc_dir / "pytorch_model.bin").is_file():
            sd = torch.load(str(sc_dir / "pytorch_model.bin"), map_location="cpu", weights_only=True)
        if sd is None:
            raise FileNotFoundError(f"no weights (model.safetensors, model.fp16.safetensors, pytorch_model.bin) "
                                    f"under {sc_dir}")
        return cls.from_state_dict(sd, vision, cfg.get("projection_dim"), mean, std, max_batch=max_batch, device=device)

    def param_names(self):
        return self._model.param_names()

    def load_state_dict(self, sd, strict=True):
        # position_ids is a buffer of older checkpoints, not a parameter
        self._model.load({k: v for k, v in sd.items() if not k.endswith("position_ids")}, strict)

    # ------------------------------------------------------------------------------------------
    def _frames(self, frames_u8):
        if frames_u8.device != self.device or frames_u8.dtype != torch.uint8 or frames_u8.dim() != 4 \
                or frames_u8.shape[-1] != 3:
            raise ValueError(f"expected uint8 RGB frames [B, H, W, 3] on {self.device}, got "
                             f"{frames_u8.dtype} {tuple(frames_u8.shape)} on {frames_u8.device}")
        if not frames_u8.is_contiguous():
            raise ValueError("frames must be contiguous")
        return frames_u8.shape[:3]

    def _on_stream(self, fn, *tensors):
        """run fn() on the checker's own stream, ordered after and before the caller's current stream"""
        cur = torch.cuda.current_stream(self.device)
        self._stream.wait_stream(cur)
        with torch.cuda.stream(self._stream):
            fn()
        for t in tensors:
            if t is not None:
                t.record_stream(self._stream)
        cur.wait_stream(self._stream)

    def _check(self, frames_u8, blackout, want_cos):
        B, H, W = self._frames(frames_u8)
        with torch.cuda.device(self.device):
            flags = torch.empty(B, dtype=torch.int32, device=self.device)
            cos = torch.empty((B, self.n_scores), dtype=torch.float32, device=self.device) if want_cos else None
            self._on_stream(lambda: N.check(N.lib().sdw_safety_check(
                self._h, N.ptr(frames_u8), B, H, W, N.ptr(flags), N.ptr(cos), int(bool(blackout)), N.stream_ptr())),
                frames_u8, flags, cos)
        return flags, cos

    def check_frames(self, frames_u8, blackout=True):
        """frames_u8: device uint8 [B, H, W, 3] (contiguous).  Returns the device bool tensor [B] of flagged frames; with
        `blackout` the flagged frames are zeroed in place, on the current stream."""
        return self._check(frames_u8, blackout, False)[0].bool()

    def scores(self, frames_u8):
        """(flags bool [B], cosine similarities fp32 [B, n_special + n_concepts], special-care concepts first) —
        the frames are left as they are."""
        flags, cos = self._check(frames_u8, False, True)
        return flags.bool(), cos

    def image_embeds(self, frames_u8, use_graph=True):
        """fp32 [B, projection_dim]: visual_projection(post_layernorm(CLS token))"""
        B, H, W = self._frames(frames_u8)
        with torch.cuda.device(self.device):
            out = torch.empty((B, self.cfg.proj_dim), dtype=torch.float32, device=self.device)
            self._on_stream(lambda: N.check(N.lib().sdw_safety_embed(
                self._h, N.ptr(frames_u8), B, H, W, N.ptr(out), int(bool(use_graph)), N.stream_ptr())), frames_u8, out)
        return out

    def preprocess(self, frames_u8):
        """(normalised pixels fp16 [B, 224, 224, 3], resized + cropped uint8 [B, 224, 224, 3]) for B <= max_batch"""
        B, H, W = self._frames(frames_u8)
        with torch.cuda.device(self.device):
            pix = torch.empty((B, 224, 224, 3), dtype=torch.float16, device=self.device)
            crop = torch.empty((B, 224, 224, 3), dtype=torch.uint8, device=self.device)
            N.check(N.lib().sdw_safety_preprocess(self._h, N.ptr(frames_u8), B, H, W, N.ptr(pix), N.ptr(crop), None,
                                                  N.stream_ptr()))
        return pix, crop
