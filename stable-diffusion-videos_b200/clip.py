"""Native CLIP text tower (sdw_clip_* in include/sdwalk.h) behind `embed_text` (stable_diffusion_pipeline.py:809-820)
and the unconditional "" encode (P:341-348).

`NativeCLIPTextEncoder` is called like the `transformers.CLIPTextModel` the reference holds as `pipe.text_encoder`:
`encoder(input_ids)[0]` is last_hidden_state [B, 77, hidden] (fp16, CUDA).  Weights come from a CLIPTextModel state dict
(`from_state_dict`, `from_hf_model`); nothing here runs on the CPU and there is no fallback to the torch module.
"""
import ctypes as C

import torch

from . import _native as N


class ClipConfig(C.Structure):
    _fields_ = [("vocab", C.c_int32), ("max_positions", C.c_int32), ("hidden", C.c_int32), ("layers", C.c_int32),
                ("heads", C.c_int32), ("intermediate", C.c_int32), ("act_gelu_erf", C.c_int32), ("eps", C.c_float),
                ("max_batch", C.c_int32)]


class NativeCLIPTextEncoder:
    def __init__(self, vocab_size=49408, max_position_embeddings=77, hidden_size=768, num_hidden_layers=12,
                 num_attention_heads=12, intermediate_size=3072, hidden_act="quick_gelu", layer_norm_eps=1e-5,
                 max_batch=8, device=None):
        if not torch.cuda.is_available():
            raise N.SdwError("the native CLIP text encoder needs a CUDA device (sm_90a); there is no CPU fallback")
        if hidden_act not in ("quick_gelu", "gelu"):
            raise ValueError(f"hidden_act {hidden_act!r}: quick_gelu (SD-1.x) or gelu (SD-2.x) only")
        self.device = torch.device(device or f"cuda:{torch.cuda.current_device()}")
        self.dtype = torch.float16
        c = ClipConfig(vocab_size, max_position_embeddings, hidden_size, num_hidden_layers, num_attention_heads,
                       intermediate_size, int(hidden_act == "gelu"), layer_norm_eps, max_batch)
        self.cfg = c
        self._model = N.NativeModel("clip", c, 256, self.device, "CLIP")
        self._h = self._model.h

    # ------------------------------------------------------------------------------------------
    @classmethod
    def from_hf_model(cls, model, max_batch=8, device=None):
        """`model`: a transformers.CLIPTextModel (any device / dtype) — used as the weight container only."""
        c = model.config
        enc = cls(c.vocab_size, c.max_position_embeddings, c.hidden_size, c.num_hidden_layers, c.num_attention_heads,
                  c.intermediate_size, c.hidden_act, c.layer_norm_eps, max_batch=max_batch, device=device)
        enc.load_state_dict(model.state_dict())
        return enc

    def param_names(self):
        return self._model.param_names()

    def load_state_dict(self, sd, strict=True):
        # position_ids is a buffer, not a parameter
        self._model.load({k: v for k, v in sd.items() if not k.endswith("position_ids")}, strict)

    def to(self, device):
        if torch.device(device).type != "cuda":
            raise N.SdwError("the native CLIP text encoder lives on the GPU it was built on")
        return self

    def __call__(self, input_ids, attention_mask=None):
        """input_ids [B, 77] integer tensor -> (last_hidden_state [B, 77, hidden] fp16,) — the tuple the reference indexes
        with [0].  The causal mask is built in; `attention_mask` is what the SD pipelines pass: None."""
        if attention_mask is not None:
            raise NotImplementedError("padding masks are not used by the Stable Diffusion pipelines")
        B, P = input_ids.shape
        if P != self.cfg.max_positions:
            raise ValueError(f"expected {self.cfg.max_positions} token positions, got {P}")
        out_all = []
        with torch.cuda.device(self.device):
            ids = input_ids.to(device=self.device, dtype=torch.int32).contiguous()
            for i0 in range(0, B, self.cfg.max_batch):
                chunk = ids[i0:i0 + self.cfg.max_batch].contiguous()
                out = torch.empty((chunk.shape[0], P, self.cfg.hidden), dtype=torch.float16, device=self.device)
                N.check(N.lib().sdw_clip_forward(self._h, N.ptr(chunk), chunk.shape[0], N.ptr(out), N.stream_ptr()))
                out_all.append(out)
        return (torch.cat(out_all) if len(out_all) > 1 else out_all[0],)
