"""ctypes binding of libsdwalk.so (the C ABI in include/sdwalk.h).

torch tensors are the only host container: every call passes `tensor.data_ptr()` plus explicit
sizes and the current CUDA stream.  There is NO CPU fallback: if the shared library is missing
or a call fails, a RuntimeError is raised.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsdwalk.so")
_lib = None


class SdwError(RuntimeError):
    pass


class StepCoef(C.Structure):
    _fields_ = [
        ("guidance", C.c_float), ("c_x", C.c_float), ("c_e", C.c_float * 5),
        ("hist_slot", C.c_int32 * 4), ("use_x_base", C.c_int32), ("save_x_base", C.c_int32),
        ("push_slot", C.c_int32), ("next_in_scale", C.c_float), ("push_e", C.c_float), ("push_x", C.c_float),
        ("c_z", C.c_float),
    ]


class FrameNoise(C.Structure):
    """sdw_frame_noise: frame f's step noise is w_a Z(key_a) + w_b Z(key_b) (include/sdwalk.h)"""
    _fields_ = [("key_a", C.c_uint64), ("key_b", C.c_uint64), ("w_a", C.c_float), ("w_b", C.c_float)]


class GemmDesc(C.Structure):
    _fields_ = [
        ("A", C.c_void_p), ("C", C.c_int32), ("W", C.c_int32), ("H", C.c_int32), ("B", C.c_int32),
        ("sW", C.c_int64), ("sH", C.c_int64), ("sB", C.c_int64),
        ("conv", C.c_int32), ("up_px", C.c_int32), ("up_py", C.c_int32),
        ("Wt", C.c_void_p), ("N", C.c_int32), ("ldb", C.c_int64), ("Kb", C.c_int64),
        ("b_batched", C.c_int32), ("sBh", C.c_int64), ("sBb", C.c_int64),
        ("bias", C.c_void_p), ("rowvec", C.c_void_p), ("rowvec_ld", C.c_int32),
        ("resid", C.c_void_p), ("ldr", C.c_int64),
        ("out", C.c_void_p), ("ldc", C.c_int64),
        ("o_sW", C.c_int64), ("o_sH", C.c_int64), ("o_sB", C.c_int64),
        ("mode", C.c_int32), ("act", C.c_int32), ("alpha", C.c_float),
        ("vt_col0", C.c_int32), ("vt_d", C.c_int32), ("vt_heads", C.c_int32), ("vt_ntok", C.c_int32),
        ("vt", C.c_void_p), ("vt_ld", C.c_int64), ("bn", C.c_int32), ("ver", C.c_int32), ("nsub", C.c_int32), ("ew", C.c_int32), ("tr", C.c_int32), ("et", C.c_int32), ("reserved0", C.c_int32),
    ]


def lib():
    """Load libsdwalk.so (once).  Fails loudly: the CUDA extension IS the product path."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise SdwError(
                f"{LIB_PATH} not built: run `python __graft_entry__.py build` "
                "(the native sm_90a library is required; there is no fallback path)")
        _lib = C.CDLL(LIB_PATH)
        _lib.sdw_last_error.restype = C.c_char_p
    return _lib


def check(rc):
    if rc != 0:
        raise SdwError(f"libsdwalk error {rc}: {lib().sdw_last_error().decode()}")


def stream_ptr():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise SdwError("libsdwalk operates on CUDA tensors only (no CPU fallback)")


class NativeModel:
    """One native engine behind the `sdw_<prefix>_*` functions (engine, clip, upsampler, safety): created from its config
    struct, bound to a zero-filled arena on `device` aligned to `align` bytes, destroyed with this object.  `h` is the
    handle the engine's own entry points take; `what` names the model in error messages."""

    def __init__(self, prefix, cfg, align, device, what):
        self.prefix, self.device, self.what = prefix, torch.device(device), what
        self._fn("destroy").restype = None
        self.h = C.c_void_p()
        check(self._fn("create")(C.byref(cfg), C.byref(self.h)))
        nbytes = C.c_uint64()
        check(self._fn("arena_bytes")(self.h, C.byref(nbytes)))
        self.arena_bytes = int(nbytes.value)
        with torch.cuda.device(self.device):
            self.arena = torch.zeros(self.arena_bytes + align, dtype=torch.uint8, device=self.device)
            base = (self.arena.data_ptr() + align - 1) // align * align
            check(self._fn("bind")(self.h, C.c_void_p(base), C.c_uint64(self.arena_bytes)))

    def _fn(self, name):
        return getattr(lib(), f"sdw_{self.prefix}_{name}")

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self._fn("destroy")(self.h)
                self.h = None
        except Exception:
            pass

    def param_names(self):
        """{name: numel} of every parameter, in the engine's registration order."""
        name, numel, out = C.c_char_p(), C.c_int64(), {}
        for i in range(self._fn("num_params")(self.h)):
            check(self._fn("param_info")(self.h, i, C.byref(name), C.byref(numel)))
            out[name.value.decode()] = int(numel.value)
        return out

    def load(self, items, strict=True):
        """Load {name: tensor} (any device / dtype, handed over as contiguous fp16) and require that every parameter is
        then loaded.  Unknown names raise when `strict` (else they are skipped) and element counts are checked, all
        before anything is loaded."""
        expected = self.param_names()
        todo = []
        for name, t in items.items():
            if name not in expected:
                if strict:
                    raise SdwError(f"unexpected {self.what} parameter {name}")
                continue
            if t.numel() != expected[name]:
                raise SdwError(f"shape mismatch for {name}: {tuple(t.shape)} has {t.numel()} elements, "
                               f"expected {expected[name]}")
            todo.append((name, t))
        keep = []  # the fp16 copies stay alive until the loads on the stream have run
        with torch.cuda.device(self.device):
            for name, t in todo:
                th = t.detach().to(device=self.device, dtype=torch.float16).contiguous()
                keep.append(th)
                check(self._fn("load_param")(self.h, name.encode(), ptr(th), C.c_int64(th.numel()), stream_ptr()))
            torch.cuda.current_stream().synchronize()
        first = C.c_char_p()
        missing = self._fn("missing_params")(self.h, C.byref(first))
        if missing:
            raise SdwError(f"{missing} {self.what} parameters not loaded (first: {first.value.decode()})")


# ----------------------------------------------------------------------------------------------
def slerp_lerp_batch(lat_a, lat_b, emb_a, emb_b, t, dot_threshold=0.9995):
    """Batched generate_inputs math (stable_diffusion_pipeline.py:466-468): returns (latents[n], embeds[n])."""
    require_cuda(lat_a, lat_b, emb_a, emb_b, t)
    assert lat_a.dtype == lat_b.dtype == emb_a.dtype == emb_b.dtype and lat_a.dtype in (torch.float16, torch.float32)
    n = t.numel()
    t = t.to(torch.float32).contiguous()
    out_lat = torch.empty((n,) + tuple(lat_a.shape[1:] if lat_a.shape[0] == 1 else lat_a.shape),
                          dtype=lat_a.dtype, device=lat_a.device)
    out_emb = torch.empty((n,) + tuple(emb_a.shape[1:] if emb_a.shape[0] == 1 else emb_a.shape),
                          dtype=emb_a.dtype, device=emb_a.device)
    check(lib().sdw_slerp_lerp_batch(ptr(lat_a.contiguous()), ptr(lat_b.contiguous()), ptr(emb_a.contiguous()),
                                     ptr(emb_b.contiguous()), ptr(t), C.c_int(n), C.c_int64(lat_a.numel()),
                                     C.c_int64(emb_a.numel()), C.c_int(lat_a.dtype == torch.float16),
                                     C.c_float(dot_threshold), ptr(out_lat), ptr(out_emb), stream_ptr()))
    return out_lat, out_emb


def pack_weight(w, geglu=False):
    """OIHW / [N,K] fp16 weight -> K-major [N][taps][ceil64(C)] layout of the GEMM kernel."""
    require_cuda(w)
    w = w.to(torch.float16).contiguous()
    if w.dim() == 2:
        w = w[:, :, None, None]
    N, Cc, kh, kw = w.shape
    cp = (Cc + 63) // 64 * 64
    out = torch.empty((N, kh * kw * cp), dtype=torch.float16, device=w.device)
    check(lib().sdw_pack_weight(ptr(w), N, Cc, kh, kw, int(geglu), ptr(out), stream_ptr()))
    return out


def pack_weight_up4(w):
    """[N, C, 3, 3] upsampler weight -> [4 parities][N][4 taps][ceil64(C)] (taps pre-summed in fp32)."""
    require_cuda(w)
    w = w.to(torch.float16).contiguous()
    N, Cc = w.shape[0], w.shape[1]
    cp = (Cc + 63) // 64 * 64
    out = torch.empty((4, N, 4 * cp), dtype=torch.float16, device=w.device)
    check(lib().sdw_pack_weight_up4(ptr(w), N, Cc, ptr(out), stream_ptr()))
    return out


def groupnorm(x, B, P, Cc, G, gamma, beta, eps, silu, y):
    """x, y: fp16 [B][P][ld] views whose last dim may be a channel slice of a wider buffer (ld = stride of dim -2)."""
    require_cuda(x, y, gamma, beta)
    check(lib().sdw_groupnorm(ptr(x), C.c_int64(x.stride(-2)), C.c_int(B), C.c_int64(P), C.c_int(Cc), C.c_int(G), ptr(gamma),
                              ptr(beta), C.c_float(eps), C.c_int(int(silu)), ptr(y), C.c_int64(y.stride(-2)), stream_ptr()))


def layernorm(x, rows, Cc, gamma, beta, eps, y):
    require_cuda(x, y, gamma, beta)
    check(lib().sdw_layernorm(ptr(x), C.c_int64(x.stride(-2)), C.c_int64(rows), C.c_int(Cc), ptr(gamma), ptr(beta),
                              C.c_float(eps), ptr(y), C.c_int64(y.stride(-2)), stream_ptr()))


def gemm(desc):
    check(lib().sdw_gemm(C.byref(desc), stream_ptr()))


def clip_embed(ids, tok, pos, rows, P, x):
    """x fp16 [rows][H] = tok[clamp(ids[r], 0, vocab - 1)] + pos[r % P]; ids int32 [rows], tok [vocab][H], pos [P][H]."""
    require_cuda(ids, tok, pos, x)
    vocab, H = tok.shape
    check(lib().sdw_clip_embed(ptr(ids), ptr(tok), ptr(pos), C.c_int(rows), C.c_int(P), C.c_int(H), C.c_int(vocab),
                               ptr(x), stream_ptr()))


def clip_attention(qkv, B, P, heads, out):
    """causal attention of the CLIP tower: qkv fp16 [B][P][3 * 64 heads] -> out fp16 [B][P][64 heads]."""
    require_cuda(qkv, out)
    check(lib().sdw_clip_attention(ptr(qkv), C.c_int(B), C.c_int(P), C.c_int(heads), ptr(out), stream_ptr()))


def clip_act(x, n, gelu_erf):
    """in place over the first n fp16 values of x: quick-GELU (gelu_erf = 0) or erf GELU (1)."""
    require_cuda(x)
    check(lib().sdw_clip_act(ptr(x), C.c_int64(n), C.c_int(int(gelu_erf)), stream_ptr()))


def safety_patch_rows(h, frames_u8, rows):
    """the safety checker's patch GEMM operand for frames_u8 [B, H, W, 3] (B <= max_batch), written into `rows`
    (fp16 [B * patches, ceil64(3 patch^2)])"""
    require_cuda(frames_u8, rows)
    B, H, W = frames_u8.shape[:3]
    check(lib().sdw_safety_preprocess(h, ptr(frames_u8), B, H, W, None, None, ptr(rows), stream_ptr()))


def safety_scores(embeds, special, special_w, concepts, concept_w, frames_u8=None):
    """the safety checker's score kernel on fp32 tables: returns (flags int32 [B], cos fp32 [B, ns + nc],
    scores fp64 [B, ns + nc]); flagged frames of `frames_u8` (uint8 [B, ...]) are zeroed in place"""
    t = [x.float().contiguous() for x in (embeds, special, special_w, concepts, concept_w)]
    require_cuda(*t, frames_u8)
    B, D = t[0].shape
    ns, nc = t[1].shape[0], t[3].shape[0]
    flags = torch.empty(B, dtype=torch.int32, device=t[0].device)
    cos = torch.empty((B, ns + nc), dtype=torch.float32, device=t[0].device)
    sc = torch.empty((B, ns + nc), dtype=torch.float64, device=t[0].device)
    fb = frames_u8[0].numel() if frames_u8 is not None else 0
    check(lib().sdw_safety_scores(ptr(t[0]), C.c_int(B), C.c_int(D), ptr(t[1]), ptr(t[2]), C.c_int(ns), ptr(t[3]),
                                  ptr(t[4]), C.c_int(nc), ptr(flags), ptr(cos), ptr(sc), ptr(frames_u8), C.c_int64(fb),
                                  stream_ptr()))
    return flags, cos, sc
