"""The sampler engine's launch plan as data: `sdw_engine_debug_ops` of a plan-only engine (no GPU, fake arena), parsed
into records, and the `sdw_gemm_desc` a GEMM record stands for."""
import ctypes as C
import os
import tempfile

# kernel launches per op line (sdw_engine_launches counts kernels; a GroupNorm is statistics, finalize, apply)
LAUNCHES = {"groupnorm": 3}
# sdw_gemm_desc fields a gemm record carries verbatim
GEMM_FIELDS = ("C", "W", "H", "B", "sW", "sH", "sB", "conv", "up_px", "up_py", "N", "ldb", "Kb", "b_batched", "sBh", "sBb",
               "ldc", "o_sW", "o_sH", "o_sB", "ldr", "rowvec_ld", "mode", "act", "alpha", "vt_col0", "vt_d", "vt_heads",
               "vt_ntok", "vt_ld")
PLAN_FIELDS = ("ver", "bn", "nsub", "ew", "tr", "et", "stages")


def _num(v):
    try:
        return int(v)
    except ValueError:
        return float(v)


def parse(text):
    """[(section, op index, kind, {key: number})] of an op listing"""
    out = []
    for line in text.splitlines():
        sec, idx, kind, *kv = line.split("\t")
        out.append((sec, int(idx), kind, {k: _num(v) for k, v in (f.split("=", 1) for f in kv)}))
    return out


def sd14_config(hw, frames, tiled=False):
    from stable_diffusion_videos_b200.configs import UNetConfig, VAEConfig
    from stable_diffusion_videos_b200.engine import EngineConfig

    u, v = UNetConfig.sd14(), VAEConfig()
    c = EngineConfig()
    c.in_channels, c.out_channels, c.num_levels, c.layers_per_block = 4, 4, len(u.block_out_channels), u.layers_per_block
    for i, ch in enumerate(u.block_out_channels):
        c.block_out_channels[i] = ch
        c.attention_heads[i] = u.heads(i)
    c.cross_attention_dim, c.ctx_tokens, c.norm_num_groups, c.norm_eps = u.cross_attention_dim, 77, u.norm_num_groups, 1e-5
    c.vae_num_levels, c.vae_layers_per_block, c.vae_norm_num_groups = len(v.block_out_channels), v.layers_per_block, v.norm_num_groups
    for i, ch in enumerate(v.block_out_channels):
        c.vae_block_out_channels[i] = ch
    c.vae_out_channels, c.vae_scale, c.vae_scaling_factor = 3, 2 ** (len(v.block_out_channels) - 1), 0.18215
    c.latent_h, c.latent_w = hw
    c.frames, c.guidance, c.max_steps = frames, 1, 64
    c.tiled = int(tiled)
    return c


def plan_only_ops(frames, hw=(64, 64), tiled=False):
    """(records, {section: kernel launches}, arena bytes) of the SD-1.4 engine at `frames`, planned on a fake arena:
    nothing is allocated or launched, so this runs without a GPU and costs no device memory next to one."""
    from stable_diffusion_videos_b200 import _native

    lib = _native.lib()
    lib.sdw_debug_plan_only(1)
    h = C.c_void_p()
    try:
        cfg = sd14_config(hw, frames, tiled)
        _native.check(lib.sdw_engine_create(C.byref(cfg), C.byref(h)))
        n = C.c_uint64()
        _native.check(lib.sdw_engine_arena_bytes(h, C.byref(n)))
        _native.check(lib.sdw_engine_bind(h, C.c_void_p(1 << 40), n))  # fake, aligned, never dereferenced
        a, b, d = C.c_int(), C.c_int(), C.c_int()
        _native.check(lib.sdw_engine_launches(h, C.byref(a), C.byref(b), C.byref(d)))
        with tempfile.TemporaryDirectory() as tmp:
            path = os.path.join(tmp, "ops.tsv")
            _native.check(lib.sdw_engine_debug_ops(h, path.encode()))
            text = open(path).read()
    finally:
        if h:
            lib.sdw_engine_destroy(h)
        lib.sdw_debug_plan_only(0)
    return parse(text), {"unet": b.value, "vae": d.value}, int(n.value)


def gemm_desc(f, A, Wt, out, bias=None, rowvec=None, resid=None, vt=None):
    """the sdw_gemm_desc of gemm record fields `f` on the given device addresses (ints), variant knobs left automatic"""
    from stable_diffusion_videos_b200 import _native

    d = _native.GemmDesc()
    for k in GEMM_FIELDS:
        setattr(d, k, f[k])
    d.A, d.Wt, d.out = A, Wt, out
    d.bias = bias if f["bias"] else None
    d.rowvec = rowvec if f["rowvec"] else None
    d.resid = resid if f["resid"] else None
    d.vt = vt if f["mode"] == 2 else None
    return d


def plan_of(desc):
    """(ver, bn, nsub, ew, tr, et, stages) the planner picks for `desc` (host only, in plan-only mode)"""
    from stable_diffusion_videos_b200 import _native

    lib = _native.lib()
    out = (C.c_int32 * 12)()
    lib.sdw_debug_plan_only(1)
    try:
        _native.check(lib.sdw_debug_plan(C.byref(desc), out))
    finally:
        lib.sdw_debug_plan_only(0)
    return tuple(out[:7])


def attention_plan_of(f):
    """(variant, grid x, y, z) the fused-attention planner picks for attention record fields `f` (plan-only mode)"""
    from stable_diffusion_videos_b200 import _native

    lib = _native.lib()
    out = (C.c_int32 * 5)()
    lib.sdw_debug_plan_only(1)
    try:
        _native.check(lib.sdw_debug_attention_plan(f["B"], f["Nq"], f["Nk"], f["heads"], f["d"], out))
    finally:
        lib.sdw_debug_plan_only(0)
    return out[0], out[2], out[3], out[4]
