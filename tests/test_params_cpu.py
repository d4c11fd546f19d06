"""The parameter table every native engine (sampler, CLIP text tower, upsampler, safety checker) shares: its keys and
element counts are the published checkpoint tables, nothing is loaded after bind, and load_param rejects what it cannot
load with a message naming the parameter, before launching anything.  Plan-only binds to a fake aligned arena; no
GPU."""
import ctypes as C
import math

import pytest

ENGINES = ["engine", "clip", "upsampler", "safety"]
# transformers' position_ids buffers, which are not parameters
POSITION_IDS = {"clip": "text_model.embeddings.position_ids",
                "safety": "vision_model.vision_model.embeddings.position_ids"}
CHECKER_EXTRA = {"visual_projection.weight": 768 * 1024, "concept_embeds": 17 * 768, "special_care_embeds": 3 * 768,
                 "concept_embeds_weights": 17, "special_care_embeds_weights": 3}


def _config_and_table(prefix):
    """(config struct, {name: numel} the engine must register)"""
    if prefix == "engine":
        from stable_diffusion_videos_b200.configs import UNetConfig, VAEConfig, unet_param_shapes, vae_param_shapes
        from test_capi_cpu import _cfg

        u, v = UNetConfig.sd14(), VAEConfig()
        want = {k: math.prod(s) for k, s in unet_param_shapes(u).items()}
        want.update({"vae." + k: math.prod(s) for k, s in vae_param_shapes(v).items()})
        return _cfg(u, v, (8, 8), 2), want
    if prefix == "clip":
        from _clip_fixtures import CONFIGS
        from transformers import CLIPTextConfig, CLIPTextModel

        from stable_diffusion_videos_b200.clip import ClipConfig

        kw = CONFIGS["sd1x-ViT-L"]
        sd = CLIPTextModel(CLIPTextConfig(**kw)).state_dict()
        cfg = ClipConfig(kw["vocab_size"], kw["max_position_embeddings"], kw["hidden_size"], kw["num_hidden_layers"],
                         kw["num_attention_heads"], kw["intermediate_size"], 0, 1e-5, 2)
        return cfg, {k: t.numel() for k, t in sd.items() if not k.endswith("position_ids")}
    if prefix == "safety":
        import _safety_oracle as so
        from transformers import CLIPVisionConfig, CLIPVisionModel

        from stable_diffusion_videos_b200.safety import CLIP_MEAN, CLIP_STD, SafetyConfig

        sd = CLIPVisionModel(CLIPVisionConfig(**so.VISION["ViT-L/14"])).state_dict()
        want = {"vision_model." + k: t.numel() for k, t in sd.items() if not k.endswith("position_ids")}
        want.update(CHECKER_EXTRA)
        cfg = SafetyConfig(1024, 24, 16, 4096, 224, 14, 768, 17, 3, 1e-5, 2, 0, (C.c_float * 3)(*CLIP_MEAN),
                           (C.c_float * 3)(*CLIP_STD))
        return cfg, want
    from stable_diffusion_videos_b200.configs import esrgan_param_shapes
    from stable_diffusion_videos_b200.upsampling import UpsamplerConfig

    return UpsamplerConfig(64, 2, 32, 16, 16, 1), {k: math.prod(s) for k, s in esrgan_param_shapes(2).items()}


@pytest.fixture(params=ENGINES)
def engine(request):
    """(prefix, lib, fn(name) -> sdw_<prefix>_<name>, unbound handle, bound handle, expected table)"""
    from stable_diffusion_videos_b200 import _native

    prefix = request.param
    lib = _native.lib()
    fn = lambda name: getattr(lib, f"sdw_{prefix}_{name}")  # noqa: E731
    fn("destroy").restype = None
    cfg, want = _config_and_table(prefix)
    handles = [C.c_void_p(), C.c_void_p()]
    for h in handles:
        _native.check(fn("create")(C.byref(cfg), C.byref(h)))
    n = C.c_uint64()
    _native.check(fn("arena_bytes")(handles[1], C.byref(n)))
    lib.sdw_debug_plan_only(1)
    try:
        _native.check(fn("bind")(handles[1], C.c_void_p(1 << 40), n))  # fake, aligned, never dereferenced
        yield prefix, lib, fn, handles[0], handles[1], want
    finally:
        lib.sdw_debug_plan_only(0)
        for h in handles:
            fn("destroy")(h)


def _table(fn, h):
    from stable_diffusion_videos_b200 import _native

    name, numel, out = C.c_char_p(), C.c_int64(), {}
    for i in range(fn("num_params")(h)):
        _native.check(fn("param_info")(h, i, C.byref(name), C.byref(numel)))
        out[name.value.decode()] = numel.value
    return out


def test_registry_is_the_published_key_table(engine):
    prefix, lib, fn, unbound, bound, want = engine
    got = _table(fn, bound)
    assert got == want
    assert list(_table(fn, unbound)) == list(got)  # one registration order, bound or not
    if prefix == "upsampler":
        assert list(got) == list(want)  # esrgan_param_shapes's order
    if prefix == "engine":  # registration order, not alphabetical
        assert list(got)[:2] == ["time_embedding.linear_1.weight", "time_embedding.linear_1.bias"]
    if prefix == "safety":  # the class embedding first, as CLIPVisionModel lists it
        assert list(got)[0] == next(iter(want))
    assert fn("param_info")(bound, len(want), None, None) == 1
    assert b"index" in lib.sdw_last_error()


def test_nothing_is_loaded_after_bind(engine):
    prefix, lib, fn, unbound, bound, want = engine
    for h in (unbound, bound):
        first = C.c_char_p()
        assert fn("missing_params")(h, C.byref(first)) == fn("num_params")(h) == len(want)
        assert first.value.decode() == next(iter(_table(fn, h)))
    assert fn("missing_params")(None, None) == -1


def test_load_param_rejects_before_launching(engine):
    """return code 1 (an argument error; a launch on this machine would fail with 2) and a message naming the
    parameter, for an unbound engine, an unknown name and a wrong element count"""
    prefix, lib, fn, unbound, bound, want = engine
    src = C.c_void_p(1 << 30)
    name, numel = next(iter(want.items()))
    assert fn("load_param")(unbound, name.encode(), src, C.c_int64(numel), None) == 1
    assert b"not bound" in lib.sdw_last_error() and name.encode() in lib.sdw_last_error()
    assert fn("load_param")(bound, b"no.such.weight", src, C.c_int64(numel), None) == 1
    assert lib.sdw_last_error().endswith(b"unknown parameter: no.such.weight")
    if prefix in POSITION_IDS:
        key = POSITION_IDS[prefix].encode()
        assert fn("load_param")(bound, key, src, C.c_int64(numel), None) == 1
        assert lib.sdw_last_error().endswith(b"unknown parameter: " + key)
    assert fn("load_param")(bound, name.encode(), src, C.c_int64(numel + 1), None) == 1
    msg = f"parameter size mismatch for {name}: expected {numel}, got {numel + 1}"
    assert lib.sdw_last_error().decode().endswith(msg)
    assert fn("missing_params")(bound, None) == len(want)
