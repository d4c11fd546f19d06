"""The safety checker without a GPU: the native parameter registry against a diffusers-layout checker state dict built
from transformers (plan-only bind), the fp64 restatement (tests/_safety_oracle.py) against transformers'
CLIPVisionModel and CLIPImageProcessorPil, and the configuration checks that raise before anything is loaded."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

import _safety_oracle as so

CHECKER_EXTRA = {"visual_projection.weight": 768 * 1024, "concept_embeds": 17 * 768, "special_care_embeds": 3 * 768,
                 "concept_embeds_weights": 17, "special_care_embeds_weights": 3}


@pytest.fixture
def registry():
    from transformers import CLIPVisionConfig, CLIPVisionModel

    from stable_diffusion_videos_b200 import _native
    from stable_diffusion_videos_b200.safety import CLIP_MEAN, CLIP_STD, SafetyConfig

    lib = _native.lib()
    lib.sdw_safety_destroy.restype = None
    kw = so.VISION["ViT-L/14"]
    sd = CLIPVisionModel(CLIPVisionConfig(**kw)).state_dict()
    want = {"vision_model." + k: t.numel() for k, t in sd.items() if not k.endswith("position_ids")}
    want.update(CHECKER_EXTRA)
    cfg = SafetyConfig(1024, 24, 16, 4096, 224, 14, 768, 17, 3, 1e-5, 2, 0, (C.c_float * 3)(*CLIP_MEAN),
                       (C.c_float * 3)(*CLIP_STD))
    h = C.c_void_p()
    _native.check(lib.sdw_safety_create(C.byref(cfg), C.byref(h)))
    n = C.c_uint64()
    _native.check(lib.sdw_safety_arena_bytes(h, C.byref(n)))
    lib.sdw_debug_plan_only(1)
    try:
        _native.check(lib.sdw_safety_bind(h, C.c_void_p(1 << 40), n))  # fake, aligned, never dereferenced
        yield lib, h, want, sd
    finally:
        lib.sdw_debug_plan_only(0)
        lib.sdw_safety_destroy(h)


def test_registry_is_the_checker_key_table(registry):
    lib, h, want, sd = registry
    name, numel, got = C.c_char_p(), C.c_int64(), {}
    for i in range(lib.sdw_safety_num_params(h)):
        assert lib.sdw_safety_param_info(h, i, C.byref(name), C.byref(numel)) == 0
        got[name.value.decode()] = numel.value
    assert got == want
    tower = {k: v for k, v in want.items() if k.startswith("vision_model.")}
    assert sum(t.numel() for k, t in sd.items() if not k.endswith("position_ids")) == sum(tower.values())
    assert len(got) == len(tower) + 5 and sum(got.values()) == sum(tower.values()) + sum(CHECKER_EXTRA.values())
    assert not any(k.endswith("position_ids") for k in got)


def test_nothing_loaded_and_bad_loads_rejected(registry):
    lib, h, want, _ = registry
    first = C.c_char_p()
    assert lib.sdw_safety_missing_params(h, C.byref(first)) == len(want)
    assert first.value.decode() == next(iter(want))
    src = C.c_void_p(1 << 30)
    assert lib.sdw_safety_load_param(h, b"vision_model.vision_model.embeddings.position_ids", src, C.c_int64(257),
                                     None) == 1
    assert lib.sdw_last_error().endswith(b"unknown parameter: vision_model.vision_model.embeddings.position_ids")
    assert lib.sdw_safety_load_param(h, b"concept_embeds", src, C.c_int64(17 * 768 + 1), None) == 1
    assert lib.sdw_last_error().decode().endswith(
        f"parameter size mismatch for concept_embeds: expected {17 * 768}, got {17 * 768 + 1}")
    assert lib.sdw_safety_missing_params(h, None) == len(want)
    assert lib.sdw_safety_missing_params(None, None) == -1


@pytest.mark.parametrize("field,value", [("hidden", 1000), ("image_size", 336), ("patch", 15), ("n_concepts", 70),
                                         ("act", 2), ("max_batch", 0)])
def test_create_rejects_bad_configs(field, value):
    from stable_diffusion_videos_b200 import _native
    from stable_diffusion_videos_b200.safety import CLIP_MEAN, CLIP_STD, SafetyConfig

    cfg = SafetyConfig(128, 2, 2, 512, 224, 32, 64, 4, 2, 1e-5, 2, 0, (C.c_float * 3)(*CLIP_MEAN),
                       (C.c_float * 3)(*CLIP_STD))
    setattr(cfg, field, value)
    h = C.c_void_p()
    assert _native.lib().sdw_safety_create(C.byref(cfg), C.byref(h)) == 1
    assert b"invalid argument" in _native.lib().sdw_last_error()


@pytest.mark.parametrize("name,layers", [("small", None), ("ViT-L/14", 2), ("ViT-L/14", None)])
@pytest.mark.parametrize("trained_like", [False, True])
def test_oracle_tower_matches_transformers(name, layers, trained_like):
    model, cfg = so.hf_vision(so.VISION[name], trained_like=trained_like, layers=layers)
    sd = so.checker_state_dict(model)
    torch.manual_seed(5)
    x = torch.randn(2, 3, 224, 224, dtype=torch.float64)
    with torch.no_grad():
        ref = model.double().vision_model(pixel_values=x).pooler_output
    got = so.vision_tower(x, sd, cfg, pooled_only=True)
    assert float((got - ref).norm() / ref.norm()) <= 1e-9
    emb = so.vision_tower(x, sd, cfg)
    assert torch.allclose(emb, ref @ sd["visual_projection.weight"].double().T, rtol=1e-9, atol=1e-12)


@pytest.mark.parametrize("hw", [(512, 512), (768, 768), (512, 768), (768, 512), (576, 1024), (64, 64)])
def test_oracle_preprocess_matches_clip_image_processor_pil(hw):
    from transformers import CLIPImageProcessorPil

    u8 = so.test_frames(2, *hw, seed=hw[0] + hw[1])
    proc = CLIPImageProcessorPil(size={"shortest_edge": 224}, crop_size={"height": 224, "width": 224})
    ref = proc([f for f in u8], return_tensors="np")["pixel_values"].astype(np.float64)
    got = so.preprocess(u8).numpy()
    assert got.shape == ref.shape == (2, 3, 224, 224)
    assert np.abs(got - ref).max() <= 3e-7


def test_decide_follows_the_diffusers_loop():
    sd = {"special_care_embeds_weights": torch.tensor([0.5, 0.5]), "concept_embeds_weights": torch.tensor([0.5, 0.5])}
    cos = torch.tensor([[0.4, 0.4, 0.495, 0.3],    # nothing special: 0.495 - 0.5 -> -0.005, not flagged
                        [0.6, 0.4, 0.495, 0.3],    # special care lifts the concept by 0.01 -> 0.005, flagged
                        [0.4, 0.4, 0.5004, 0.3],   # rounds to 0.0: not flagged
                        [0.4, 0.4, 0.5006, 0.3]])  # rounds to 0.001: flagged
    flags, scores = so.decide(None, sd, cos=cos)
    assert flags.tolist() == [False, True, False, True]
    assert scores.dtype == np.float64 and scores[1, 0] == np.round(np.float64(np.float32(0.6)) - 0.5, 3)


@pytest.mark.parametrize("field,value", [("resample", 2), ("do_resize", False), ("do_center_crop", False),
                                         ("crop_size", {"height": 256, "width": 256}), ("size", {"shortest_edge": 256}),
                                         ("size", {"height": 224, "width": 224}), ("crop_size", {"shortest_edge": 224}),
                                         ("image_mean", [0.5]), ("do_normalize", False)])
def test_preprocessor_config_rejects_what_it_cannot_honour(field, value):
    from stable_diffusion_videos_b200.safety import check_preprocessor_config

    pc = {"crop_size": 224, "do_center_crop": True, "do_normalize": True, "do_resize": True, "resample": 3,
          "size": 224, "image_mean": list(so.CLIP_MEAN), "image_std": list(so.CLIP_STD)}
    assert check_preprocessor_config(pc) == (so.CLIP_MEAN, so.CLIP_STD)
    both = dict(pc, size={"shortest_edge": 224}, crop_size={"height": 224, "width": 224})
    assert check_preprocessor_config(both) == (so.CLIP_MEAN, so.CLIP_STD)
    pc[field] = value
    with pytest.raises(NotImplementedError, match=field.split("_")[0] if field == "image_mean" else field):
        check_preprocessor_config(pc)


def test_from_pretrained_checker_needs_its_folders(tmp_path):
    import _fake_checkpoint as fc

    from stable_diffusion_videos_b200.pipeline import StableDiffusionWalkPipeline

    fc.write_checkpoint(str(tmp_path), with_weights=False)
    with pytest.raises(FileNotFoundError, match="safety_checker"):
        StableDiffusionWalkPipeline.from_pretrained(str(tmp_path), safety_checker=True)
    (tmp_path / "safety_checker").mkdir()
    (tmp_path / "safety_checker" / "config.json").write_text(json.dumps({"projection_dim": 768}))
    with pytest.raises(FileNotFoundError, match="feature_extractor"):
        StableDiffusionWalkPipeline.from_pretrained(str(tmp_path), safety_checker=True)


def test_pipeline_rejects_other_checkers():
    from stable_diffusion_videos_b200.pipeline import NativeVAE, StableDiffusionWalkPipeline
    from stable_diffusion_videos_b200.configs import VAEConfig

    vae = NativeVAE(VAEConfig(), {})
    with pytest.raises(ValueError):
        StableDiffusionWalkPipeline(vae, None, None, None, None, safety_checker=object())
    with pytest.raises(TypeError):
        StableDiffusionWalkPipeline(vae, None, None, None, None, safety_checker=object(), feature_extractor={})


def test_pipeline_to_another_device_than_the_checker_raises():
    from types import SimpleNamespace

    from stable_diffusion_videos_b200._native import SdwError
    from stable_diffusion_videos_b200.configs import VAEConfig
    from stable_diffusion_videos_b200.pipeline import NativeVAE, StableDiffusionWalkPipeline

    pipe = StableDiffusionWalkPipeline(NativeVAE(VAEConfig(), {}), None, None, None, None)
    pipe.safety_checker = SimpleNamespace(device=torch.device("cuda", 1))  # a checker built on cuda:1
    assert pipe.to("cuda:1") is pipe
    with pytest.raises(SdwError, match="cuda:1"):
        pipe.to("cuda:0")
