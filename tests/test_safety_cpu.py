"""The safety checker without a GPU: the fp64 restatement (tests/_safety_oracle.py) against transformers'
CLIPVisionModel and CLIPImageProcessorPil, and the configuration checks that raise before anything is loaded.  Its
native parameter registry is tested with the other engines' in test_params_cpu.py."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

import _safety_oracle as so

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
