"""Real-ESRGAN upsampler without a GPU: the architecture's key / shape table (oracle, configs.py and the native registry
agree, 16,697,987 parameters), the arena size, the BLOCK_N 32 planner rules, the planned op list, checkpoint loading
and the options that must raise."""
import ctypes as C
import math

import numpy as np
import pytest
import torch


def _oracle_state_dict(num_block, seed=0):
    from stable_diffusion_videos_b200.configs import esrgan_param_shapes

    g = torch.Generator().manual_seed(seed)
    return {k: torch.randn(s, generator=g) * 0.01 for k, s in esrgan_param_shapes(num_block).items()}


def _create(num_block=23, h=512, w=512, frames=1):
    from stable_diffusion_videos_b200 import _native
    from stable_diffusion_videos_b200.upsampling import UpsamplerConfig

    lib = _native.lib()
    cfg = UpsamplerConfig(64, num_block, 32, h, w, frames)
    eng = C.c_void_p()
    _native.check(lib.sdw_upsampler_create(C.byref(cfg), C.byref(eng)))
    return lib, eng


def test_param_count_and_key_table_match_the_native_registry():
    from oracle.esrgan import rrdbnet
    from stable_diffusion_videos_b200.configs import esrgan_param_shapes

    shapes = esrgan_param_shapes(23)
    assert sum(math.prod(s) for s in shapes.values()) == 16_697_987
    # the oracle consumes this table: a 1-block network runs on it, and it needs every key of it
    sd = _oracle_state_dict(1)
    y = rrdbnet(torch.rand(1, 3, 4, 4), sd, 1)
    assert y.shape == (1, 3, 16, 16)
    for k in sd:
        with pytest.raises(KeyError):
            rrdbnet(torch.rand(1, 3, 4, 4), {j: v for j, v in sd.items() if j != k}, 1)
    lib, eng = _create(23)
    try:
        from stable_diffusion_videos_b200 import _native

        got = {}
        name, numel = C.c_char_p(), C.c_int64()
        for i in range(lib.sdw_upsampler_num_params(eng)):
            _native.check(lib.sdw_upsampler_param_info(eng, i, C.byref(name), C.byref(numel)))
            got[name.value.decode()] = numel.value
        assert got == {k: math.prod(s) for k, s in shapes.items()}
        assert list(got) == list(shapes)  # registration order too
    finally:
        lib.sdw_upsampler_destroy(eng)


def test_arena_size_and_bad_configs():
    from stable_diffusion_videos_b200.upsampling import UpsamplerConfig

    lib, eng = _create(23, 512, 512, 1)
    n = C.c_uint64()
    assert lib.sdw_upsampler_arena_bytes(eng, C.byref(n)) == 0
    lib.sdw_upsampler_destroy(eng)
    # two 2048^2 x 64 fp16 maps (1.07 GB) plus ~34 MB of packed weights
    assert 1.05e9 < n.value < 1.2e9, n.value
    lib2, eng2 = _create(6, 512, 512, 2)
    lib2.sdw_upsampler_arena_bytes(eng2, C.byref(n))
    lib2.sdw_upsampler_destroy(eng2)
    assert 2.1e9 < n.value < 2.2e9, n.value
    h = C.c_void_p()
    for bad in (UpsamplerConfig(32, 23, 32, 64, 64, 1), UpsamplerConfig(64, 23, 16, 64, 64, 1),
                UpsamplerConfig(64, 0, 32, 64, 64, 1), UpsamplerConfig(64, 23, 32, 64, 64, 0)):
        assert lib.sdw_upsampler_create(C.byref(bad), C.byref(h)) == 1


def _desc(N, C_=64, W=64, H=64, B=1, **kw):
    from stable_diffusion_videos_b200._native import GemmDesc

    d = GemmDesc()
    d.A, d.C, d.W, d.H, d.B = 1 << 30, C_, W, H, B
    d.sW, d.sH, d.sB = C_, W * C_, W * H * C_
    d.conv = 1
    d.Wt, d.N = 2 << 30, N
    d.out, d.ldc = 3 << 30, N
    d.alpha = 1.0
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def test_block_n_32_planner_rules():
    from stable_diffusion_videos_b200 import _native

    lib = _native.lib()
    lib.sdw_debug_plan_only(1)
    try:
        out = (C.c_int32 * 12)()
        # explicit BLOCK_N 32 on single CTAs (also when the version is left to the planner)
        for ver in (1, 0):
            assert lib.sdw_debug_plan(C.byref(_desc(32, bn=32, ver=ver)), out) == 0
            assert out[0] == 1 and out[1] == 32
        assert lib.sdw_debug_plan(C.byref(_desc(256, bn=32, ver=0)), out) == 0 and out[0] == 1
        # never on CTA pairs
        assert lib.sdw_debug_plan(C.byref(_desc(256, bn=32, ver=2)), out) == 1
        assert b"BLOCK_N" in lib.sdw_last_error()
        # the automatic plan of an existing N = 32 shape is unchanged: single CTAs, BLOCK_N 64
        assert lib.sdw_debug_plan(C.byref(_desc(32)), out) == 0
        assert out[0] == 1 and out[1] == 64
        # C = 96 / 160 reads of a 192-pitch dense-block buffer into a 32-channel slice
        for c in (96, 160):
            d = _desc(32, C_=c, bn=32, ver=1, act=2)
            d.sW, d.sH, d.sB, d.ldc = 192, 64 * 192, 64 * 64 * 192, 192
            d.out = (3 << 30) + 2 * c
            assert lib.sdw_debug_plan(C.byref(d), out) == 0 and out[1] == 32
        # activations: 3 is not one
        assert lib.sdw_debug_plan(C.byref(_desc(64, act=3)), out) == 1
    finally:
        lib.sdw_debug_plan_only(0)


@pytest.mark.parametrize("num_block,hw,frames", [(23, (512, 512), 2), (1, (37, 53), 3), (2, (8, 8), 1)])
def test_op_list_plans_without_a_gpu(num_block, hw, frames):
    """bind() plans every GEMM of the static op list (tensor maps validated, not encoded; nothing launched)."""
    from stable_diffusion_videos_b200 import _native

    lib, eng = _create(num_block, hw[0], hw[1], frames)
    lib.sdw_debug_plan_only(1)
    try:
        n = C.c_uint64()
        _native.check(lib.sdw_upsampler_arena_bytes(eng, C.byref(n)))
        _native.check(lib.sdw_upsampler_bind(eng, C.c_void_p(1 << 40), n))
    finally:
        lib.sdw_debug_plan_only(0)
        lib.sdw_upsampler_destroy(eng)


# ---- checkpoint loading -----------------------------------------------------------------------
def _tiny_sd():
    from stable_diffusion_videos_b200.configs import esrgan_param_shapes

    return {k: torch.zeros(s) for k, s in esrgan_param_shapes(2).items()}


@pytest.mark.parametrize("wrap", [None, "params_ema", "params"])
def test_from_pretrained_file_and_directory(tmp_path, wrap):
    from stable_diffusion_videos_b200.upsampling import HUB_FILENAME, RealESRGANModel

    sd = _tiny_sd()
    sd["conv_last.bias"] = torch.tensor([1.0, 2.0, 3.0])
    obj = sd if wrap is None else {wrap: sd}
    if wrap == "params_ema":  # params_ema wins over params, as in RealESRGANer
        obj["params"] = {"junk": torch.zeros(1)}
    torch.save(obj, tmp_path / HUB_FILENAME)
    for src in (tmp_path / HUB_FILENAME, str(tmp_path / HUB_FILENAME), tmp_path):
        m = RealESRGANModel.from_pretrained(src)
        assert m.num_block == 2 and m.state["conv_last.bias"].tolist() == [1.0, 2.0, 3.0]
        assert m.state["conv_last.bias"].dtype == torch.float16


def test_from_pretrained_hub_id_uses_hf_hub_download(tmp_path, monkeypatch):
    import huggingface_hub

    from stable_diffusion_videos_b200.upsampling import HUB_FILENAME, RealESRGANModel

    torch.save({"params_ema": _tiny_sd()}, tmp_path / "local.pth")
    calls = []

    def fake_download(repo_id, filename, **kw):
        calls.append((repo_id, filename))
        return str(tmp_path / "local.pth")

    monkeypatch.setattr(huggingface_hub, "hf_hub_download", fake_download)
    m = RealESRGANModel.from_pretrained()
    assert calls == [("nateraw/real-esrgan", HUB_FILENAME)] and m.num_block == 2


@pytest.mark.parametrize("edit", ["missing", "extra", "shape"])
def test_from_pretrained_is_strict(tmp_path, edit):
    from stable_diffusion_videos_b200.upsampling import RealESRGANModel

    sd = _tiny_sd()
    if edit == "missing":
        del sd["body.1.rdb3.conv5.bias"]
    elif edit == "extra":
        sd["body.1.rdb3.conv6.bias"] = torch.zeros(64)
    else:
        sd["conv_hr.weight"] = torch.zeros(64, 64, 1, 1)
    torch.save({"params_ema": sd}, tmp_path / "m.pth")
    with pytest.raises((KeyError, ValueError)):
        RealESRGANModel.from_pretrained(tmp_path / "m.pth")


def test_from_random_initialisation():
    from stable_diffusion_videos_b200.upsampling import RealESRGANModel

    m = RealESRGANModel.from_random(seed=3, num_block=2)
    w = m.state["body.0.rdb1.conv1.weight"].float()
    assert abs(w.std().item() - 0.1 * math.sqrt(2 / (64 * 9))) < 2e-3
    assert m.state["body.0.rdb1.conv1.bias"].abs().max() == 0
    assert m.state["conv_first.weight"].abs().max() <= 1 / math.sqrt(27) + 1e-3
    assert torch.equal(m.state["conv_hr.weight"], RealESRGANModel.from_random(seed=3, num_block=2).state["conv_hr.weight"])


@pytest.mark.parametrize("kw", [dict(tile=128), dict(pre_pad=10), dict(fp32=True)])
def test_unsupported_options_raise(kw):
    from stable_diffusion_videos_b200.upsampling import RealESRGANModel

    with pytest.raises(NotImplementedError):
        RealESRGANModel(state_dict=_tiny_sd(), **kw)


def test_tiled_pipeline_with_upsample_raises(tmp_path):
    from stable_diffusion_videos_b200.pipeline import StableDiffusionWalkPipeline

    pipe = StableDiffusionWalkPipeline.__new__(StableDiffusionWalkPipeline)
    pipe.unet = pipe.vae = None
    pipe.tiled, pipe.upsampler = True, None
    with pytest.raises(NotImplementedError):
        pipe.make_clip_frames("a", "b", 0, 1, num_interpolation_steps=2, save_path=tmp_path, height=64, width=64,
                              upsample=True)


def test_u8_pre_and_post_processing_of_the_oracle():
    """x = fp16(u / 255) and out = round(clamp(y, 0, 1) * 255): the identity-like 1-block network with zero weights maps
    every frame to a constant from the biases."""
    from oracle.esrgan import upsample_u8

    sd = {k: torch.zeros_like(v) for k, v in _oracle_state_dict(1).items()}
    sd["conv_last.bias"] = torch.tensor([-0.1, 0.5, 1.2])
    u8, y = upsample_u8(np.zeros((1, 3, 5, 3), np.uint8), sd, 1)
    assert u8.shape == (1, 12, 20, 3) and (u8[..., 0] == 0).all() and (u8[..., 1] == 128).all()
    assert (u8[..., 2] == 255).all() and np.allclose(y[..., 2], 1.2)
