"""The native safety checker on the GPU: preprocessing bit-exact with Pillow, the image tower against the fp64 restatement
(tests/_safety_oracle.py) with the fp16-storage calibration, the score kernel bit-exact with diffusers' loop, the whole
checker's flags, and the pipeline's filtering in __call__ and walk."""
import numpy as np
import pytest
import torch
from PIL import Image

import _safety_oracle as so

pytestmark = pytest.mark.gpu

SIZES = [(512, 512), (768, 768), (512, 768), (768, 512), (576, 1024), (64, 64)]
TINY14 = dict(hidden_size=128, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2, image_size=224,
              patch_size=14, hidden_act="quick_gelu", layer_norm_eps=1e-5)


def _checker(vision, sd, max_batch=8):
    from stable_diffusion_videos_b200.safety import NativeSafetyChecker

    return NativeSafetyChecker.from_state_dict(sd, vision, max_batch=max_batch, device="cuda")


@pytest.fixture(scope="module")
def tiny():
    model, cfg = so.hf_vision(TINY14, trained_like=True, seed=1)
    sd = so.checker_state_dict(model, proj=64, seed=1)
    return _checker(TINY14, sd), sd, TINY14


# ---- preprocessing --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hw", SIZES)
def test_preprocess_is_pillow_exact(tiny, hw):
    from transformers import CLIPImageProcessorPil

    chk = tiny[0]
    u8 = so.test_frames(3, *hw, seed=hw[0] * 7 + hw[1])
    pix, crop = chk.preprocess(torch.from_numpy(u8).cuda())
    want = np.stack([so.resize_crop_u8(f) for f in u8])
    assert np.array_equal(crop.cpu().numpy(), want)
    ref = CLIPImageProcessorPil()([f for f in u8], return_tensors="np")["pixel_values"].transpose(0, 2, 3, 1)
    ref16 = torch.from_numpy(np.ascontiguousarray(ref)).half()
    ulp = (ref16.float().abs().clamp(min=2 ** -14) * 2 ** -10)
    assert ((pix.cpu().float() - ref16.float()).abs() <= ulp).all()


def test_patch_rows_pad_columns_are_zero(tiny):
    from stable_diffusion_videos_b200 import _native

    chk = tiny[0]
    u8 = torch.from_numpy(so.test_frames(2, 96, 128)).cuda()
    rows = torch.full((2 * 256, 640), float("nan"), dtype=torch.float16, device="cuda")
    _native.safety_patch_rows(chk._h, u8, rows)
    torch.cuda.synchronize()
    assert (rows[:, 588:] == 0).all() and torch.isfinite(rows[:, :588]).all()
    pix, _ = chk.preprocess(u8)
    # row 17 = sample 0, patch (1, 1): columns (c, ky, kx)
    want = pix[0, 14:28, 14:28, :].permute(2, 0, 1).reshape(-1)
    assert torch.equal(rows[17, :588], want)


# ---- the tower ------------------------------------------------------------------------------------------------------
def _errs(got, ref):
    e = (got - ref).abs()
    return float((got - ref).norm() / ref.norm()), float(torch.quantile((e / ref.abs().clamp(min=1)).flatten(), 0.999))


@pytest.mark.parametrize("name", ["tiny14", "ViT-L/14-2"])
@pytest.mark.parametrize("trained_like", [False, True])
@pytest.mark.parametrize("B,max_batch", [(1, 8), (3, 8), (5, 2)])
def test_tower_against_fp64(name, trained_like, B, max_batch):
    kw = TINY14 if name == "tiny14" else so.VISION["ViT-L/14"]
    model, cfg = so.hf_vision(kw, trained_like=trained_like, seed=2, layers=None if name == "tiny14" else 2)
    sd = so.checker_state_dict(model, seed=2)
    chk = _checker(cfg, sd, max_batch=max_batch)
    u8 = so.test_frames(B, 512, 512, seed=B)
    got = chk.image_embeds(torch.from_numpy(u8).cuda()).double().cpu()
    x = so.preprocess(u8)
    ref = so.vision_tower(x, sd, cfg)
    o16 = so.vision_tower(x, sd, cfg, fp16_storage=True)
    (rn, pn), (ro, po) = _errs(got, ref), _errs(o16, ref)
    print(f"tower {name} trained_like={trained_like} B={B}: rel-L2 ratio {rn / ro:.2f}, p99.9 ratio {pn / po:.2f}")
    assert rn <= 1.25 * ro and pn <= 1.25 * po, (rn, ro, pn, po)


def test_graph_replay_equals_eager(tiny):
    chk = tiny[0]
    u8 = torch.from_numpy(so.test_frames(5, 256, 320, seed=9)).cuda()
    a = chk.image_embeds(u8, use_graph=True)
    b = chk.image_embeds(u8, use_graph=False)
    c = chk.image_embeds(u8, use_graph=True)
    assert torch.equal(a, b) and torch.equal(a, c)


# ---- scores ---------------------------------------------------------------------------------------------------------
def test_scores_match_the_diffusers_loop_bit_for_bit():
    from stable_diffusion_videos_b200 import _native

    g = torch.Generator().manual_seed(0)
    D, ns, nc, B = 768, 3, 17, 8
    emb = torch.randn(B, D, generator=g)
    special, concepts = torch.randn(ns, D, generator=g), torch.randn(nc, D, generator=g)
    concepts[:6] = emb[:6] + 0.3 * torch.randn(6, D, generator=g)  # cosines well above 0
    special[0] = emb[5] + 0.3 * torch.randn(D, generator=g)
    sw, cw = torch.full((ns,), 0.9), torch.full((nc,), 0.9)
    dev = [t.cuda() for t in (emb, special, sw, concepts, cw)]
    _, cos, _ = _native.safety_scores(*dev)
    cos = cos.cpu()
    # image 0: concept 0 scores exactly 0 (threshold = its own cosine): not flagged
    cw[0] = cos[0, ns + 0]
    # images 1, 2: scores 0.0005 -+ 1e-6 (rounds to 0.0 / 0.001); image 3: -0.0005 - 1e-6
    cw[1] = float(cos[1, ns + 1]) - 0.0005 + 1e-6
    cw[2] = float(cos[2, ns + 2]) - 0.0005 - 1e-6
    cw[3] = float(cos[3, ns + 3]) + 0.0005 + 1e-6
    # image 5: special concept 0 fires, lifting concept 5 from (-0.01, 0] to flagged
    sw[0] = float(cos[5, 0]) - 0.2
    cw[5] = float(cos[5, ns + 5]) + 0.006
    cw[4] = 1.0
    # images 4, 6, 7: nothing flagged
    sd = {"special_care_embeds_weights": sw, "concept_embeds_weights": cw}
    frames = torch.full((B, 4, 5, 3), 7, dtype=torch.uint8, device="cuda")
    flags, cos2, scores = _native.safety_scores(emb.cuda(), special.cuda(), sw.cuda(), concepts.cuda(), cw.cuda(), frames)
    want_flags, want_scores = so.decide(None, sd, cos=cos2.cpu())
    assert torch.equal(cos2.cpu(), cos)
    assert np.array_equal(flags.cpu().numpy().astype(bool), want_flags)
    assert np.array_equal(scores.cpu().numpy(), want_scores)  # bit-identical float64
    assert want_flags.tolist() == [False, False, True, False, False, True, False, False]
    assert want_scores[0, ns] == 0.0 and want_scores[5, 0] > 0
    fr = frames.cpu().numpy()
    assert (fr[want_flags] == 0).all() and (fr[~want_flags] == 7).all()
    # the fp32 cosines against float64
    assert torch.allclose(cos, so.cosines(emb, {"special_care_embeds": special, "concept_embeds": concepts}),
                          rtol=0, atol=2e-6)


# ---- the whole checker ----------------------------------------------------------------------------------------------
def _concepts_for(embeds, flagged, sd, margin=0.05, nc=17, ns=3):
    """concept tables under which exactly `flagged` (indices of `embeds`) are flagged, each at least `margin` above its
    concept's threshold while every other image stays at least `margin` below every threshold.  Concept k points from
    the nearest point of the convex hull of the unflagged images' unit embeddings to image k's, which maximises that
    gap; the threshold sits in the middle.  Margins are measured on the fp16 tables the checker is handed."""
    from scipy.optimize import nnls

    E = torch.nn.functional.normalize(torch.as_tensor(embeds).double(), dim=1)
    rest = [i for i in range(E.shape[0]) if i not in flagged]
    sd = dict(sd)
    g = torch.Generator().manual_seed(7)
    P = E.shape[1]
    concepts = torch.randn(nc, P, generator=g, dtype=torch.float64)
    cw = torch.full((nc,), 1.0, dtype=torch.float64)  # unreachable
    R = E[rest].numpy()
    for j, k in enumerate(flagged):
        lam, _ = nnls(np.vstack([R.T, 1e3 * np.ones((1, len(rest)))]), np.concatenate([E[k].numpy(), [1e3]]))
        c = E[k] - torch.from_numpy(R.T @ lam)
        concepts[j] = (c / c.norm()).half().double()
        above, below = float(E[k] @ concepts[j]), float((E[rest] @ concepts[j]).max())
        cw[j] = (above + below) / 2
    sd["concept_embeds"] = concepts.float().half().float()
    sd["concept_embeds_weights"] = cw.float().half().float()
    sd["special_care_embeds"] = torch.randn(ns, P, generator=g).half().float()
    sd["special_care_embeds_weights"] = torch.full((ns,), 1.0)
    cos = so.cosines(torch.as_tensor(embeds), sd).double()[:, ns:] - sd["concept_embeds_weights"].double()
    got = min(min(float(cos[k, j]) for j, k in enumerate(flagged)), -float(cos[rest].max()))
    assert got >= margin, got
    return sd


def test_whole_checker_flags_match_the_oracle():
    model, cfg = so.hf_vision(TINY14, trained_like=True, seed=3)
    sd = so.checker_state_dict(model, seed=3)
    u8 = so.test_frames(6, 512, 512, seed=3)
    ref = so.vision_tower(so.preprocess(u8), sd, cfg)
    sd = _concepts_for(ref, [1, 2], sd, margin=0.05)
    want, _ = so.decide(ref, sd)
    assert want.tolist() == [False, True, True, False, False, False]
    chk = _checker(cfg, sd, max_batch=4)
    frames = torch.from_numpy(u8).cuda()
    flags, cos = chk.scores(frames)
    assert flags.cpu().numpy().tolist() == want.tolist()
    assert so.decide(None, sd, cos=cos.cpu())[0].tolist() == want.tolist()
    # eager tower + score kernel = the graph-replayed checker, bit for bit
    from stable_diffusion_videos_b200 import _native

    emb = chk.image_embeds(frames, use_graph=False)
    f2, cos2, _ = _native.safety_scores(emb, *(sd[k].cuda() for k in ("special_care_embeds",
                                                                       "special_care_embeds_weights", "concept_embeds",
                                                                       "concept_embeds_weights")))
    assert torch.equal(cos2, cos) and torch.equal(f2.bool(), flags)
    out = chk.check_frames(frames.clone(), blackout=False)
    assert torch.equal(out, flags)
    blk = frames.clone()
    chk.check_frames(blk, blackout=True)
    assert (blk[flags] == 0).all() and torch.equal(blk[~flags], frames[~flags])


# ---- the pipeline ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pipe():
    from _helpers import TINY_UNET, TINY_VAE, make_oracle, product_cfgs

    from stable_diffusion_videos_b200.pipeline import (NativeUNet, NativeVAE, StableDiffusionWalkPipeline,
                                                       SyntheticTextEncoder, SyntheticTokenizer)
    from stable_diffusion_videos_b200.schedulers import PNDMScheduler

    unet, vae = make_oracle(TINY_UNET, TINY_VAE)
    ucfg, vcfg = product_cfgs(TINY_UNET, TINY_VAE)
    usd = {k: v.half() for k, v in unet.state_dict().items()}
    vsd = {k: v.half() for k, v in vae.state_dict().items()}
    parts = (NativeVAE(vcfg, vsd), SyntheticTextEncoder(TINY_UNET.cross_attention_dim), SyntheticTokenizer(),
             NativeUNet(ucfg, usd), PNDMScheduler())
    plain = StableDiffusionWalkPipeline(*parts).to("cuda")
    model, cfg = so.hf_vision(TINY14, trained_like=True, seed=4)
    return plain, parts, so.checker_state_dict(model, seed=4)


def _with_checker(parts, sd, frames, flagged):
    from stable_diffusion_videos_b200.pipeline import StableDiffusionWalkPipeline

    probe = _checker(TINY14, sd)
    emb = probe.image_embeds(torch.from_numpy(np.ascontiguousarray(frames)).cuda()).cpu()
    sd = _concepts_for(emb, flagged, sd, margin=0.01)  # pipeline frames: flags only need to be unambiguous
    chk = _checker(TINY14, sd, max_batch=2)
    return StableDiffusionWalkPipeline(*parts, safety_checker=chk, feature_extractor={}).to("cuda"), sd


def test_call_blacks_out_flagged_images(pipe):
    plain, parts, sd = pipe
    kw = dict(height=64, width=64, num_inference_steps=3)
    g = lambda: torch.Generator(device="cuda").manual_seed(5)  # noqa: E731
    base = plain(["0", "1", "2"], generator=g(), **kw)
    assert base.nsfw_content_detected is None
    frames = np.stack([np.asarray(im) for im in base.images])
    p, _ = _with_checker(parts, sd, frames, [1])
    out = p(["0", "1", "2"], generator=g(), **kw)
    assert out.nsfw_content_detected == [False, True, False]
    got = np.stack([np.asarray(im) for im in out.images])
    assert (got[1] == 0).all() and np.array_equal(got[[0, 2]], frames[[0, 2]])
    arr = p(["0", "1", "2"], generator=g(), output_type="np", **kw)
    assert arr.nsfw_content_detected == [False, True, False] and (arr.images[1] == 0).all() and arr.images[0].max() > 0
    tup = p(["0", "1", "2"], generator=g(), return_dict=False, **kw)
    assert tup[1] == [False, True, False] and all(np.array_equal(np.asarray(a), np.asarray(b))
                                                  for a, b in zip(tup[0], out.images))


def _read(root):
    files = sorted(p.relative_to(root).as_posix() for p in root.glob("**/*.png"))
    return files, np.stack([np.asarray(Image.open(root / f)) for f in files])


def test_walk_saves_flagged_frames_black(pipe, tmp_path):
    from stable_diffusion_videos_b200.upsampling import RealESRGANModel

    plain, parts, sd = pipe
    kw = dict(seeds=[42, 1337, 2022], num_interpolation_steps=[3, 3], fps=3, num_inference_steps=3, height=64,
              width=64, batch_size=2, make_video=False, output_dir=str(tmp_path))  # 3 frames per clip: a tail batch
    plain.walk(["0", "1", "2"], name="plain", **kw)
    files, base = _read(tmp_path / "plain")
    # a full batch's second frame and the last, tail-batch frame (frames 2 and 3 are the same image: clip 0 ends where
    # clip 1 starts)
    flagged = [1, 5]
    p, _ = _with_checker(parts, sd, base, flagged)
    p.walk(["0", "1", "2"], name="checked", **kw)
    f2, got = _read(tmp_path / "checked")
    assert [f.replace("checked", "plain") for f in f2] == files
    keep = [i for i in range(len(files)) if i not in flagged]
    assert (got[flagged] == 0).all() and np.array_equal(got[keep], base[keep])
    for i in keep:  # byte-identical files
        a = (tmp_path / "plain" / files[i]).read_bytes()
        assert a == (tmp_path / "checked" / f2[i]).read_bytes()
    # resume recomputes deleted frames through the checker
    clip = tmp_path / "checked" / "checked_000001"
    (clip / "frame000002.png").unlink()
    (clip / "frame000001.png").unlink()
    p.walk(name="checked", resume=True, output_dir=str(tmp_path), batch_size=2, make_video=False)
    _, again = _read(tmp_path / "checked")
    assert np.array_equal(again, got)
    # upsample=True: a flagged frame on disk is the upsampler applied to a black frame
    up = RealESRGANModel.from_random(4, num_block=1)
    plain.upsampler = p.upsampler = up
    p.walk(["0", "1", "2"], name="up", upsample=True, **kw)
    plain.walk(["0", "1", "2"], name="plain_up", upsample=True, **kw)
    _, gu = _read(tmp_path / "up")
    _, pu = _read(tmp_path / "plain_up")
    black = up.upsample_frames(torch.zeros((1, 16, 16, 3), dtype=torch.uint8, device="cuda")).cpu().numpy()[0]
    assert all(np.array_equal(gu[i], black) for i in flagged)
    assert np.array_equal(gu[keep], pu[keep])


def test_from_pretrained_loads_the_checker(pipe, tmp_path):
    import json

    import _fake_checkpoint as fc
    from safetensors.torch import save_file

    from stable_diffusion_videos_b200.pipeline import StableDiffusionWalkPipeline

    _, _, sd = pipe
    fc.write_checkpoint(str(tmp_path))
    (tmp_path / "safety_checker").mkdir()
    (tmp_path / "feature_extractor").mkdir()
    u8 = so.test_frames(4, 64, 64, seed=11)
    probe = _checker(TINY14, sd)
    sd = _concepts_for(probe.image_embeds(torch.from_numpy(u8).cuda()).cpu(), [0, 3], sd, margin=0.01)
    sd["vision_model.vision_model.embeddings.position_ids"] = torch.arange(257)[None]
    save_file({k: v.half().contiguous() if v.is_floating_point() else v.contiguous() for k, v in sd.items()},
              str(tmp_path / "safety_checker" / "model.safetensors"))
    json.dump({"projection_dim": 768, "vision_config": TINY14},
              open(tmp_path / "safety_checker" / "config.json", "w"))
    json.dump({"crop_size": 224, "do_center_crop": True, "do_normalize": True, "do_resize": True, "resample": 3,
               "size": 224, "image_mean": list(so.CLIP_MEAN), "image_std": list(so.CLIP_STD)},
              open(tmp_path / "feature_extractor" / "preprocessor_config.json", "w"))
    p = StableDiffusionWalkPipeline.from_pretrained(str(tmp_path), safety_checker=True)
    hand = _checker(TINY14, {k: v for k, v in sd.items() if not k.endswith("position_ids")})
    frames = torch.from_numpy(u8).cuda()
    want = hand.check_frames(frames.clone(), blackout=False)
    assert want.cpu().tolist() == [True, False, False, True]
    assert torch.equal(p.safety_checker.check_frames(frames.clone(), blackout=False), want)
    assert StableDiffusionWalkPipeline.from_pretrained(str(tmp_path)).safety_checker is None
