"""The sampler at the benchmarked batch: full SD-1.4 at 64 x 64 latents (512 x 512 frames), F = 30 frames per call
(UNet batch 60, VAE batch 30), PNDM-10, guidance 7.5, replayed as a CUDA graph, with the fp16-rounded seed-0 weights of
tests/golden/make_golden_full.py.

(a) Against the fp32 oracle without new fixtures: the `full_pndm10_f2` inputs with T tiled 15 times; every frame pair
    (2j, 2j + 1) meets tests/test_golden_full_gpu.py's criteria (TOL_X x the calibrated spread) against the fixture pair.
    Inside the batch, frames with the same inputs are bit-identical: no op mixes samples or depends on where a sample
    sits in the batch.
(b) Frames stay independent: 30 distinct frames, each with its own negative embedding ([F, 77, D] unconditional batch),
    match the same frame sampled by a 1-frame engine: uint8 frames within 2 LSB, latents rel-L2 within TOL_X x the
    calibrated fp16-storage spread.  The two engines differ in reduction order only (GroupNorm chunk counts, GEMM
    plans), but with fp16 activations one changed rounding anywhere spreads through the remaining layers and steps:
    measured on an H100 80GB HBM3 (700 W), every frame sits at 1.29e-3 .. 1.34e-3 latents rel-L2 (1.0 x the calibrated
    spread, 1.29e-3) and 1 LSB, so half the spread is not a bound this sampler meets.
(c) Two graph replays of the 30-frame engine are bit-identical.
(d) Tiled mode: `debug_vae` of a tiled 30-frame engine matches the 1-frame tiled decode of each frame (frames within
    2 LSB, raw rel-L2 within TOL_X x the calibrated raw spread; measured 1.04e-3 .. 1.06e-3 and 1 LSB); it pads and
    crops 4 GB activations.
"""
import gc
import json
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
G = os.path.join(HERE, "golden")
sys.path.insert(0, G)

pytestmark = pytest.mark.gpu

F = 30
CASE = "full_pndm10_f2"
TOL_X = 1.25  # tests/test_golden_full_gpu.py
_CACHE = {}


def _cal():
    return json.load(open(os.path.join(G, "calibration.json")))[CASE]


def _weights():
    if "w" not in _CACHE:
        import make_golden_full as mg
        from _helpers import make_oracle, product_cfgs

        ou, ov = mg.model_cfgs("sd14")
        unet, vae = make_oracle(ou, ov, seed=0)
        _CACHE["w"] = (product_cfgs(ou, ov), unet.state_dict(), vae.state_dict())
    return _CACHE["w"]


def _engine(frames, tiled=False, steps=True):
    key = (frames, tiled)
    if key not in _CACHE:
        from stable_diffusion_videos_b200 import schedulers as S
        from stable_diffusion_videos_b200.engine import Engine

        (ucfg, vcfg), usd, vsd = _weights()
        eng = Engine(ucfg, vcfg, (64, 64), frames, ctx_tokens=77, tiled=tiled)
        eng.load_state_dict(usd, vsd)
        if steps:
            eng.set_scheduler(S.PNDMScheduler(), 10, 7.5)
        print(f"\nengine F={frames} tiled={tiled}: arena {eng._model.arena_bytes} bytes")
        _CACHE[key] = eng
    return _CACHE[key]


def _drop_engines():
    for k in [k for k in _CACHE if k != "w"]:
        del _CACHE[k]
    gc.collect()
    torch.cuda.empty_cache()


def _inputs(T, unc):
    import make_golden_full as mg
    from stable_diffusion_videos_b200 import _native

    inp = mg.case_inputs(CASE)
    lat, emb = _native.slerp_lerp_batch(inp["la"].cuda(), inp["lb"].cuda(), inp["ea"].cuda(), inp["eb"].cuda(),
                                        torch.tensor(T, dtype=torch.float32).cuda())
    return lat, emb, (inp["unc"] if unc is None else unc).half().cuda()


def _rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def test_30_frames_match_the_fp32_oracle():
    import make_golden_full as mg

    gold = np.load(os.path.join(G, CASE + ".npz"))
    cal = _cal()
    eng = _engine(F)
    lat, emb, unc = _inputs(list(mg.CASES[CASE]["T"]) * (F // 2), None)
    u8, fin = eng.sample(lat, emb, unc, use_graph=True, return_latents=True)
    _, raw = eng.sample(lat, emb, unc, use_graph=True, return_raw=True)
    torch.cuda.synchronize()
    u8, fin = u8.cpu().numpy(), fin.cpu().numpy()
    raw = raw.cpu().numpy()[:, ::mg.RAW_STRIDE, ::mg.RAW_STRIDE]
    assert np.isfinite(fin).all() and np.isfinite(raw).all()
    for i in range(2, F):
        assert np.array_equal(u8[i], u8[i % 2]) and np.array_equal(fin[i], fin[i % 2]), i
    gl, gf, gr = gold["latents"], gold["frames"], gold["raw"].astype(np.float32)
    worst = {}
    for j in range(F // 2):
        s = slice(2 * j, 2 * j + 2)
        d = np.abs(u8[s].astype(np.int32) - gf.astype(np.int32))
        got = {"latents_rel_l2": _rel(fin[s], gl), "raw_rel_l2": _rel(raw[s], gr), "frames_mean_lsb": float(d.mean()),
               "frames_p999_lsb": float(np.quantile(d, 0.999))}
        for k, v in got.items():
            worst[k] = max(worst.get(k, 0.0), v)
            assert v <= TOL_X * cal[k], (j, k, v, "limit", TOL_X * cal[k])
    print("\n(a) worst frame pair vs the fp32 oracle:", worst)


def test_30_frames_are_independent_of_the_batch():
    from oracle.pipeline import synthetic_embedding

    cal = _cal()
    D = 768
    uncs = torch.cat([synthetic_embedding(1000 + i, dim=D).half() for i in range(F)])
    T = np.linspace(0.0, 1.0, F)
    lat, emb, unc = _inputs(T, uncs)
    eng = _engine(F)
    u8, fin = eng.sample(lat, emb, unc, use_graph=True, return_latents=True)
    # (c) a second replay of the same graph: bit-identical
    u8b, finb = eng.sample(lat, emb, unc, use_graph=True, return_latents=True)
    torch.cuda.synchronize()
    assert torch.equal(u8, u8b) and torch.equal(fin, finb)
    _CACHE["fin30"] = fin
    one = _engine(1)
    rels, lsbs = [], []
    for i in range(F):
        u1, f1 = one.sample(lat[i:i + 1], emb[i:i + 1], unc[i:i + 1], use_graph=True, return_latents=True)
        torch.cuda.synchronize()
        rels.append(_rel(fin[i:i + 1].cpu().numpy(), f1.cpu().numpy()))
        lsbs.append(int((u8[i].int() - u1[0].int()).abs().max()))
    print(f"\n(b) F=30 vs F=1 per frame: latents rel-L2 max {max(rels):.3e} mean {np.mean(rels):.3e}; "
          f"uint8 max |diff| {max(lsbs)} (per frame {lsbs})")
    assert max(rels) <= TOL_X * cal["latents_rel_l2"], rels
    assert max(lsbs) <= 2, lsbs


def test_tiled_30_frame_decode_matches_single_frames():
    cal = _cal()
    fin = _CACHE.get("fin30")
    if fin is None:
        fin = torch.randn(F, 4, 64, 64, generator=torch.Generator().manual_seed(5)).cuda() * 6
    fin = fin.clone()
    _drop_engines()
    eng = _engine(F, tiled=True, steps=False)
    u8, raw = eng.debug_vae(fin)
    torch.cuda.synchronize()
    u8, raw = u8.cpu(), raw.cpu()
    _drop_engines()
    one = _engine(1, tiled=True, steps=False)
    rels, lsbs = [], []
    for i in range(F):
        u1, r1 = one.debug_vae(fin[i:i + 1])
        torch.cuda.synchronize()
        rels.append(_rel(raw[i].numpy(), r1[0].cpu().numpy()))
        lsbs.append(int((u8[i].int() - u1[0].cpu().int()).abs().max()))
    print(f"\n(d) tiled VAE F=30 vs F=1: raw rel-L2 max {max(rels):.3e}; uint8 max |diff| {max(lsbs)}; "
          f"peak device memory {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")
    _drop_engines()
    assert max(rels) <= TOL_X * cal["raw_rel_l2"], rels
    assert max(lsbs) <= 2, lsbs
