"""End-to-end GPU parity at the BENCHMARKED configuration (BASELINE.json configs[1]: SD-1.4 full widths, 64x64 latents,
512x512 frames) and the named sampler/model variants (configs[3] SD-2.1 numerics, configs[4] K-LMS / guidance 15),
against committed oracle fixtures (tests/golden/<case>.npz, generator tests/golden/make_golden_full.py).

The loop under test is stable_diffusion_pipeline.py:412-438 (51 UNet calls for PNDM-50, CFG, scheduler.step, VAE decode,
post-process) through the C ABI (`sdw_engine_sample`, CUDA graph replay).

Tolerances are CALIBRATED (SURVEY.md §8d): tests/golden/calibration.json records, per case, the spread between the fp32
oracle and the same oracle with fp16 storage emulation (what the reference's own fp16 CUDA pipeline stores).  The native
path (fp16 activations, fp32 accumulate, fp32 latent state) must sit within TOL_X x that spread of the fp32 oracle.
With SDW_PARITY_DIR set, the measured metrics of each case are written there as parity_<case>.json.
"""
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

TOL_X = 1.25  # native-vs-oracle error allowed as a multiple of the calibrated fp16-storage spread
FLOOR = {"latents_rel_l2": 0.0, "raw_rel_l2": 0.0, "frames_mean_lsb": 0.0, "frames_p999_lsb": 1.0}  # no slack beyond TOL_X x spread


def _run_native(case):
    import make_golden_full as mg
    from _helpers import make_oracle, product_cfgs
    from stable_diffusion_videos_b200 import _native
    from stable_diffusion_videos_b200.engine import Engine
    from stable_diffusion_videos_b200 import schedulers as S

    c = mg.CASES[case]
    ou, ov = mg.model_cfgs(c["model"])
    unet, vae = make_oracle(ou, ov, seed=0)  # the same fp16-rounded weights the fixture run used
    ucfg, vcfg = product_cfgs(ou, ov)
    inp = mg.case_inputs(case)
    F = len(c["T"])
    eng = Engine(ucfg, vcfg, c["hw"], F, ctx_tokens=77)
    eng.load_state_dict(unet.state_dict(), vae.state_dict())
    del unet, vae
    sched = {"pndm": S.PNDMScheduler, "lms": S.LMSDiscreteScheduler, "ddim": S.DDIMScheduler,
             "ddim_v": lambda: S.DDIMScheduler(prediction_type="v_prediction")}[c["sched"]]()
    eng.set_scheduler(sched, c["steps"], c["guidance"])
    # inputs through the product's own slerp/lerp kernel (generate_inputs, P:457-479)
    T = torch.tensor(inp["T"], dtype=torch.float32).cuda()
    lat, emb = _native.slerp_lerp_batch(inp["la"].cuda(), inp["lb"].cuda(), inp["ea"].cuda(), inp["eb"].cuda(), T)
    unc = inp["unc"].half().cuda()
    u8, fin = eng.sample(lat, emb, unc, use_graph=True, return_latents=True)
    _, raw = eng.sample(lat, emb, unc, use_graph=True, return_raw=True)
    torch.cuda.synchronize()
    return u8.cpu().numpy(), fin.cpu().numpy(), raw.cpu().numpy()[:, ::mg.RAW_STRIDE, ::mg.RAW_STRIDE]


@pytest.mark.parametrize("case", ["full_pndm10_f2", "full_pndm50_f1", "full_lms50_f1", "sd21_ddim50_f1"])
def test_native_matches_full_size_golden(case):
    path = os.path.join(G, case + ".npz")
    if not os.path.exists(path):
        pytest.fail(f"fixture {path} missing: run tests/golden/make_golden_full.py {case}")
    gold = np.load(path)
    cal = json.load(open(os.path.join(G, "calibration.json")))[case]
    u8, fin, raw = _run_native(case)
    assert np.isfinite(fin).all() and np.isfinite(raw).all()
    gl, gf, gr = gold["latents"], gold["frames"], gold["raw"].astype(np.float32)
    d = np.abs(u8.astype(np.int32) - gf.astype(np.int32))
    got = {
        "latents_rel_l2": float(np.linalg.norm(fin - gl) / np.linalg.norm(gl)),
        "raw_rel_l2": float(np.linalg.norm(raw - gr) / np.linalg.norm(gr)),
        "frames_mean_lsb": float(d.mean()),
        "frames_p999_lsb": float(np.quantile(d, 0.999)),
        "frames_max_lsb": int(d.max()),
        "frames_frac_within_2": float((d <= 2).mean()),
    }
    out_dir = os.environ.get("SDW_PARITY_DIR")
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, f"parity_{case}.json"), "w") as f:
            json.dump({"native_vs_fp32_oracle": got, "fp16_storage_oracle_vs_fp32_oracle": cal}, f, indent=1)
    for k, floor in FLOOR.items():
        limit = max(TOL_X * cal[k], floor)
        assert got[k] <= limit, (case, k, got[k], "limit", limit, "calibrated spread", cal[k])
