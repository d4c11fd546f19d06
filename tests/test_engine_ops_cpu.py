"""The engine's op listing (`sdw_engine_debug_ops`) is the engine: every line parses, the lines account for every kernel
launch `sdw_engine_launches` reports, and each GEMM / attention record re-plans, from its fields alone, to the plan the
engine holds.  The standalone replays of tests/test_engine_ops_gpu.py rebuild their launches from these records, so this
is what makes them run the engine's exact launches.  Plan-only mode on a fake arena: no GPU."""
from collections import Counter

import pytest

from _engine_ops import LAUNCHES, PLAN_FIELDS, attention_plan_of, gemm_desc, plan_of, plan_only_ops

KINDS = {"gemm", "attention", "groupnorm", "layernorm", "softmax_rows", "conv_in_small", "conv_out_small", "vae_in",
         "wrap_pad", "crop"}


@pytest.fixture(scope="module", params=[(1, False), (30, False), (30, True)], ids=["F1", "F30", "F30-tiled"])
def listing(request):
    F, tiled = request.param
    recs, launches, arena = plan_only_ops(F, tiled=tiled)
    return F, tiled, recs, launches, arena


def test_listing_covers_every_launch(listing):
    F, tiled, recs, launches, _ = listing
    assert recs and {k for _, _, k, _ in recs} <= KINDS
    for sec in ("unet", "vae"):
        lines = [r for r in recs if r[0] == sec]
        assert sum(LAUNCHES.get(k, 1) for _, _, k, _ in lines) == launches[sec], sec
        idx = sorted({i for _, i, _, _ in lines})
        assert idx == list(range(len(idx))), sec  # one record (or more) per op, none missing
    kinds = Counter(k for _, _, k, _ in recs)
    assert (kinds["wrap_pad"] > 0) == tiled and (kinds["crop"] > 0) == tiled
    # the VAE mid-block attention (d = 512) runs unfused in chunks of two samples: 15 QK^T / softmax / PV triples at F = 30
    assert kinds["softmax_rows"] == (F + 1) // 2
    vae_batched = [f for s, _, k, f in recs if s == "vae" and k == "gemm" and f["b_batched"]]
    assert len(vae_batched) == 2 * kinds["softmax_rows"] and all(f["B"] <= 2 for f in vae_batched)


def test_gemm_records_replan_to_the_engine_plan(listing):
    _, _, recs, _, _ = listing
    base = 1 << 40
    seen = 0
    for sec, i, kind, f in recs:
        if kind != "gemm":
            continue
        out = base + (8 << 30)
        d = gemm_desc(f, A=out if f["in_alias"] else base, Wt=base + (2 << 30), out=out, bias=base + (3 << 30),
                      rowvec=base + (4 << 30), resid=out if f["res_alias"] else base + (5 << 30), vt=base + (6 << 30))
        assert plan_of(d) == tuple(f[k] for k in PLAN_FIELDS), (sec, i, f)
        seen += 1
    assert seen > 100


def test_attention_records_replan_to_the_engine_plan(listing):
    _, _, recs, _, _ = listing
    att = [f for _, _, k, f in recs if k == "attention"]
    assert len(att) == 32  # 16 transformer blocks x (self, cross)
    for f in att:
        assert attention_plan_of(f) == (f["variant"], f["gx"], f["gy"], f["gz"]), f


def test_batch_30_records_scale_with_the_batch():
    """the F = 30 listing is the F = 1 listing with the batch scaled (UNet 60, VAE 30): same ops, same order, and the
    fields other than batch extents, batch strides and the planner's choices agree"""
    r1, _, _ = plan_only_ops(1)
    r30, _, a30 = plan_only_ops(30)
    assert len([r for r in r1 if r[0] == "unet"]) == len([r for r in r30 if r[0] == "unet"])
    for (s1, _, k1, f1), (s30, _, k30, f30) in zip([r for r in r1 if r[0] == "unet"], [r for r in r30 if r[0] == "unet"]):
        assert (s1, k1) == (s30, k30)
        if k1 == "gemm":
            assert (f1["C"], f1["N"], f1["conv"], f1["mode"], f1["ldc"]) == (f30["C"], f30["N"], f30["conv"], f30["mode"], f30["ldc"])
            assert f1["B"] * f1["W"] * 60 == f30["B"] * f30["W"] * 2
        elif k1 == "groupnorm":
            assert (f1["B"], f30["B"]) == (2, 60) and f1["P"] == f30["P"]
    assert 10e9 < a30 < 80e9  # the 30-frame engine fits an 80 GB card next to the CUDA context
