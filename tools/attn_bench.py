"""Micro-benchmark of the fused attention kernel on the SD-1.4 shapes (CUDA events, warm)."""
import ctypes as C
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from stable_diffusion_videos_b200 import _native as n  # noqa: E402


def bench(B, heads, Nq, Nk, d, iters=10):
    Cc = heads * d
    q = torch.randn(B, Nq, Cc, device="cuda").half()
    k = torch.randn(B, Nk, Cc, device="cuda").half()
    vt_ld = (Nk + 7) // 8 * 8
    vt = torch.randn(B, heads, d, vt_ld, device="cuda").half()
    out = torch.empty(B, Nq, Cc, device="cuda", dtype=torch.float16)

    def run():
        n.check(n.lib().sdw_attention(n.ptr(q), C.c_int64(Cc), n.ptr(k), C.c_int64(Cc), n.ptr(vt), C.c_int64(vt_ld),
                                      B, Nq, Nk, heads, d, n.ptr(out), C.c_int64(Cc), n.stream_ptr()))
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        run()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    flop = 4.0 * B * heads * Nq * Nk * d
    pairs = B * heads * Nq * Nk
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    mufu_floor_us = pairs / (16 * n_sm * 1.98e9) * 1e6  # one ex2 per score, 16 / clk / SM at the 1980 MHz boost clock
    return ms, flop / ms / 1e9, mufu_floor_us


if __name__ == "__main__":
    F = int(os.environ.get("F", "8"))
    shapes = [("self 64x64 d40", 2 * F, 8, 4096, 4096, 40), ("cross 64x64 d40", 2 * F, 8, 4096, 77, 40),
                                  ("self 32x32 d80", 2 * F, 8, 1024, 1024, 80), ("self 16x16 d160", 2 * F, 8, 256, 256, 160),
              ("cross 32x32 d80", 2 * F, 8, 1024, 77, 80)]
    if os.environ.get("ONLY_SELF"):  # A/B runs of the dominant shape only
        shapes = shapes[:1]
    for name, B, h, Nq, Nk, d in shapes:
        ms, tf, floor = bench(B, h, Nq, Nk, d)
        print(f"{name:18s} B={B:3d} {ms*1e3:9.1f} us {tf:8.1f} TFLOP/s  (all-MUFU exp floor {floor:7.1f} us)", flush=True)
