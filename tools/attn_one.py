"""one attention shape, a few launches — target for `ncu --set full -k regex:attn_kernel`."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from attn_bench import bench  # noqa: E402

if __name__ == "__main__":
    B, h, Nq, Nk, d = [int(v) for v in os.environ.get("SHAPE", "16,8,4096,4096,40").split(",")]
    ms, tf, floor = bench(B, h, Nq, Nk, d, iters=2)
    print(f"{ms*1e3:.1f} us {tf:.1f} TFLOP/s")
