"""Before / after comparison of two built trees of this project on one GPU, alternating them so that drift of the clock
or of other work on the host hits both alike.

Usage: python tools/ab_compare.py OLD_TREE NEW_TREE OUT_DIR [--bench-runs 2] [--F 30]

Each tree must have been built (`__graft_entry__.build()` or `build.py`) and is run from its own directory.  Per round,
`bench.py --gpus 1 --steps 3 --warmup 3 --no-cpu-baseline --dump-outputs` runs in OLD and then in NEW; afterwards
`tools/attn_bench.py` (all five attention shapes) and `tools/op_profile.py` (per-op time of one UNet forward) run once
per tree at batch F.  Everything is written under OUT_DIR, with the card's name, power limit and clocks, and
OUT_DIR/summary.json collects the bench values and the frame differences (NEW - OLD, in uint8 levels); the dumped
frames themselves are deleted."""
import argparse
import json
import os
import shutil
import subprocess
import sys

import numpy as np


def _run(cmd, cwd, log, env=None, timeout=1800):
    e = dict(os.environ)
    e.update(env or {})
    with open(log, "w") as f:
        r = subprocess.run(cmd, cwd=cwd, stdout=subprocess.PIPE, stderr=f, text=True, env=e, timeout=timeout)
        f.write("\n==== stdout ====\n" + r.stdout)
    if r.returncode != 0:
        raise RuntimeError(f"{cmd} in {cwd} exited {r.returncode}; see {log}")
    return r.stdout


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("out")
    ap.add_argument("--bench-runs", type=int, default=2)
    ap.add_argument("--F", type=int, default=30)
    a = ap.parse_args()
    a.out = os.path.abspath(a.out)  # the commands below run inside each tree
    os.makedirs(a.out, exist_ok=True)
    trees = {"old": os.path.abspath(a.old), "new": os.path.abspath(a.new)}
    py = sys.executable
    summary = {"gpu": subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                                      "--format=csv,noheader"], capture_output=True, text=True).stdout.strip(),
               "bench": {"old": [], "new": []}}
    print(summary["gpu"], flush=True)

    for r in range(a.bench_runs):
        for tag, tree in trees.items():
            dump = os.path.join(a.out, f"frames_{tag}_{r}")
            out = _run([py, "bench.py", "--gpus", "1", "--steps", "3", "--warmup", "3", "--no-cpu-baseline",
                        "--dump-outputs", dump], tree, os.path.join(a.out, f"bench_{tag}_{r}.log"))
            res = json.loads(out.strip().splitlines()[-1])
            rl = res["roofline"]
            row = {"value": res["value"], "ms_per_step": res["ms_per_step"], "attn_us": rl["us_per_launch"],
                   "xu_frac": rl["xu_frac"], "clocks": res.get("clocks")}
            summary["bench"][tag].append(row)
            print(f"bench {tag} run {r}: {row['value']:.4f} frames/s, {row['ms_per_step']:.1f} ms/step, "
                  f"attention {row['attn_us']:.1f} us (xu_frac {row['xu_frac']:.3f})", flush=True)

    env = {"F": str(a.F)}
    for tag, tree in trees.items():
        out = _run([py, "tools/attn_bench.py"], tree, os.path.join(a.out, f"attn_bench_{tag}.log"), env)
        summary[f"attn_bench_{tag}"] = out.strip().splitlines()
        print(f"attn_bench {tag}:\n{out}", flush=True)
    for tag, tree in trees.items():
        out = _run([py, "tools/op_profile.py", os.path.join(a.out, f"op_profile_{tag}.tsv")], tree,
                   os.path.join(a.out, f"op_profile_{tag}.log"), env)
        summary[f"op_profile_{tag}"] = out.strip().splitlines()[:12]
        print(f"op_profile {tag}:\n" + "\n".join(out.strip().splitlines()[:12]), flush=True)

    frames = {(t, r): np.load(os.path.join(a.out, f"frames_{t}_{r}", "frames.npy"))
              for t in trees for r in range(a.bench_runs)}
    d = frames[("new", 0)] - frames[("old", 0)]
    summary["frames_new_minus_old"] = {"max_abs": float(np.abs(d).max()), "mean_abs": float(np.abs(d).mean()),
                                       "frac_changed": float((d != 0).mean())}
    summary["frames_same_build_equal"] = {t: bool(np.array_equal(frames[(t, 0)], frames[(t, r)]))
                                          for t in trees for r in range(1, a.bench_runs)}
    for t in trees:  # the dumps are large; the differences above are what is kept
        for r in range(a.bench_runs):
            shutil.rmtree(os.path.join(a.out, f"frames_{t}_{r}"))
    vo = [x["value"] for x in summary["bench"]["old"]]
    vn = [x["value"] for x in summary["bench"]["new"]]
    summary["speedup_value"] = (sum(vn) / len(vn)) / (sum(vo) / len(vo))
    with open(os.path.join(a.out, "summary.json"), "w") as f:
        json.dump(summary, f, indent=1)
    print(json.dumps({k: summary[k] for k in ("gpu", "frames_new_minus_old", "frames_same_build_equal",
                                               "speedup_value")}), flush=True)


if __name__ == "__main__":
    main()
