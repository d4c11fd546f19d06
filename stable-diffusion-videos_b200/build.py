"""Build recipe for libsdwalk.so (sm_90a only; nvcc cross-compiles without a GPU).

`python stable-diffusion-videos_b200/build.py` or `__graft_entry__.build()`.
The .so is built in-tree next to this file, so the package imports straight from the repository.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libsdwalk.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v",
]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stale(obj, src):
    if not os.path.exists(obj):
        return True
    t = os.path.getmtime(obj)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    deps += [src, os.path.join(HERE, "..", "include", "sdwalk.h"), __file__]
    return any(os.path.getmtime(d) > t for d in deps)


def _compile(src):
    obj = os.path.join(HERE, "build", os.path.basename(src)[:-3] + ".o")
    if not _stale(obj, src):
        return obj, ""
    r = subprocess.run([NVCC, *FLAGS, "-c", src, "-o", obj], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    return obj, r.stderr


def build(verbose=False):
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    srcs = [os.path.join(CSRC, f) for f in _sources()]
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        res = list(ex.map(_compile, srcs))
    objs = [o for o, _ in res]
    log = "".join(l for _, l in res)
    if verbose and log:
        print(log)
    if any(l for _, l in res) or not os.path.exists(OUT) or any(os.path.getmtime(o) > os.path.getmtime(OUT) for o in objs):
        r = subprocess.run([NVCC, "-shared", "-o", OUT, *objs, "-gencode", "arch=compute_90a,code=sm_90a",
                            "-lcudart", "-ldl"], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(os.path.join(HERE, "build", "ptxas.log"), "a") as f:
        f.write(log)
    return OUT


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv))
