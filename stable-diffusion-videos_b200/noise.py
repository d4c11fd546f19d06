"""Host side of the stochastic samplers' step noise (DDIM eta > 0, Euler ancestral).

The noise itself is generated inside the fused step kernel (include/sdwalk.h, sdw_frame_noise): frame f's noise at step
s is w_a Z(key_a, s) + w_b Z(key_b, s) with Z a counter-based Philox normal field.  This module builds the per-frame
table of keys and weights:

  walk frame at position T between seeds (a, b): keys (a, b) mod 2^64, weights (cos(pi T / 2), sin(pi T / 2)) in fp64,
      exactly (1, 0) at T = 0 and (0, 1) at T = 1.  This is the slerp the init latents get (utils.slerp) at the angle
      pi / 2 of two independent noise fields: every element keeps unit variance, neighbouring frames get nearly the same
      noise, and T = 1 of one clip and T = 0 of the next use the same seed's stream.
  __call__ image: (k, k, 1, 0) with k one non-negative int64 drawn from the caller's generator per image.

So a frame's noise depends on its seeds and T only, never on the batch it is rendered in, on a resume or on frame
sharding.  The reference draws this noise from torch's global RNG instead (unseeded, per frame and step), which nobody
can reproduce; this is the one place where the native sampler deliberately computes something else.
"""
import math

import numpy as np
import torch

from ._native import FrameNoise

_MASK64 = (1 << 64) - 1


def walk_weights(t):
    """(w_a, w_b) of the frame at interpolation position t, in fp64"""
    t = float(t)
    if t == 0.0:
        return 1.0, 0.0
    if t == 1.0:
        return 0.0, 1.0
    return math.cos(math.pi * t / 2), math.sin(math.pi * t / 2)


def walk_table(T, seed_a, seed_b):
    """[len(T)] FrameNoise entries of walk frames at positions T between two keyframe seeds"""
    ka, kb = int(seed_a) & _MASK64, int(seed_b) & _MASK64
    out = (FrameNoise * len(T))()
    for i, t in enumerate(T):
        w_a, w_b = walk_weights(t)
        out[i] = FrameNoise(ka, kb, w_a, w_b)
    return out


def call_table(keys):
    """[len(keys)] FrameNoise entries of independent images: key k with weight 1"""
    out = (FrameNoise * len(keys))()
    for i, k in enumerate(keys):
        out[i] = FrameNoise(int(k) & _MASK64, int(k) & _MASK64, 1.0, 0.0)
    return out


def draw_call_keys(n, generator, device):
    """one non-negative int64 per image from `generator` (or the default generator of `device` when None)"""
    dev = generator.device if generator is not None else torch.device(device)
    return torch.randint(0, 2 ** 63 - 1, (n,), generator=generator, device=dev, dtype=torch.int64).tolist()


def pad_table(table, n):
    """the table extended to n entries by repeating its last one (the padded tail frames of a batch)"""
    out = (FrameNoise * n)()
    for i in range(n):
        out[i] = table[min(i, len(table) - 1)]
    return out


def as_numpy(table):
    """the table as a numpy structured array (key_a, key_b uint64; w_a, w_b float32)"""
    dt = np.dtype([("key_a", "<u8"), ("key_b", "<u8"), ("w_a", "<f4"), ("w_b", "<f4")])
    return np.frombuffer(bytes(table), dtype=dt).copy() if len(table) else np.zeros(0, dtype=dt)


def to_device(table, device):
    """the table's 24-byte entries as a uint8 CUDA tensor [n * 24]"""
    raw = np.frombuffer(bytes(table), dtype=np.uint8).copy()
    return torch.from_numpy(raw).to(device)
