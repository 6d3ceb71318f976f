"""Seeded inputs of the reconstruction-evaluation golden (oracle/make_golden_recon.py), regenerated bit for bit by the
tests instead of being stored: per case, ImageNet-normalised fp32 inputs x and stand-in "reconstructions" rec = x plus
seeded noise, split into batches whose last one is ragged."""
from __future__ import annotations

import torch

# name -> (H, W, batch sizes)
CASES = {"64x64": (64, 64, (3, 3, 1)), "48x80": (48, 80, (2, 2, 1))}
SEED = 20261017


def recon_inputs(name: str):
    """(x, rec): fp32 [N, 3, H, W] each, N = sum of the case's batch sizes."""
    H, W, batches = CASES[name]
    N = sum(batches)
    g = torch.Generator().manual_seed(SEED + H * 1000 + W)
    x = torch.randn(N, 3, H, W, generator=g) * 1.2
    rec = x + 0.3 * torch.randn(N, 3, H, W, generator=g)
    rec[0, :, :4, :4] = x[0, :, :4, :4]          # a patch reproduced exactly
    return x, rec


def batch_slices(name: str):
    _, _, batches = CASES[name]
    out, s = [], 0
    for b in batches:
        out.append(slice(s, s + b))
        s += b
    return out
