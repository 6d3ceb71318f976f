"""Seeded stand-in trunk taps of the linear-probe golden run (oracle/make_golden_probe.py -> tests/golden/probe_tiny.*).
Plain torch on the CPU generator, so the GPU tests regenerate exactly the taps the reference was fed."""
from __future__ import annotations

import torch

D, C, B, HW, STEPS, N_EVAL, SEED, TAP_SEED = 64, 37, 128, 5, 30, 256, 0, 1234
ROWS = list(range(16)) + [C - 1]     # classes whose final weight rows are stored in full


def probe_taps(step: int, batch: int = B, dtype=torch.float32):
    """Step `step`'s taps (step -1 = the held-out set): ([(patch [b, HW, D], cls [b, D])] x 4 blocks, labels [b]).
    Class-dependent means so that the classifiers have something to learn."""
    g = torch.Generator().manual_seed(TAP_SEED)
    centres = torch.randn(C, 5, D, generator=g)
    g = torch.Generator().manual_seed(TAP_SEED + 1 + step if step >= 0 else TAP_SEED - 1)
    labels = torch.randint(0, C, (batch,), generator=g)
    c = centres[labels]
    feats = []
    for i in range(4):
        cls = 0.5 * c[:, i] + torch.randn(batch, D, generator=g)
        patch = 0.5 * c[:, 4:5] + torch.randn(batch, HW, D, generator=g)
        feats.append((patch.to(dtype), cls.to(dtype)))
    return feats, labels


def linear_input(feats, n: int):
    """create_linear_input(feats, n, use_avgpool=True) (tools/test_linear_probing_hf.py:137-152) without its final
    .float(), so that the fp64 arm stays fp64."""
    out = torch.cat([cls for _, cls in feats[-n:]] + [feats[-1][0].mean(dim=1)], dim=-1)
    return out.reshape(out.shape[0], -1)
