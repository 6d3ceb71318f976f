"""The high-resolution golden fixtures (oracle/make_golden_hires.py) are complete, self-describing and small."""
import json
import os

import numpy as np
import pytest

from tests.util import GOLDEN

NAMES = ["tiny512", "tiny_rect", "small512"]


def load_hires_arrays(name):
    """hires_<name>.npz as fp32 arrays: uint16 entries are bf16 bit patterns (stored that way because it is lossless)."""
    g = dict(np.load(os.path.join(GOLDEN, f"hires_{name}.npz")))
    return {k: (v.astype(np.uint32) << 16).view(np.float32) if v.dtype == np.uint16 else v for k, v in g.items()}


def test_hires_fixtures_are_small():
    sizes = {f"{n}.{ext}": os.path.getsize(os.path.join(GOLDEN, f"hires_{n}.{ext}")) for n in NAMES for ext in ("npz", "json")}
    assert sum(sizes.values()) <= 4 * 2**20, sizes
    assert max(sizes.values()) <= 2**20, sizes


@pytest.mark.parametrize("name", NAMES)
def test_hires_fixture_shapes(name):
    with open(os.path.join(GOLDEN, f"hires_{name}.json")) as f:
        meta = json.load(f)
    g = load_hires_arrays(name)
    (Hi, Wi), s, B = meta["image_hw"], meta["recon_stride"], meta["batch"]
    assert Hi % 16 == 0 and Wi % 16 == 0 and (Hi // 16) * (Wi // 16) > 256 and 16 % s == 0
    for tag in ("fp32", "bf16"):
        assert g[f"latents_{tag}"].shape == (B, 64, Hi // 16, Wi // 16)
        assert g[f"recon_{tag}"].shape == (B, 3, Hi // s, Wi // s)
        assert g[f"cls_{tag}"].shape == (B, meta["config"]["vision_embed_dim"])
        for k in ("latents", "recon", "img_feat", "cls"):
            assert g[f"{k}_{tag}"].dtype == np.float32 and np.isfinite(g[f"{k}_{tag}"]).all()
    assert set(meta["ref_sensitivity_1e-6"]) == {"latents", "recon", "img_feat", "cls"}
