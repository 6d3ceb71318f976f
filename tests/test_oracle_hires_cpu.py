"""CPU: the oracle restatement (oracle/vtp_oracle.py) against the REAL reference's outputs above 256x256
(tests/golden/hires_tiny512, hires_tiny_rect from oracle/make_golden_hires.py), under the bounds of
test_oracle_golden.py::test_oracle_matches_golden.  This pins the oracle that tests/test_train_hires_gpu.py
differentiates as the reference of the high-resolution training step."""
import json
import os

import pytest
import torch

from oracle import vtp_oracle as vo
from oracle.seeded import seeded_images, seeded_state_dict
from tests.test_hires_golden_cpu import load_hires_arrays
from tests.util import GOLDEN, rel


@pytest.mark.parametrize("name", ["tiny512", "tiny_rect"])
def test_oracle_matches_hires_golden(name):
    with open(os.path.join(GOLDEN, f"hires_{name}.json")) as f:
        meta = json.load(f)
    g = {k: torch.from_numpy(v) for k, v in load_hires_arrays(name).items()}
    c, (Hi, Wi), s = meta["config"], meta["image_hw"], meta["recon_stride"]
    sd = seeded_state_dict(meta["spec"], seed=0, **meta.get("seed_opts", {}))
    x = seeded_images(meta["batch"], Hi, Wi)
    assert abs(x.double().sum().item() - g["x_checksum"][0].item()) < 1e-6  # same seeded inputs as at generation
    dv, hv = c["vision_depth"], c["vision_num_heads"]
    dd, hd = c["decoder_depth"], c["decoder_num_heads"]
    with torch.no_grad():
        lat = vo.reconstruction_latents(x, sd, depth=dv, heads=hv)
        rec = vo.decode_latents(lat, sd, depth=dd, heads=hd)[..., ::s, ::s]
        fi = vo.clip_image_feature(x, sd, depth=dv, heads=hv)
        # fp32: 1e-5, or the reference's own response to a 1e-6 input perturbation where that is larger
        sens = meta["ref_sensitivity_1e-6"]
        e = {"latents": rel(lat, g["latents_fp32"]), "recon": rel(rec, g["recon_fp32"]), "img_feat": rel(fi, g["img_feat_fp32"])}
        print(name, "fp32", e, sens)
        for k, v in e.items():
            assert v < max(1e-5, sens[k]), (k, v, sens[k])
        # autocast-bf16 restatement: same rounding points, different accumulation order
        latb = vo.reconstruction_latents(x, sd, depth=dv, heads=hv, mode="bf16")
        recb = vo.decode_latents(g["latents_bf16"], sd, depth=dd, heads=hd, mode="bf16")[..., ::s, ::s]
        fib = vo.clip_image_feature(x, sd, depth=dv, heads=hv, mode="bf16")
        eb = {"latents": rel(latb, g["latents_bf16"]), "recon": rel(recb, g["recon_bf16"]),
              "img_feat": rel(fib, g["img_feat_bf16"])}
        print(name, "bf16", eb)
        assert max(eb.values()) < 1e-2, eb
