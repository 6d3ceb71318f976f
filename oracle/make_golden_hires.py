"""TEST INFRASTRUCTURE ONLY — generates tests/golden/hires_*.{npz,json}: the REAL reference (oracle/ref_harness.py) on
seeded weights/inputs (oracle/seeded.py) at image sizes above 256x256, i.e. more than 256 patch tokens per image.

    python -m oracle.make_golden_hires [name ...]

Same model kwargs and seeding as oracle/make_golden.py, same stored outputs minus the text tower.  To keep every fixture
file small: reconstructions are stored subsampled as recon[..., ::RECON_STRIDE, ::RECON_STRIDE] (every 16x16 decoder
token is still sampled), and outputs whose values are all exactly bf16 (most of the autocast run) are stored losslessly
as their upper 16 bits, dtype uint16 (tests/test_hires_gpu.py widens them back to fp32)."""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_harness as rh  # noqa: E402
from oracle.make_golden import CONFIGS as BASE  # noqa: E402
from oracle.seeded import seeded_images, seeded_state_dict  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
RECON_STRIDE = 8

CONFIGS = {
    # name: (make_golden config, B, (image H, image W))
    "tiny512": ("tiny", 1, (512, 512)),     # trunk T = 1025, decoder HW = 1024
    # 21 x 33 = 693 patches: ragged last tile (the TMA box reads the next image's rows, which must be masked),
    # non-square RoPE grid, 21 x 33 decoder
    "tiny_rect": ("tiny", 2, (336, 528)),
    "small512": ("small", 1, (512, 512)),   # VTP-Small depth 12 at T = 1025
}


def _compact(a: np.ndarray) -> np.ndarray:
    """fp32 array -> uint16 bf16 bit patterns when that is lossless, else unchanged."""
    bits = a.view(np.uint32)
    return (bits >> 16).astype(np.uint16) if not (bits & 0xFFFF).any() else a


def main():
    rh.import_reference()
    from vtp.models.vtp_hf import VTPConfig, VTPModel

    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(os.cpu_count())
    only = set(sys.argv[1:])
    s = RECON_STRIDE
    for name, (base, B, (Hi, Wi)) in CONFIGS.items():
        if only and name not in only:
            continue
        entry = BASE[base]
        kw = entry[0]
        seed_opts = entry[4] if len(entry) > 4 else {}
        m = VTPModel(VTPConfig(**kw)).eval()
        spec = {k: list(v.shape) for k, v in m.state_dict().items()}
        m.load_state_dict(seeded_state_dict(spec, seed=0, **seed_opts))
        x = seeded_images(B, Hi, Wi)
        out = {}
        with torch.no_grad():
            for tag, ctx in (("fp32", torch.autocast("cpu", enabled=False)),
                             ("bf16", torch.autocast("cpu", dtype=torch.bfloat16))):
                with ctx:
                    lat = m.get_reconstruction_latents(x)
                    out[f"latents_{tag}"] = lat.float().numpy()
                    out[f"recon_{tag}"] = m.get_latents_decoded_images(lat).float()[..., ::s, ::s].contiguous().numpy()
                    out[f"img_feat_{tag}"] = m.get_clip_image_feature(x).float().numpy()
                    out[f"cls_{tag}"] = m.get_last_layer_feature(x)["cls_token"].float().numpy()
        # the reference's own response to a 1e-6 relative input perturbation (see oracle/make_golden.py)
        with torch.no_grad():
            xp = x * (1 + 1e-6)
            relf = lambda a, b: float(((a.float() - torch.from_numpy(b)).norm() / torch.from_numpy(b).norm()))
            latp = m.get_reconstruction_latents(xp)
            sens = {"latents": relf(latp, out["latents_fp32"]),
                    "recon": relf(m.get_latents_decoded_images(latp)[..., ::s, ::s], out["recon_fp32"]),
                    "img_feat": relf(m.get_clip_image_feature(xp), out["img_feat_fp32"]),
                    "cls": relf(m.get_last_layer_feature(xp)["cls_token"], out["cls_fp32"])}
        out["x_checksum"] = np.array([x.double().sum().item(), x.double().abs().sum().item()])
        np.savez_compressed(os.path.join(OUT, f"hires_{name}.npz"),
                            **{k: _compact(v) if v.dtype == np.float32 else v for k, v in out.items()})
        with open(os.path.join(OUT, f"hires_{name}.json"), "w") as f:
            json.dump({"config": kw, "batch": B, "image_hw": [Hi, Wi], "recon_stride": s, "spec": spec,
                       "reference_commit": "5ce1eb6", "torch": torch.__version__, "seed_opts": seed_opts,
                       "ref_sensitivity_1e-6": sens}, f)
        dev = {k: relf(torch.from_numpy(out[f"{k}_bf16"]), out[f"{k}_fp32"]) for k in ("latents", "recon", "img_feat", "cls")}
        print(name, "reference sensitivity to 1e-6 input perturbation:", sens)
        print(name, "reference bf16-autocast vs fp32:", dev)


if __name__ == "__main__":
    main()
