"""Host side of the reconstruction evaluator (vtp_b200/recon_eval.py): the SSIM restatements the GPU tests measure
against, the weight-file loader of LPIPSMetric, the command line, the PNG index formula and the rank aggregation."""
import math

import numpy as np
import pytest
import torch

from tests.ssim_ref import C1, ssim_torchmetrics_form, ssim_valid_fp64

# the sizes of tests/test_recon_eval_gpu.py
GPU_SIZES = [(11, 11), (64, 64), (48, 80), (256, 256), (512, 512), (256, 384)]


@pytest.mark.parametrize("H,W", [(11, 11), (16, 23), (64, 64), (48, 80)])
def test_ssim_restatements_agree(H, W):
    g = torch.Generator().manual_seed(H * 1000 + W)
    x = torch.rand(3, 3, H, W, generator=g)
    y = (x + 0.1 * torch.randn(3, 3, H, W, generator=g)).clamp(0, 1)
    a = ssim_torchmetrics_form(x, y)
    b = ssim_valid_fp64(x, y)
    assert torch.allclose(a.double(), b, rtol=0, atol=2e-6), (a, b)


def test_ssim_constant_images_analytic():
    """Constant images: σ = 0, so SSIM = (2ab + C1) / (a² + b² + C1)."""
    a, b = float(torch.tensor(0.3)), float(torch.tensor(0.7))   # the fp32 values the images hold
    x = torch.full((1, 3, 20, 17), a)
    y = torch.full((1, 3, 20, 17), b)
    want = (2 * a * b + C1) / (a * a + b * b + C1)
    assert abs(float(ssim_valid_fp64(x, y)) - want) < 1e-11
    # fp32: E[x²] − μ² cancels to a few ulp of 0.49, which C2 = 9e-4 scales up
    assert abs(float(ssim_torchmetrics_form(x, y)) - want) < 1e-3


@pytest.mark.parametrize("H,W", GPU_SIZES)
def test_ssim_tf32_yardstick(H, W):
    """The reference's own SSIM error on an H100 (TF32 conv operands) against fp64, the scale the GPU test's SSIM
    tolerance is a fraction of, stands well clear of fp32 rounding at the GPU test's sizes: half of it is a bound an
    fp32-accurate kernel can meet and a TF32-accurate one cannot."""
    g = torch.Generator().manual_seed(7)
    x = torch.rand(4, 3, H, W, generator=g)
    y = (x + 0.05 * torch.randn(4, 3, H, W, generator=g)).clamp(0, 1)
    exact = ssim_valid_fp64(x, y)
    tf32 = (ssim_torchmetrics_form(x, y, tf32=True).double() - exact).abs().max().item()
    fp32 = (ssim_torchmetrics_form(x, y).double() - exact).abs().max().item()
    assert tf32 > 16 * fp32, (tf32, fp32)


def _write_weight_files(tmp_path, drop=None):
    import torchvision

    vgg = torchvision.models.vgg16(weights=None).state_dict()
    if drop in vgg:
        del vgg[drop]
    g = torch.Generator().manual_seed(0)
    lin = {f"lin{k}.model.1.weight": torch.rand(1, c, 1, 1, generator=g) for k, c in enumerate((64, 128, 256, 512, 512))}
    lin["scaling_layer.shift"] = torch.zeros(1, 3, 1, 1)       # extra keys are ignored
    if drop in lin:
        del lin[drop]
    torch.save(vgg, tmp_path / "vgg16.pth")
    torch.save(lin, tmp_path / "lin.pth")
    return vgg, lin


def test_weight_file_loader(tmp_path):
    from vtp_b200.lpips import VGG_CFG, load_weight_files

    vgg, lin = _write_weight_files(tmp_path)
    vw, vb, lw = load_weight_files(str(tmp_path / "vgg16.pth"), str(tmp_path / "lin.pth"))
    assert len(vw) == len(vb) == 13 and len(lw) == 5
    chans = [c for c in VGG_CFG if c != "M"]
    cin = 3
    for w, b, c in zip(vw, vb, chans):
        assert tuple(w.shape) == (c, cin, 3, 3) and tuple(b.shape) == (c,)
        cin = c
    assert torch.equal(vw[0], vgg["features.0.weight"]) and torch.equal(vb[12], vgg["features.28.bias"])
    assert torch.equal(lw[4], lin["lin4.model.1.weight"])


@pytest.mark.parametrize("drop", ["features.12.bias", "lin3.model.1.weight"])
def test_weight_file_loader_names_missing_key(tmp_path, drop):
    from vtp_b200.lpips import load_weight_files

    _write_weight_files(tmp_path, drop=drop)
    with pytest.raises(KeyError, match=drop.replace(".", r"\.")):
        load_weight_files(str(tmp_path / "vgg16.pth"), str(tmp_path / "lin.pth"))


REFERENCE_FLAGS = ["--model_path", "M", "--data_path", "D", "--output_path", "O", "--batch_size", "7", "--num_workers", "0",
                   "--device", "cuda:1", "--precision", "fp32", "--no_save_images", "--use_ddp", "--local_rank", "3",
                   "--max_samples", "11"]


def test_cli_accepts_reference_flags():
    from vtp_b200.recon_eval import build_parser

    a = build_parser().parse_args(REFERENCE_FLAGS + ["--lpips_vgg", "v.pth", "--lpips_lin", "l.pth"])
    assert (a.model_path, a.data_path, a.output_path, a.batch_size, a.num_workers) == ("M", "D", "O", 7, 0)
    assert (a.device, a.precision, a.no_save_images, a.use_ddp, a.local_rank, a.max_samples) == ("cuda:1", "fp32", True,
                                                                                                 True, 3, 11)
    assert (a.lpips_vgg, a.lpips_lin) == ("v.pth", "l.pth")
    d = build_parser().parse_args(["--model_path", "M", "--data_path", "D"])
    assert (d.output_path, d.batch_size, d.num_workers, d.device, d.precision) == ("reconstruction_output", 32, 4, "cuda:0",
                                                                                 "bf16")
    assert not d.no_save_images and not d.use_ddp and d.max_samples is None and d.lpips_vgg is None


def test_cli_rejects_fp16():
    from vtp_b200.recon_eval import main

    with pytest.raises(NotImplementedError):
        main(["--model_path", "M", "--data_path", "D", "--precision", "fp16"])


def test_png_indices():
    """test_reconstruction_hf.py:404-407 with a DistributedSampler of 2 ranks, batch 4 and 13 images (padded to 14)."""
    from vtp_b200.recon_eval import png_indices

    total, bs, world = 13, 4, 2
    seen = []
    for rank in range(world):
        per_rank = 7                      # ceil(13 / 2): the sampler repeats one sample to pad
        for bi, s in enumerate(range(0, per_rank, bs)):
            n = min(bs, per_rank - s)
            want = []
            for j in range(n):
                i = bi * bs * world + rank * bs + j
                if i >= total:
                    break
                want.append(i)
            got = png_indices(bi, bs, world, rank, n, total)
            assert got == want
            seen += got
    assert len(seen) == len(set(seen))
    # the reference's quirk: rank 1's short last batch (3 images) leaves file 11 unwritten, so a sharded run writes
    # fewer than `total` PNGs and the skip-if-present check can never fire for it
    assert sorted(seen) == [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 12]
    assert png_indices(0, 4, 1, 0, 4, None) == [0, 1, 2, 3]


def test_rank_aggregation_arithmetic():
    """Each rank's mean, then the mean over ranks (test_reconstruction_hf.py:417-422); batch means for SSIM / LPIPS."""
    from vtp_b200.recon_eval import rank_mean

    assert rank_mean(None, 4, "cpu") is None
    assert rank_mean(2.5, 1, "cpu") == 2.5
    # the reference's SSIM over a ragged split: mean of batch means, not the mean over images
    batches = [np.array([0.5, 0.7, 0.9]), np.array([0.1])]
    ref = np.mean([b.mean() for b in batches])
    assert math.isclose(ref, (0.7 + 0.1) / 2)
    assert not math.isclose(ref, np.concatenate(batches).mean())


# ---------------------------------------------------------------------------------------------------------- golden
def _golden():
    import json
    import os

    root = os.path.join(os.path.dirname(__file__), "golden")
    with open(os.path.join(root, "recon_tiny.json")) as f:
        meta = json.load(f)
    return meta, np.load(os.path.join(root, "recon_tiny.npz"))


@pytest.mark.parametrize("case", ["64x64", "48x80"])
def test_golden_inputs_regenerate(case):
    from oracle.recon_inputs import recon_inputs

    meta, _ = _golden()
    x, rec = recon_inputs(case)
    assert float(x.double().abs().sum()) == meta["cases"][case]["x_abs_sum"]
    assert float(rec.double().abs().sum()) == meta["cases"][case]["rec_abs_sum"]


def _denorm_cpu(t):
    from vtp_b200.recon_eval import IMAGENET_DEFAULT_MEAN, IMAGENET_DEFAULT_STD

    sub = torch.tensor([-m / s for m, s in zip(IMAGENET_DEFAULT_MEAN, IMAGENET_DEFAULT_STD)]).view(1, 3, 1, 1)
    div = torch.tensor([1.0 / s for s in IMAGENET_DEFAULT_STD]).view(1, 3, 1, 1)
    return torch.clamp((t - sub) / div, 0, 1)


@pytest.mark.parametrize("case", ["64x64", "48x80"])
def test_psnr_and_uint8_restatement_reproduce_golden(case):
    """The fp64 PSNR formula the GPU tests use as truth and the uint8 conversion reproduce the reference's own outputs."""
    from oracle.recon_inputs import recon_inputs

    meta, g = _golden()
    x, rec = recon_inputs(case)
    o, r = _denorm_cpu(x), _denorm_cpu(rec)
    d = o.double() * 255 - r.double() * 255
    psnr64 = (20 * torch.log10(255.0 / torch.sqrt((d ** 2).mean((1, 2, 3))))).numpy()
    assert np.allclose(psnr64, g[f"{case}_psnr64"], rtol=0, atol=1e-12)
    gap = meta["cases"][case]["psnr_fp32_gap"]
    assert 0 < gap < 1e-4
    assert np.array_equal((o.permute(0, 2, 3, 1).numpy() * 255.0).astype(np.uint8), g[f"{case}_u8_ref"])
    assert np.array_equal((r.permute(0, 2, 3, 1).numpy() * 255.0).astype(np.uint8), g[f"{case}_u8_rec"])


@pytest.mark.parametrize("case", ["64x64", "48x80"])
def test_oracle_lpips_reproduces_golden(case):
    """oracle.vtp_oracle.lpips (the restatement the LPIPS kernels were built against) equals the reference's module:
    in fp64 up to the ScalingLayer constants' fp32 rounding, in fp32 well inside the golden's TF32-vs-fp64 gap."""
    from oracle import vtp_oracle as vo
    from oracle.recon_inputs import batch_slices, recon_inputs
    from vtp_b200.lpips import random_weights

    meta, g = _golden()
    vw, vb, lw = random_weights(0)
    x, rec = recon_inputs(case)
    o, r = _denorm_cpu(x), _denorm_cpu(rec)
    with torch.no_grad():
        v64 = vo.lpips(o.double() * 2.0 - 1.0, r.double() * 2.0 - 1.0, [w.double() for w in vw],
                       [b.double() for b in vb], [l.double() for l in lw]).flatten().numpy()
        v32 = vo.lpips(o * 2.0 - 1.0, r * 2.0 - 1.0, vw, vb, lw).flatten().double().numpy()
    gap = meta["cases"][case]["lpips_tf32_gap"]
    assert gap > 0
    # the reference's ScalingLayer constants are fp32 buffers; the restatement's fp64 run uses the decimal values
    assert np.allclose(v64, g[f"{case}_lpips64"], rtol=1e-7, atol=0)
    assert np.abs(v32 - g[f"{case}_lpips64"]).max() <= gap / 16
    blp = [float(g[f"{case}_lpips64"][sl].mean()) for sl in batch_slices(case)]
    assert np.allclose(blp, g[f"{case}_blp64"], rtol=1e-14, atol=0)
