"""Reconstruction evaluation on the device (vtp_b200/recon_eval.py, csrc/recon_metrics.cu, LPIPSMetric in lpips.py).

Tolerances are tied to the reference's own error on an H100: the reference computes PSNR in fp32 torch and SSIM / LPIPS
with cuDNN convolutions, which default to TF32.  Each metric here must sit within half of that error (measured on the
same inputs: fp32 torch PSNR, TF32-rounded conv operands for SSIM and LPIPS) from an fp64 evaluation."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import vtp_oracle as vo
from tests.ssim_ref import round_tf32, ssim_torchmetrics_form, ssim_valid_fp64
from vtp_b200 import lib
from vtp_b200.recon_eval import IMAGENET_DEFAULT_MEAN, IMAGENET_DEFAULT_STD

pytestmark = pytest.mark.gpu

SUB = [-m / s for m, s in zip(IMAGENET_DEFAULT_MEAN, IMAGENET_DEFAULT_STD)]
DIV = [1.0 / s for s in IMAGENET_DEFAULT_STD]


def _sub_div():
    return (torch.tensor(SUB, dtype=torch.float32, device="cuda"), torch.tensor(DIV, dtype=torch.float32, device="cuda"))


def _pair(B, H, W, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 3, H, W, generator=g) * 1.2
    rec = x + 0.15 * torch.randn(B, 3, H, W, generator=g)
    return x.cuda(), rec.to(dtype).cuda()


def _denorm(t, sub, div):
    """transform_rev + clamp (test_reconstruction_hf.py:371-376), torch fp32 on the device."""
    return torch.clamp((t.float() - sub.view(1, 3, 1, 1)) / div.view(1, 3, 1, 1), 0, 1)


def _run_kernels(x, rec, lp=False, u8=True):
    sub, div = _sub_div()
    B, _, H, W = x.shape
    sse = torch.empty(B, min(H, 16), dtype=torch.float64, device="cuda")
    part = torch.empty(B, lib.recon_ssim_tiles(H, W), dtype=torch.float64, device="cuda")
    u8r = torch.empty(B, H, W, 3, dtype=torch.uint8, device="cuda") if u8 else None
    u8o = torch.empty_like(u8r) if u8 else None
    lpb = torch.empty(B, 2, 3, H, W, dtype=torch.float32, device="cuda") if lp else None
    lib.recon_pixels(x, rec, sub, div, sse, u8_ref=u8r, u8_rec=u8o, lp=lpb)
    lib.recon_ssim(x, rec, sub, div, part)
    psnr = torch.empty(B, dtype=torch.float64, device="cuda")
    ssim = torch.empty(B, device="cuda")
    acc = torch.zeros(8, dtype=torch.float64, device="cuda")
    lib.recon_finalise(sse, part, None, H, W, psnr, ssim, None, acc)
    torch.cuda.synchronize()
    return dict(u8r=u8r, u8o=u8o, psnr=psnr, ssim=ssim, acc=acc, lp=lpb)


SIZES = [(11, 11, 1), (64, 64, 50), (48, 80, 5), (256, 256, 4), (512, 512, 2), (256, 384, 3)]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("H,W,B", SIZES)
def test_pixels_psnr_ssim(H, W, B, dtype):
    x, rec = _pair(B, H, W, dtype, seed=H * 7 + W + B)
    out = _run_kernels(x, rec)
    sub, div = _sub_div()
    o, r = _denorm(x, sub, div), _denorm(rec, sub, div)
    # uint8: bit-identical with the reference's numpy conversion and with vtp_image_to_u8
    assert torch.equal(out["u8r"], (o.permute(0, 2, 3, 1) * 255.0).to(torch.uint8))
    assert torch.equal(out["u8o"], (r.permute(0, 2, 3, 1) * 255.0).to(torch.uint8))
    if W % 4 == 0:
        want = torch.empty_like(out["u8o"])
        lib.image_to_u8(rec, sub, div, want)
        assert torch.equal(out["u8o"], want)
    # PSNR: fp64 truth, the reference's fp32 calculate_psnr as the yardstick
    d64 = o.double() * 255 - r.double() * 255
    psnr64 = 20 * torch.log10(255.0 / torch.sqrt((d64 ** 2).mean((1, 2, 3))))
    ref32 = torch.stack([20 * torch.log10(torch.tensor(255.0, device="cuda") / torch.sqrt(torch.mean((o[i] * 255.0 - r[i] * 255.0) ** 2)))
                         for i in range(B)]).double()
    yard = (ref32 - psnr64).abs().max().item()
    err = (out["psnr"].double() - psnr64).abs().max().item()
    assert err <= 0.5 * yard, (err, yard)
    # SSIM: fp64 truth, TF32 conv operands (cuDNN's default on an H100) as the yardstick
    oc, rc = o.cpu(), r.cpu()
    s64 = ssim_valid_fp64(oc, rc)
    yard = (ssim_torchmetrics_form(oc, rc, tf32=True).double() - s64).abs().max().item()
    err = (out["ssim"].double().cpu() - s64).abs().max().item()
    assert err <= 0.5 * yard, (err, yard)
    # accumulators: Σ PSNR, images, batch-mean SSIM, batches
    a = out["acc"].cpu().tolist()
    assert a[1] == B and a[4] == 1
    assert a[0] == pytest.approx(float(out["psnr"].double().sum()), rel=1e-12)
    assert a[2] == pytest.approx(float(out["ssim"].double().mean()), rel=1e-12)


def test_psnr_inf_for_identical_images():
    x, _ = _pair(3, 32, 32, torch.float32, seed=1)
    out = _run_kernels(x, x.clone())
    assert torch.isinf(out["psnr"]).all() and (out["psnr"] > 0).all()
    assert torch.allclose(out["ssim"], torch.ones(3, device="cuda"), atol=1e-6)


def test_kernels_repeat_bit_identical():
    x, rec = _pair(7, 96, 128, torch.float32, seed=2)
    a, b = _run_kernels(x, rec, lp=True), _run_kernels(x, rec, lp=True)
    for k in ("u8r", "u8o", "psnr", "ssim", "acc", "lp"):
        assert torch.equal(a[k], b[k]), k


# ---------------------------------------------------------------------------------------------------------- LPIPS
def lpips_ref(x, y, vw, vb, lw, tf32: bool):
    """utils/lpips.py:84-100 restated (as oracle.vtp_oracle.lpips) on x's device: in fp64, or in fp32 with every conv
    operand rounded to TF32 (what cuDNN's default conv precision does on an H100)."""
    dt = torch.float32 if tf32 else torch.float64
    rnd = round_tf32 if tf32 else (lambda t: t)
    dev = x.device
    shift = torch.tensor(vo.LPIPS_SHIFT, dtype=dt, device=dev)[None, :, None, None]
    scale = torch.tensor(vo.LPIPS_SCALE, dtype=dt, device=dev)[None, :, None, None]

    def feats(t):
        t = (t.to(dt) - shift) / scale
        outs, ci = [], 0
        for c in vo.VGG_CFG:
            if c == "M":
                t = F.max_pool2d(t, 2, 2)
            else:
                t = F.relu(F.conv2d(rnd(t), rnd(vw[ci].to(dev, dt)), vb[ci].to(dev, dt), padding=1))
                if ci in vo.LPIPS_TAPS:
                    outs.append(t)
                ci += 1
        return outs

    fx, fy = feats(x), feats(y)
    val = 0
    for k in range(5):
        nx = fx[k] / (torch.sqrt(torch.sum(fx[k] ** 2, dim=1, keepdim=True)) + 1e-10)
        ny = fy[k] / (torch.sqrt(torch.sum(fy[k] ** 2, dim=1, keepdim=True)) + 1e-10)
        val = val + F.conv2d(rnd((nx - ny) ** 2), rnd(lw[k].to(dev, dt))).mean([2, 3], keepdim=True)
    return val.flatten().double().cpu()


@pytest.mark.parametrize("B,H,W", [(3, 64, 64), (1, 256, 256), (2, 64, 128), (1, 512, 512), (1, 256, 384)])
def test_lpips_metric_against_fp64(B, H, W):
    """Per-image LPIPS of LPIPSMetric (bf16x3 conv GEMMs with fp32 output: the K = 96 conv1_1 GEMM and the implicit-conv
    GEMMs with conv_C = 3C) within half the TF32 reference's distance from fp64."""
    from vtp_b200.lpips import LPIPSMetric, random_weights

    vw, vb, lw = random_weights(0)
    x, rec = _pair(B, H, W, torch.float32, seed=11 + H)
    out = _run_kernels(x, rec, lp=True)
    m = LPIPSMetric(vw, vb, lw, chunk=2)
    part = m.parts(out["lp"])
    got = part.sum(1).cpu()
    sub, div = _sub_div()
    o, r = _denorm(x, sub, div) * 2 - 1, _denorm(rec, sub, div) * 2 - 1
    with torch.no_grad():
        want = lpips_ref(o, r, vw, vb, lw, tf32=False)
        tf = lpips_ref(o, r, vw, vb, lw, tf32=True)
    yard = (tf - want).abs().max().item()
    err = (got - want).abs().max().item()
    assert yard > 0
    assert err <= 0.5 * yard, (err, yard, got, want)
    assert torch.equal(part, m.parts(out["lp"]))          # repeat: bit-identical


def test_empty_bands_sum_to_zero():
    """nbands = 16 at H = 40 gives bands of 3 rows, the last two past row 39: they hold 0 and PSNR is unchanged."""
    x, rec = _pair(2, 40, 24, torch.float32, seed=5)
    sub, div = _sub_div()
    sse16 = torch.full((2, 16), float("nan"), dtype=torch.float64, device="cuda")
    sse1 = torch.empty((2, 1), dtype=torch.float64, device="cuda")
    lib.recon_pixels(x, rec, sub, div, sse16)
    lib.recon_pixels(x, rec, sub, div, sse1)
    torch.cuda.synchronize()
    assert torch.equal(sse16[:, 14:], torch.zeros(2, 2, dtype=torch.float64, device="cuda"))
    assert torch.allclose(sse16.sum(1), sse1[:, 0], rtol=1e-12, atol=0)


def test_argument_checks():
    x, rec = _pair(1, 16, 16, torch.float32, seed=6)
    sub, div = _sub_div()
    sse = torch.empty((1, 4), dtype=torch.float64, device="cuda")
    with pytest.raises(lib.VtpError, match="sub3"):
        lib.recon_pixels(x, rec, sub.cpu(), div, sse)
    with pytest.raises(lib.VtpError, match="div3"):
        lib.recon_ssim(x, rec, sub, div.double(), torch.empty((1, 1), dtype=torch.float64, device="cuda"))
    part = torch.empty((1, 1), dtype=torch.float64, device="cuda")
    ps, ss, lps = (torch.empty(1, dtype=torch.float64, device="cuda"), torch.empty(1, device="cuda"),
                   torch.empty(1, device="cuda"))
    with pytest.raises(lib.VtpError, match="lp_part"):
        lib.recon_finalise(sse, part, torch.zeros((2, 3), dtype=torch.float64, device="cuda"), 16, 16, ps, ss, lps,
                           torch.zeros(8, dtype=torch.float64, device="cuda"))
    f = torch.zeros((2, 4, 64), device="cuda")
    with pytest.raises(lib.VtpError, match="CUDA"):
        lib.lpips_tap_metric(f, torch.zeros(64, device="cuda"), 1, 4, 64, torch.zeros((1, 4), dtype=torch.float64), 0, 4)


# ---------------------------------------------------------------------------------------------------------- golden
@pytest.mark.parametrize("case", ["64x64", "48x80"])
def test_against_reference_golden(case):
    """The reference's own outputs (oracle/make_golden_recon.py: its calculate_psnr, transform_rev + clamp + uint8 and
    its LPIPS module) on the golden's regenerated inputs, batch by batch with the ragged last batch: uint8 arrays
    bit-identical, per-image PSNR and per-image / per-batch LPIPS within half of the golden's own fp32 (PSNR) and TF32
    (LPIPS) distance from its fp64 run.  LPIPSMetric does not take 48x80 (W % 64), so that case checks PSNR and uint8."""
    import json

    from oracle.recon_inputs import batch_slices, recon_inputs
    from vtp_b200.lpips import LPIPSMetric, random_weights

    root = os.path.join(os.path.dirname(__file__), "golden")
    meta = json.load(open(os.path.join(root, "recon_tiny.json")))["cases"][case]
    g = np.load(os.path.join(root, "recon_tiny.npz"))
    x, rec = recon_inputs(case)
    H, W = x.shape[-2:]
    lp_ok = H % 16 == 0 and W % 64 == 0
    m = LPIPSMetric(*random_weights(0)) if lp_ok else None
    acc = torch.zeros(8, dtype=torch.float64, device="cuda")
    sub, div = _sub_div()
    psnr, lpv, u8r, u8o = [], [], [], []
    for sl in batch_slices(case):
        xb, rb = x[sl].cuda(), rec[sl].cuda()
        B = xb.shape[0]
        sse = torch.empty(B, 16, dtype=torch.float64, device="cuda")
        part = torch.empty(B, lib.recon_ssim_tiles(H, W), dtype=torch.float64, device="cuda")
        ur, uo = (torch.empty(B, H, W, 3, dtype=torch.uint8, device="cuda") for _ in range(2))
        lp = torch.empty(B, 2, 3, H, W, device="cuda") if lp_ok else None
        lib.recon_pixels(xb, rb, sub, div, sse, u8_ref=ur, u8_rec=uo, lp=lp)
        lib.recon_ssim(xb, rb, sub, div, part)
        ps = torch.empty(B, dtype=torch.float64, device="cuda")
        ss, ll = torch.empty(B, device="cuda"), torch.empty(B, device="cuda")
        lib.recon_finalise(sse, part, m.parts(lp) if lp_ok else None, H, W, ps, ss, ll if lp_ok else None, acc)
        psnr.append(ps.cpu())
        lpv.append(ll.cpu())
        u8r.append(ur.cpu())
        u8o.append(uo.cpu())
    assert np.array_equal(torch.cat(u8r).numpy(), g[f"{case}_u8_ref"])
    assert np.array_equal(torch.cat(u8o).numpy(), g[f"{case}_u8_rec"])
    err = np.abs(torch.cat(psnr).numpy() - g[f"{case}_psnr64"]).max()
    assert err <= 0.5 * meta["psnr_fp32_gap"], (err, meta["psnr_fp32_gap"])
    a = acc.cpu().tolist()
    nb = len(batch_slices(case))
    assert a[1] == x.shape[0] and a[4] == nb
    assert abs(a[0] / a[1] - g[f"{case}_psnr64"].mean()) <= 0.5 * meta["psnr_fp32_gap"]
    if lp_ok:
        gap = meta["lpips_tf32_gap"]
        err = np.abs(torch.cat(lpv).double().numpy() - g[f"{case}_lpips64"]).max()
        assert err <= 0.5 * gap, (err, gap)
        err = abs(a[3] / nb - g[f"{case}_blp64"].mean())                # the mean of per-batch means
        assert err <= 0.5 * gap, (err, gap)


def test_lpips_metric_rejects_unsupported_shape():
    from vtp_b200.lpips import LPIPSMetric

    m = LPIPSMetric.random_init(0)
    with pytest.raises(ValueError, match="48x80"):
        m.parts(torch.zeros(1, 2, 3, 48, 80, device="cuda"))


# ---------------------------------------------------------------------------------------------------------- evaluator
def _tiny_model(tmp_path):
    from oracle.seeded import seeded_state_dict
    from vtp_b200.config import preset
    from vtp_b200.model import VTPModel

    cfg = preset("tiny")
    m = VTPModel(cfg)
    m.load_state_dict(seeded_state_dict({k: list(v.shape) for k, v in m.state_dict().items()}, seed=0))
    path = tmp_path / "model"
    m.save_pretrained(str(path))
    return str(path), m.cuda().eval()


def _weight_files(tmp_path):
    from vtp_b200.lpips import VGG_FEATURE_INDEX, random_weights

    vw, vb, lw = random_weights(0)
    vgg = {}
    for j, w, b in zip(VGG_FEATURE_INDEX, vw, vb):
        vgg[f"features.{j}.weight"], vgg[f"features.{j}.bias"] = w, b
    torch.save(vgg, tmp_path / "vgg16.pth")
    torch.save({f"lin{k}.model.1.weight": l for k, l in enumerate(lw)}, tmp_path / "lin.pth")
    return str(tmp_path / "vgg16.pth"), str(tmp_path / "lin.pth")


def test_graph_replay_equals_eager(tmp_path):
    from vtp_b200.lpips import LPIPSMetric
    from vtp_b200.recon_eval import ReconstructionEvaluator

    _, model = _tiny_model(tmp_path)
    lp = LPIPSMetric.random_init(0)
    batches = [_pair(4, 64, 64, torch.float32, seed=s)[0] for s in range(3)] + [_pair(2, 64, 64, torch.float32, seed=9)[0]]
    res = []
    for use_graph in (False, True, True):
        ev = ReconstructionEvaluator(model, lpips=lp, precision="bf16", use_graph=use_graph)
        for b in batches:
            ev.add(b)
        res.append((ev.result(), ev.per_image()))
        ev.close()
    for r, p in res[1:]:
        assert r == res[0][0]
        for k in ("psnr", "ssim", "lpips"):
            assert torch.equal(p[k], res[0][1][k]), k
    assert res[0][0]["num_samples"] == 14


def _image_folder(root, n):
    from PIL import Image

    rng = np.random.default_rng(0)
    for i in range(n):
        d = root / f"class{i % 2}"
        d.mkdir(parents=True, exist_ok=True)
        h, w = int(rng.integers(200, 400)), int(rng.integers(200, 400))
        arr = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
        img = Image.fromarray(arr)
        img.save(d / (f"img{i}.png" if i % 2 else f"img{i}.jpg"))


def test_cli_end_to_end(tmp_path):
    """python -m vtp_b200.recon_eval on a synthetic ImageFolder of 7 mixed-size JPEG / PNG images at batch 3 (ragged last
    batch) against the reference loop restated in eager torch over the same model outputs."""
    from PIL import Image
    from torchvision.datasets import ImageFolder

    from vtp_b200.recon_eval import main, make_transform

    mpath, model = _tiny_model(tmp_path)
    vgg, lin = _weight_files(tmp_path)
    data = tmp_path / "data"
    _image_folder(data, 7)
    outp = tmp_path / "out"
    args = ["--model_path", mpath, "--data_path", str(data), "--output_path", str(outp), "--batch_size", "3",
            "--num_workers", "0", "--device", "cuda:0", "--lpips_vgg", vgg, "--lpips_lin", lin]
    got = main(args)
    # the reference's loop, restated in eager torch
    from vtp_b200.lpips import load_weight_files

    vw, vb, lw = load_weight_files(vgg, lin)
    ds = ImageFolder(str(data), transform=make_transform(model.config.image_size))
    sub, div = _sub_div()
    psnr_v, ssim_v, lpips_v, ssim_y, lpips_y = [], [], [], [], []
    for s in range(0, 7, 3):
        imgs = torch.stack([ds[i][0] for i in range(s, min(7, s + 3))]).cuda()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            lat = model.get_reconstruction_latents(imgs)
        rec = model.get_latents_decoded_images(lat)
        o, r = _denorm(imgs, sub, div), _denorm(rec, sub, div)
        for i in range(o.shape[0]):
            d = (o[i].double() * 255 - r[i].double() * 255)
            psnr_v.append(float(20 * torch.log10(255.0 / torch.sqrt((d ** 2).mean()))))
        oc, rc = o.cpu(), r.cpu()
        s64 = ssim_valid_fp64(oc, rc)
        ssim_v.append(float(s64.mean()))
        ssim_y.append((ssim_torchmetrics_form(oc, rc, tf32=True).double() - s64).abs().max().item())
        with torch.no_grad():
            l64 = lpips_ref(o * 2 - 1, r * 2 - 1, vw, vb, lw, tf32=False)
            l32 = lpips_ref(o * 2 - 1, r * 2 - 1, vw, vb, lw, tf32=True)
        lpips_v.append(float(l64.mean()))
        lpips_y.append((l32 - l64).abs().max().item())
        for i in range(o.shape[0]):
            k = s + i
            ref_png = np.asarray(Image.open(outp / "reference" / f"ref_{k:06d}.png"))
            rec_png = np.asarray(Image.open(outp / "reconstructed" / f"rec_{k:06d}.png"))
            assert np.array_equal(ref_png, (o[i].permute(1, 2, 0).cpu().numpy() * 255.0).astype(np.uint8))
            assert np.array_equal(rec_png, (r[i].permute(1, 2, 0).cpu().numpy() * 255.0).astype(np.uint8))
    assert got["num_samples"] == 7 and got["fid"] is None
    assert abs(got["psnr"] - np.mean(psnr_v)) < 1e-4
    assert abs(got["ssim"] - np.mean(ssim_v)) <= 0.5 * max(ssim_y)
    assert abs(got["lpips"] - np.mean(lpips_v)) <= 0.5 * max(lpips_y)
    # images present: generation is skipped, as the reference does
    again = main(args)
    assert again == {"fid": None, "psnr": None, "lpips": None, "ssim": None, "num_samples": 7}
    assert len(os.listdir(outp / "reconstructed")) == 7


# ---------------------------------------------------------------------------------------------------------- 2 GPUs
def _free_port():
    import socket

    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _dist_worker(rank, world, port, tmp, out):
    import torch.distributed as dist
    from torch.utils.data import DistributedSampler

    from oracle.seeded import seeded_state_dict
    from vtp_b200.config import preset
    from vtp_b200.lpips import LPIPSMetric
    from vtp_b200.model import VTPModel
    from vtp_b200.recon_eval import ReconstructionEvaluator

    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    m = VTPModel(preset("tiny"))
    m.load_state_dict(seeded_state_dict({k: list(v.shape) for k, v in m.state_dict().items()}, seed=0))
    m = m.cuda().eval()
    lp = LPIPSMetric.random_init(0)
    N, bs = 7, 3
    data = _pair(N, 64, 64, torch.float32, seed=77)[0].cpu()
    idx = list(DistributedSampler(range(N), num_replicas=world, rank=rank, shuffle=False))   # padded: repeats sample 0
    shard = data[idx]
    sharded = ReconstructionEvaluator(m, lpips=lp, save_dir=tmp, batch_size=bs, total=N)      # world / rank from dist
    solo = ReconstructionEvaluator(m, lpips=lp, world=1, rank=0)                               # this rank's shard alone
    for s in range(0, len(idx), bs):
        sharded.add(shard[s:s + bs].cuda())
        solo.add(shard[s:s + bs].cuda())
    res, own = sharded.result(), solo.result()
    sharded.close()
    solo.close()
    out[rank] = (res, own, sharded.world, len(idx))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_run_equals_reference_ddp_arithmetic(tmp_path):
    """Two ranks over 7 images at batch 3 (DistributedSampler pads rank 1 with a repeat of image 0): every metric is the
    mean over ranks of each rank's own mean (test_reconstruction_hf.py:417-422), num_samples = images per rank * world
    (8, padding included), and the PNGs are the files of the reference's index formula."""
    import torch.multiprocessing as mp

    from vtp_b200.recon_eval import png_indices

    world = 2
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_dist_worker, args=(world, _free_port(), str(tmp_path), out), nprocs=world, join=True)
    own = [out[r][1] for r in range(world)]
    for r in range(world):
        res, _, w, n = out[r]
        assert w == world and n == 4
        assert res["num_samples"] == 8
        for k in ("psnr", "ssim", "lpips"):
            assert res[k] == pytest.approx((own[0][k] + own[1][k]) / 2, rel=1e-15, abs=0), k
    want = sorted(i for r in range(world) for b in range(2) for i in png_indices(b, 3, world, r, 3 if b == 0 else 1, 7))
    got = sorted(int(f[4:10]) for f in os.listdir(tmp_path / "reconstructed"))
    assert got == want
    assert sorted(int(f[4:10]) for f in os.listdir(tmp_path / "reference")) == want
