"""FID on the device (vtp_b200/fid.py, csrc/fid.cu) against torch and the fp64 reference network (oracle/fid_inception.py).

The yardstick for the features is what pytorch-fid runs on an H100: the fp32 network with cuDNN's default TF32
convolutions, modelled by TF32-rounded conv operands.  Each image's features must lie within half of that network's
distance from the fp64 network."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.fid_inception import features as oracle_features
from oracle.fid_inception import fid_inception, set_operand_rounding
from tests.ssim_ref import round_tf32
from vtp_b200 import fid, lib

pytestmark = pytest.mark.gpu


def _u8(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8).cuda()


@pytest.mark.parametrize("H,W", [(64, 64), (256, 256), (48, 80), (299, 299), (512, 512), (11, 13)])
def test_resize_bit_identical_to_torch(H, W):
    u8 = _u8(3, H, W, seed=H * 7 + W)
    out = torch.full((3, 299, 299, 3), float("nan"), device="cuda")
    lib.fid_resize(u8, out)
    x = F.interpolate(u8.permute(0, 3, 1, 2).float() / 255, size=(299, 299), mode="bilinear", align_corners=False)
    want = (2 * x - 1).permute(0, 2, 3, 1)
    assert torch.equal(out, want), (out - want).abs().max().item()


CONV_SHAPES = sorted({v[2:] for v in fid.CONVS.values() if v[2:] != (1, 1, 1, 0, 0)})


@pytest.mark.parametrize("kh,kw,s,ph,pw", CONV_SHAPES)
def test_im2col3_every_conv_geometry(kh, kw, s, ph, pw):
    B, H, W, C, ld, c0 = 2, 17, 13, 16, 28, 8
    x = torch.randn(B, H, W, ld, device="cuda")
    x[..., :c0] = float("nan")                              # channels outside the slice must not be read
    x[..., c0 + C:] = float("nan")
    Ho, Wo = lib.fid_conv_out(H, W, kh, kw, s, ph, pw)
    out = torch.full((B * Ho * Wo, kh * kw * 3 * C), float("nan"), dtype=torch.bfloat16, device="cuda")
    lib.fid_im2col3(x, out, B, H, W, C, (kh, kw), s, (ph, pw), c0=c0)
    xs = x[..., c0:c0 + C].permute(0, 3, 1, 2)
    xp = F.pad(xs, (pw, pw, ph, ph))
    taps = [xp[:, :, dy:dy + (Ho - 1) * s + 1:s, dx:dx + (Wo - 1) * s + 1:s] for dy in range(kh) for dx in range(kw)]
    ref = torch.stack(taps, 1).permute(0, 3, 4, 1, 2).reshape(B * Ho * Wo, kh * kw, C)   # [M, taps, C] fp32
    o = out.view(B * Ho * Wo, kh * kw, 3, C)
    hi = ref.to(torch.bfloat16)
    lo = (ref - hi.float()).to(torch.bfloat16)
    assert torch.equal(o[:, :, 0], hi) and torch.equal(o[:, :, 1], hi) and torch.equal(o[:, :, 2], lo)
    rec = o[:, :, 1].float() + o[:, :, 2].float()
    exact = (ref - hi.float()) == lo.float()
    assert torch.equal(rec[exact], ref[exact])
    assert ((rec - ref).abs() <= 2.0 ** -17 * ref.abs()).all()


def test_im2col3_stem():
    B, H, W = 2, 299, 299
    x = torch.randn(B, H, W, 3, device="cuda")
    Ho, Wo = lib.fid_conv_out(H, W, 3, 3, 2, 0, 0)
    out = torch.full((B * Ho * Wo, 96), float("nan"), dtype=torch.bfloat16, device="cuda")
    lib.fid_im2col3(x, out, B, H, W, 3, (3, 3), 2, (0, 0))
    xs = x.permute(0, 3, 1, 2)
    taps = [xs[:, :, dy:dy + 2 * Ho - 1:2, dx:dx + 2 * Wo - 1:2] for dy in range(3) for dx in range(3)]
    ref = torch.zeros(B * Ho * Wo, 32, device="cuda")
    ref[:, :27] = torch.stack(taps, 1).permute(0, 3, 4, 1, 2).reshape(-1, 27)
    hi = ref.to(torch.bfloat16)
    lo = (ref - hi.float()).to(torch.bfloat16)
    assert torch.equal(out, torch.cat([hi, hi, lo], 1))


@pytest.mark.parametrize("mode", [lib.FID_POOL_MAX2, lib.FID_POOL_MAX1, lib.FID_POOL_AVG1])
@pytest.mark.parametrize("H,W", [(35, 35), (17, 17), (8, 8), (147, 147)])
def test_pool_into_channel_slice(mode, H, W):
    B, C, ld, c0 = 2, 24, 40, 8
    x = torch.randn(B, H, W, C, device="cuda")
    Ho, Wo = lib.fid_conv_out(H, W, 3, 3, 2, 0, 0) if mode == lib.FID_POOL_MAX2 else (H, W)
    out = torch.full((B, Ho, Wo, ld), float("nan"), device="cuda")
    lib.fid_pool(x, out, B, H, W, mode, c0)
    assert out[..., :c0].isnan().all() and out[..., c0 + C:].isnan().all()
    got = out[..., c0:c0 + C].permute(0, 3, 1, 2)
    xs = x.permute(0, 3, 1, 2)
    if mode == lib.FID_POOL_MAX2:
        assert torch.equal(got, F.max_pool2d(xs, 3, 2))
    elif mode == lib.FID_POOL_MAX1:
        assert torch.equal(got, F.max_pool2d(xs, 3, 1, 1))
    else:
        want = F.avg_pool2d(xs.double(), 3, 1, 1, count_include_pad=False)
        mag = F.avg_pool2d(xs.double().abs(), 3, 1, 1, count_include_pad=False)
        assert ((got.double() - want).abs() <= 9 * 2.0 ** -24 * mag + 1e-30).all()


# ---------------------------------------------------------------------------------------------------------- network
@pytest.fixture(scope="module")
def net():
    return fid.FIDInception.random_init(0)


@pytest.fixture(scope="module")
def oracles():
    sd = fid.random_weights(0)
    n64 = fid_inception(sd, dtype=torch.float64, device="cuda")
    n32 = fid_inception(sd, dtype=torch.float32, device="cuda")
    set_operand_rounding(n32, round_tf32)
    return n64, n32


@pytest.mark.parametrize("B,H,W", [(50, 256, 256), (5, 64, 96)])
def test_features_against_fp64_with_tf32_yardstick(net, oracles, B, H, W):
    """B = 50 runs as chunks of 16, 16, 16 and a ragged 2."""
    u8 = _u8(B, H, W, seed=B + H)
    got = net.features(u8).double()
    img = u8.permute(0, 3, 1, 2).float() / 255
    n64, n32 = oracles
    want = torch.cat([oracle_features(n64, img[s:s + 10]) for s in range(0, B, 10)])
    tf = torch.cat([oracle_features(n32, img[s:s + 10]).double() for s in range(0, B, 10)])
    err = (got - want).abs().amax(1)
    yard = (tf - want).abs().amax(1)
    ratio = (err / yard).max().item()
    print(f"features {B}x{H}x{W}: max per-image err / TF32 yardstick = {ratio:.4f}; err max {err.max().item():.3e}, "
          f"yard min {yard.min().item():.3e}; feature mean {want.mean().item():.3f}, dead pool3 channels "
          f"{(want.amax(0) == 0).double().mean().item():.4f}")
    assert (yard > 0).all()
    assert ratio <= 0.5
    assert 0.05 < want.mean().item() < 20            # activations O(1) with the stand-in weights
    assert (want.amax(0) == 0).double().mean().item() <= 0.02


def test_moments_sums_rows_and_determinism(net):
    B = 20
    u8 = _u8(B, 64, 64, seed=3)
    feat = net.features(u8).double().cpu()
    st = fid.FIDStatistics()
    rows = torch.tensor([13], dtype=torch.int32, device="cuda")
    net.accumulate(u8, st, rows)
    f = feat[:13]
    S2 = np.triu(st.S2.cpu().numpy())
    want2 = np.triu((f.T @ f).numpy())
    assert np.linalg.norm(S2 - want2) <= 1e-12 * np.linalg.norm(want2)
    assert np.linalg.norm(st.S1.cpu().numpy() - f.sum(0).numpy()) <= 1e-12 * np.linalg.norm(f.sum(0).numpy())
    assert st.count() == 13
    # rows at or above `rows` change nothing, even NaN ones
    last = torch.randn(B, 64, 2048, device="cuda").abs()
    last[13:] = float("nan")
    a, b = fid.FIDStatistics(), fid.FIDStatistics()
    lib.fid_moments(last, rows, a.S2, a.S1, a.n)
    lib.fid_moments(last[:13].contiguous(), torch.tensor([13], dtype=torch.int32, device="cuda"), b.S2, b.S1, b.n)
    assert torch.equal(a.buf, b.buf) and not a.buf.isnan().any()
    # two launches and a graph replay are bit-identical with eager
    c, d = fid.FIDStatistics(), fid.FIDStatistics()
    net.accumulate(u8, c, rows)
    assert torch.equal(c.buf, st.buf)
    net.accumulate(u8, d, rows)          # warm-up of every shape before capture
    d.reset()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        net.accumulate(u8, d, rows)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(d.buf, st.buf)


def _pytorch_fid_formula(f1, f2):
    """pytorch-fid's statistics restated on fp32 features (np.mean, np.cov) and its distance."""
    f1, f2 = f1.cpu().numpy(), f2.cpu().numpy()
    return fid.frechet_distance(np.mean(f1, axis=0), np.cov(f1, rowvar=False), np.mean(f2, axis=0),
                                np.cov(f2, rowvar=False))


def test_fid_full_rank_against_pytorch_fid_formula(net):
    N, bs = 2304, 64
    sts, feats = [fid.FIDStatistics(), fid.FIDStatistics()], [[], []]
    for side in range(2):
        for s in range(0, N, bs):
            u8 = _u8(bs, 32, 32, seed=10_000 * side + s)
            if side:
                u8 = (u8.float() * 0.8).to(torch.uint8)
            net.accumulate(u8, sts[side], bs)
            feats[side].append(net.features(u8))
    got = fid.frechet_distance(*sts[0].mu_sigma(), *sts[1].mu_sigma())
    want = _pytorch_fid_formula(torch.cat(feats[0]), torch.cat(feats[1]))
    rel = abs(got - want) / abs(want)
    print(f"FID N = 2 x {N}: device moments {got:.10g}, pytorch-fid formula on the device features {want:.10g}, rel {rel:.2e}")
    assert rel <= 1e-6


# ---------------------------------------------------------------------------------------------------------- tools
def _weights_file(tmp_path):
    p = str(tmp_path / "fid_inception_random.pth")
    torch.save(fid.random_weights(0), p)
    return p


def test_recon_eval_rfid(tmp_path):
    from tests.test_recon_eval_gpu import _image_folder, _tiny_model, _weight_files
    from vtp_b200.recon_eval import main

    mpath, _ = _tiny_model(tmp_path)
    vgg, lin = _weight_files(tmp_path)
    w = _weights_file(tmp_path)
    data = tmp_path / "data"
    _image_folder(data, 7)
    outp = tmp_path / "out"
    args = ["--model_path", mpath, "--data_path", str(data), "--output_path", str(outp), "--batch_size", "3",
            "--num_workers", "0", "--device", "cuda:0", "--lpips_vgg", vgg, "--lpips_lin", lin]
    plain = main(args)
    assert plain["fid"] is None
    outp2 = tmp_path / "out2"
    args2 = [a if a != str(outp) else str(outp2) for a in args] + ["--fid_weights", w]
    got = main(args2)
    assert isinstance(got["fid"], float)
    for k in ("psnr", "ssim", "lpips", "num_samples"):
        assert got[k] == plain[k], k
    model = fid.FIDInception.from_file(w)
    want = fid.fid_from_paths([str(outp2 / "reference"), str(outp2 / "reconstructed")], model=model)
    print(f"rFID in the step {got['fid']!r}, from the PNGs {want!r}")
    assert got["fid"] == pytest.approx(want, rel=1e-9)
    again = main(args2)                                      # PNGs present: the skip path computes rFID from them
    assert again["fid"] == pytest.approx(got["fid"], rel=1e-9) and again["psnr"] is None


def test_cli_two_folders_and_save_stats(tmp_path, capsys):
    from PIL import Image

    model = fid.FIDInception.random_init(0)
    w = _weights_file(tmp_path)
    rng = np.random.default_rng(0)
    dirs = [tmp_path / "a", tmp_path / "b"]
    arrs = [[], []]
    for k, d in enumerate(dirs):
        d.mkdir()
        for i in range(9):
            shape = (40, 56, 3) if i % 4 == 3 else (48, 48, 3)      # a size change starts a new batch
            a = rng.integers(0, 256 - 60 * k, size=shape, dtype=np.uint8)
            Image.fromarray(a).save(d / f"img{i:02d}.png")
            arrs[k].append(a)
    with pytest.raises(RuntimeError, match="Invalid path"):
        fid.main([str(dirs[0]), str(tmp_path / "missing"), "--weights", w])
    got = fid.main([str(dirs[0]), str(dirs[1]), "--weights", w, "--batch-size", "4", "--num-workers", "2"])
    assert "FID: " in capsys.readouterr().out
    # each file's features one at a time, in the sorted file order: the CLI's batching (by size, then batch_size) and
    # row counts must give the statistics of exactly these, up to the fp64 summation order
    feats = [torch.cat([model.features(torch.from_numpy(a[None]).cuda()) for a in arrs[k]]) for k in range(2)]
    for k in range(2):
        mu, sigma = fid.statistics_of_path(str(dirs[k]), model, batch_size=4, num_workers=2)
        f = feats[k].double().cpu().numpy()
        assert np.abs(mu - f.mean(0)).max() <= 1e-12 * np.abs(f).max()
        want_s = np.cov(f, rowvar=False)
        assert np.linalg.norm(sigma - want_s) <= 1e-10 * np.linalg.norm(want_s)
    # with 9 images the covariances are singular and sqrtm of their product is ill-conditioned: rounding-level
    # differences in sigma move the distance by ~1e-8 relative
    want = _pytorch_fid_formula(*feats)
    assert got == pytest.approx(want, rel=1e-6)
    npz = str(tmp_path / "a.npz")
    fid.main([str(dirs[0]), npz, "--weights", w, "--save-stats"])
    with pytest.raises(RuntimeError, match="Existing output file"):
        fid.main([str(dirs[0]), npz, "--weights", w, "--save-stats"])
    from_npz = fid.main([npz, str(dirs[1]), "--weights", w])
    assert from_npz == pytest.approx(got, rel=1e-5)             # mu is stored in fp32, as pytorch-fid stores it


# ---------------------------------------------------------------------------------------------------------- 2 GPUs
def _dist_worker(rank, world, port, tmp, wpath, out):
    import torch.distributed as dist

    from oracle.seeded import seeded_state_dict
    from vtp_b200.config import preset
    from vtp_b200.model import VTPModel
    from vtp_b200.recon_eval import ReconstructionEvaluator

    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    m = VTPModel(preset("tiny"))
    m.load_state_dict(seeded_state_dict({k: list(v.shape) for k, v in m.state_dict().items()}, seed=0))
    m = m.cuda().eval()
    from torch.utils.data import DistributedSampler

    N, bs = 7, 3
    g = torch.Generator().manual_seed(77)
    data = torch.randn(N, 3, 64, 64, generator=g) * 1.2
    idx = list(DistributedSampler(range(N), num_replicas=world, rank=rank, shuffle=False))
    shard = data[idx]
    ev = ReconstructionEvaluator(m, save_dir=tmp, batch_size=bs, total=N, fid=fid.FIDInception.from_file(wpath))
    for s in range(0, len(idx), bs):
        ev.add(shard[s:s + bs].cuda())
    res = ev.result()
    ev.close()
    out[rank] = res["fid"]
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_rfid_covers_exactly_the_written_pngs(tmp_path):
    import torch.multiprocessing as mp

    from tests.test_recon_eval_gpu import _free_port

    w = _weights_file(tmp_path)
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_dist_worker, args=(2, _free_port(), str(tmp_path), w, out), nprocs=2, join=True)
    assert out[1] is None and isinstance(out[0], float)
    want = fid.fid_from_paths([str(tmp_path / "reference"), str(tmp_path / "reconstructed")],
                              model=fid.FIDInception.from_file(w))
    assert out[0] == pytest.approx(want, rel=1e-9)
