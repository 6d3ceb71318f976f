"""vtp_crop_augment (csrc/data.cu) per pixel against the fp64 restatement tests/photo_ref.py, bit-identity of an all-off
table with vtp_crop_resize_norm, buffer safety, determinism, argument errors, and TrainBatchPipeline(photometric=...).

The reference input is lib.crop_resize_norm(mean=0, std=1) on the same boxes and flips: both kernels share one bilinear
sampler, so that is the augment kernel's own pre-photometric value and the check isolates the photometric stages.
Errors are in [0, 1] units (output error x std) against photo_ref.PHOTO_TOL; pixels whose fp64 pre-solarise value lies
within photo_ref.SOLARIZE_BAND of the threshold are left out, and must be fewer than 0.1 %."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import photo_ref as pr
from vtp_b200 import lib
from vtp_b200.data import IMAGENET_MEAN, IMAGENET_STD, PHOTO_OFF, PhotometricAug, photometric_params, random_resized_crop_boxes

pytestmark = pytest.mark.gpu

MEAN, STD = IMAGENET_MEAN, IMAGENET_STD
PAD = 2            # NaN sentinel crops on each side of the output
WORST = {}         # case -> largest error measured, printed by the last test


def _src(B=5, H=150, W=170, seed=0):
    """uint8 NHWC: smooth colour fields plus noise, so every hue sector, both clamps and the solarise threshold occur"""
    g = torch.Generator().manual_seed(seed)
    coarse = torch.rand(B, 3, 5, 5, generator=g)
    x = torch.nn.functional.interpolate(coarse, size=(H, W), mode="bilinear", align_corners=False)
    x = 0.85 * x + 0.15 * torch.rand(B, 3, H, W, generator=g)
    return (x * 255).round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous().cuda()


def _geom(src, N, seed=0):
    B, H, W, _ = src.shape
    rng = np.random.default_rng(seed)
    boxes = torch.from_numpy(random_resized_crop_boxes(rng, N, H, W, (0.05, 1.0))).cuda()
    idx = torch.from_numpy(rng.integers(0, B, N).astype(np.int32)).cuda()
    flips = torch.from_numpy((rng.random(N) < 0.5).astype(np.uint8)).cuda()
    return idx, boxes, flips


def _augment(src, idx, boxes, flips, params, S):
    N = params.shape[0]
    full = torch.full((N + 2 * PAD, 3, S, S), float("nan"), device="cuda")
    out = full[PAD:PAD + N]
    ws = torch.empty(N, device="cuda")
    lib.crop_augment(src, idx, boxes, flips, params, ws, out, mean=MEAN, std=STD)
    torch.cuda.synchronize()
    assert torch.isnan(full[:PAD]).all() and torch.isnan(full[PAD + N:]).all()
    return out


def _plain(src, idx, boxes, flips, N, S, mean=MEAN, std=STD):
    out = torch.empty(N, 3, S, S, device="cuda")
    lib.crop_resize_norm(src, idx, boxes, flips, out, mean=mean, std=std)
    torch.cuda.synchronize()
    return out


def _check(case, table, S, seed=0, src=None):
    """per-pixel error of vtp_crop_augment against photo_ref on crops cut with `table` (np [N, 8])"""
    src = _src(seed=seed) if src is None else src
    N = table.shape[0]
    idx, boxes, flips = _geom(src, N, seed)
    params = torch.from_numpy(np.ascontiguousarray(table, dtype=np.float32)).cuda()
    out = _augment(src, idx, boxes, flips, params, S)
    again = _augment(src, idx, boxes, flips, params, S)
    assert torch.equal(out, again), "repeat launches differ"
    x01 = _plain(src, idx, boxes, flips, N, S, mean=(0, 0, 0), std=(1, 1, 1)).double()
    std = torch.tensor(STD, dtype=torch.float64, device="cuda")[:, None, None]
    worst, excluded = 0.0, 0
    for n in range(N):
        row = params[n].double().cpu().numpy()
        pre = pr.pre_solarize(x01[n], row)
        ref = pr.normalize(pr.solarize(pre, float(row[7])), MEAN, STD)
        err = (out[n].double() - ref).abs() * std
        near = (pre - float(row[7])).abs() < pr.SOLARIZE_BAND
        excluded += int(near.sum())
        worst = max(worst, err[~near].max().item())
    assert excluded < 1e-3 * out.numel(), (case, excluded)
    WORST[case] = max(WORST.get(case, 0.0), worst)
    assert worst <= pr.PHOTO_TOL, (case, worst, pr.PHOTO_TOL)


def _rows(n, code=-1, f=(1.0, 1.0, 1.0, 0.0), gray=0, sigma=0.0, t=2.0):
    return np.tile(np.array([*f, code, gray, sigma, t], dtype=np.float32), (n, 1))


@pytest.mark.parametrize("S", [5, 33, 96, 256, 512])
def test_all_off_table_is_bit_identical_to_crop_resize_norm(S):
    src = _src()
    N = 7
    idx, boxes, flips = _geom(src, N, seed=S)
    params = torch.tensor([PHOTO_OFF] * N, dtype=torch.float32, device="cuda")
    assert torch.equal(_augment(src, idx, boxes, flips, params, S), _plain(src, idx, boxes, flips, N, S))


STAGES = {
    "brightness": dict(code=0, f=(1.37, 1.0, 1.0, 0.0)),
    "contrast": dict(code=0, f=(1.0, 0.63, 1.0, 0.0)),
    "saturation": dict(code=0, f=(1.0, 1.0, 1.18, 0.0)),
    "hue": dict(code=0, f=(1.0, 1.0, 1.0, -0.07)),
    "grayscale": dict(gray=1),
    "blur": dict(sigma=1.3),
    "solarize": dict(t=128 / 255),
}


@pytest.mark.parametrize("stage", list(STAGES))
def test_each_stage_alone(stage):
    _check(stage, _rows(6, **STAGES[stage]), 96)


def test_all_24_orders():
    rng = np.random.default_rng(1)
    t = _rows(24)
    t[:, 0:3] = rng.uniform(0.6, 1.4, (24, 3))
    t[:, 3] = rng.uniform(-0.1, 0.1, 24)
    t[:, 4] = np.arange(24)
    _check("orders", t, 64)


def test_everything_on():
    t = _rows(8, code=0, f=(1.3, 0.7, 1.15, 0.08), gray=0, sigma=1.1, t=128 / 255)
    t[:, 4] = [3, 7, 11, 14, 16, 19, 21, 23]
    t[4:, 5] = 1
    _check("everything", t, 96)


def test_extreme_tables():
    rows = []
    for f in ((0.0, 0.0, 0.0, 0.5), (1.4, 1.4, 1.4, -0.5), (0.0, 1.4, 0.0, -0.5), (1.4, 0.0, 1.4, 0.5)):
        for code in (0, 23):
            for sigma in (0.05, 5.0):
                rows.append(_rows(1, code=code, f=f, sigma=sigma, t=128 / 255)[0])
    _check("extreme", np.stack(rows), 48)


@pytest.mark.parametrize("S", [5, 33, 97])
def test_ragged_tiles_and_smallest_crop(S):
    """S = 33 / 97 leave 1-pixel tile tails; at S = 5 the 4-pixel halo reaches the opposite border"""
    aug = PhotometricAug()
    t = photometric_params(np.random.default_rng(S), 24, aug, 1.0, 0.5)
    _check(f"S={S}", t, S)


def test_many_local_crops_in_one_launch():
    aug = PhotometricAug()
    t = photometric_params(np.random.default_rng(7), 2048, aug, aug.blur_p[2], 0.0)
    _check("2048 local crops", t, 96, src=_src(B=64, H=120, W=140, seed=3))


def test_argument_errors():
    src = _src(B=1, H=40, W=40)
    idx, boxes, flips = _geom(src, 4)
    params = torch.tensor([PHOTO_OFF] * 4, dtype=torch.float32, device="cuda")
    ws = torch.empty(4, device="cuda")
    with pytest.raises(lib.VtpError, match="S >= 5"):
        lib.crop_augment(src, idx, boxes, flips, params, ws, torch.empty(4, 3, 4, 4, device="cuda"))
    store = torch.zeros(4 * 8 + 1, device="cuda")
    with pytest.raises(lib.VtpError, match="aligned"):
        lib.crop_augment(src, idx, boxes, flips, store[1:].view(4, 8), ws, torch.empty(4, 3, 8, 8, device="cuda"))
    out = torch.full((4, 3, 8, 8), float("nan"), device="cuda")
    m = (C.c_float * 3)(*MEAN)
    sd = (C.c_float * 3)(*STD)
    raw = lib.load().vtp_crop_augment
    st = torch.cuda.current_stream().cuda_stream
    p = lambda t: t.data_ptr()
    good = [p(src), 1, 40, 40, p(idx), p(boxes), p(flips), p(params), p(ws), p(out), 4, 8, m, sd, st]
    for k, bad in ((7, store.data_ptr() + 4), (0, None), (4, None), (5, None), (7, None), (8, None), (9, None), (10, 0),
                   (11, 4)):
        args = list(good)
        args[k] = bad
        assert raw(*args) != 0, (k, bad)
    torch.cuda.synchronize()
    assert torch.isnan(out).all()          # nothing launched
    assert raw(*good) == 0
    torch.cuda.synchronize()
    assert not torch.isnan(out).any()


def _pipeline_steps(image_size, local_size, B, seed, steps=3):
    from oracle.seeded import seeded_captions
    from tests import test_train_gpu as tt
    from vtp_b200.data import TrainBatchPipeline

    tr = tt._setup("tiny").tr
    src = (torch.rand(B, image_size + 40, image_size + 60, 3, generator=torch.Generator().manual_seed(seed)) * 255).to(
        torch.uint8)
    ids = seeded_captions(B, 77, 1000)
    aug = PhotometricAug()
    pipes = [TrainBatchPipeline("cuda", image_size=image_size, local_size=local_size, n_local=2, seed=seed,
                                photometric=p) for p in (aug, None)]
    rng = np.random.default_rng([seed, 1])     # the pipeline's photometric seeding, reproduced
    off = lambda t: (t[:, 4] < 0) & (t[:, 5] == 0) & (t[:, 6] == 0) & (t[:, 7] == 2.0)
    n_off = 0
    for p in pipes:
        p.submit(src, ids)
    for _ in range(steps):
        (a, b) = [p.get() for p in pipes]
        for p in pipes:
            p.submit(src, ids)
        for k in ("image", "rec_image", "mask_indices", "masks_weight", "text"):
            assert torch.equal(a[k], b[k]), k
        tg = np.concatenate([photometric_params(rng, B, aug, aug.blur_p[0], 0.0),
                             photometric_params(rng, B, aug, aug.blur_p[1], aug.solarize_p)])
        tl = photometric_params(rng, 2 * B, aug, aug.blur_p[2], 0.0)
        for key, t in (("global_crops", tg), ("local_crops", tl)):
            for n in range(t.shape[0]):
                assert torch.equal(a[key][n], b[key][n]) == bool(off(t)[n]), (key, n, t[n])
            n_off += int(off(t).sum())
        loss = tr.train_step(a).cpu()
        assert torch.isfinite(loss).all(), loss
    for p in pipes:
        p.get()
        p.close()
    assert n_off > 0        # the seeds are chosen so that some crop draws an all-off row


@pytest.mark.parametrize("sizes", [(64, 32, 4, 3), (512, 192, 2, 1)], ids=["64-32", "512-192"])
def test_pipeline_with_photometric_augmentation(sizes):
    _pipeline_steps(*sizes)


def test_zz_report_worst_errors():
    print("\nlargest per-pixel error, [0, 1] units:", {k: f"{v:.2e}" for k, v in WORST.items()},
          f"bound {pr.PHOTO_TOL:.1e}")
