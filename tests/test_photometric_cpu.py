"""Photometric augmentations without a GPU: tests/photo_ref.py against torchvision.transforms.v2.functional in fp64,
seeded mutations of the stage chain that the GPU bound must catch, and the statistics of the host sampler
(vtp_b200.data.photometric_params)."""
import numpy as np
import pytest
import torch
from scipy import stats

from tests import photo_ref as pr
from vtp_b200.data import PHOTO_OFF, PhotometricAug, photometric_params

EXACT = 1e-12


def _img(S, seed=0):
    """fp64 [3, S, S] in [0, 1]: a smooth colour field plus noise, so that every hue sector and both clamps occur"""
    g = torch.Generator().manual_seed(seed)
    coarse = torch.rand(1, 3, 4, 4, generator=g, dtype=torch.float64)
    x = torch.nn.functional.interpolate(coarse, size=(S, S), mode="bilinear", align_corners=False)[0]
    return (0.8 * x + 0.2 * torch.rand(3, S, S, generator=g, dtype=torch.float64)).clamp(0, 1)


def _row(code=-1, f=(1.3, 0.7, 1.15, 0.08), gray=0, sigma=0.0, t=2.0):
    return np.array([*f, code, gray, sigma, t], dtype=np.float64)


# ------------------------------------------------------------------------------------------------------ torchvision
tv = pytest.importorskip("torchvision.transforms.v2.functional", reason="torchvision is not installed")


def _tv_hue(x, dh):
    """adjust_hue computes in fp32 whatever the input dtype; its own _rgb_to_hsv / _hsv_to_rgb kept in fp64"""
    from torchvision.transforms.v2.functional._color import _hsv_to_rgb, _rgb_to_hsv

    h, s, v = _rgb_to_hsv(x).unbind(-3)
    return _hsv_to_rgb(torch.stack(((h + dh).remainder(1.0), s, v), -3))


def _tv_jitter(x, row):
    for op in pr.ORDERS[int(row[4])]:
        f = float(row[op])
        x = (lambda: tv.adjust_brightness(x, f), lambda: tv.adjust_contrast(x, f), lambda: tv.adjust_saturation(x, f),
             lambda: _tv_hue(x, f))[op]()
    return x


def _close(a, b, tol=EXACT):
    assert (a - b).abs().max().item() <= tol


def test_each_op_matches_torchvision():
    x = _img(33)
    for f in (0.0, 0.6, 1.0, 1.4):
        _close(pr.brightness(x, f), tv.adjust_brightness(x, f))
        _close(pr.contrast(x, f), tv.adjust_contrast(x, f))
        _close(pr.saturation(x, f), tv.adjust_saturation(x, f))
    for dh in (-0.5, -0.1, -0.03, 0.0, 0.07, 0.1, 0.5):
        _close(pr.hue(x, dh), _tv_hue(x, dh))
        _close(pr.hue(x, dh), tv.adjust_hue(x, dh), 1e-6)       # the public op, in its fp32
    _close(pr.grayscale(x), tv.rgb_to_grayscale(x, num_output_channels=3))
    for t in (0.2, 128 / 255, 0.9):
        _close(pr.solarize(x, t), tv.solarize(x, t))


def test_all_jitter_orders_match_torchvision():
    x = _img(24, seed=1)
    for code in range(24):
        row = _row(code)
        _close(pr.jitter(x, row), _tv_jitter(x, row))
        # grayscale after the jitter
        _close(pr.pre_solarize(x, _row(code, gray=1)), tv.rgb_to_grayscale(_tv_jitter(x, row), num_output_channels=3))


@pytest.mark.parametrize("S", [5, 33, 96])
def test_blur_matches_torchvision(S):
    x = _img(S, seed=2)
    for sigma in (0.1, 0.7, 2.0):
        _close(pr.blur(x, sigma), tv.gaussian_blur(x, [9, 9], [sigma, sigma]))


def test_whole_chain_matches_torchvision():
    x = _img(40, seed=3)
    mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    row = _row(17, f=(0.8, 1.3, 0.9, -0.06), gray=0, sigma=1.3, t=128 / 255)
    y = tv.solarize(tv.gaussian_blur(_tv_jitter(x, row), [9, 9], [1.3, 1.3]), 128 / 255)
    _close(pr.apply(x, row, mean, std), tv.normalize(y, list(mean), list(std)))
    _close(pr.apply(x, np.array(PHOTO_OFF), mean, std), tv.normalize(x, list(mean), list(std)))


# ------------------------------------------------------------------------------------------------------ mutations
def _reference(x, row):
    return pr.solarize(pr.pre_solarize(x, row), float(row[7]))


def _mutants(x, row):
    """name -> (mutated chain output, the correct one) for each seeded bug"""
    code, sigma, t = int(row[4]), float(row[6]), float(row[7])
    ok = _reference(x, row)

    def chain(jit=None, gray_first=False, blur_fn=None, solar_first=False):
        y = x
        if gray_first:
            y = pr.grayscale(y)
        y = (jit or pr.jitter)(y, row)
        if row[5] and not gray_first:
            y = pr.grayscale(y)
        if solar_first:
            y = pr.solarize(y, t)
        y = (blur_fn or pr.blur)(y, sigma)
        return y if solar_first else pr.solarize(y, t)

    rev = row.copy()
    rev[4] = pr.ORDERS.index(tuple(reversed(pr.ORDERS[code])))
    neg = row.copy()
    neg[3] = -row[3]
    out = {
        "replicate padding": chain(blur_fn=lambda y, s: pr.blur(y, s, mode="replicate")),
        "blur radius 3": chain(blur_fn=lambda y, s: pr.blur(y, s, radius=3)),
        "blur radius 5": chain(blur_fn=lambda y, s: pr.blur(y, s, radius=5)),
        "contrast mean before the preceding ops": chain(jit=lambda y, r: pr.jitter(y, r, mean=pr.gray(y).mean())),
        "jitter order reversed": _reference(x, rev),
        "hue shift negated": _reference(x, neg),
        "grayscale before jitter": chain(gray_first=True),
        "solarise before blur": chain(solar_first=True),
    }
    saved = pr.GRAY
    pr.GRAY = (0.299, 0.587, 0.114)
    try:
        out["0.299 in place of 0.2989"] = _reference(x, row)
    finally:
        pr.GRAY = saved
    return {k: (v, ok) for k, v in out.items()}


def test_seeded_mutations_are_caught_with_margin():
    """each mutation moves some pixel of the test crops by at least 2x the GPU bound (in [0, 1] units).  The crops have
    contrast after brightness (so the early mean differs), a large hue shift, grayscale on, blur sigma 2 and a
    solarise threshold the blurred image crosses."""
    worst = {}
    for S, seed in ((33, 4), (96, 5)):
        x = _img(S, seed)
        for code in (pr.ORDERS.index((0, 1, 3, 2)), pr.ORDERS.index((3, 0, 1, 2))):
            for gray in (0, 1):
                row = _row(code, f=(1.4, 0.6, 1.2, 0.1), gray=gray, sigma=2.0, t=0.5)
                for name, (bad, ok) in _mutants(x, row).items():
                    worst[name] = max(worst.get(name, 0.0), (bad - ok).abs().max().item())
    for name, d in worst.items():
        assert d >= 2 * pr.PHOTO_TOL, (name, d, pr.PHOTO_TOL)
    print({k: f"{v / pr.PHOTO_TOL:.0f}x" for k, v in worst.items()})


# ------------------------------------------------------------------------------------------------------ host sampler
N_DRAWS = 200_000


def _within(count, n, p, k=5.0):
    return abs(count - n * p) <= k * np.sqrt(n * p * (1 - p)) + 1e-9


def test_sampler_statistics():
    aug = PhotometricAug()
    views = {"global1": (aug.blur_p[0], 0.0), "global2": (aug.blur_p[1], aug.solarize_p), "local": (aug.blur_p[2], 0.0)}
    for name, (bp, sp) in views.items():
        t = photometric_params(np.random.default_rng(11), N_DRAWS, aug, bp, sp)
        assert t.dtype == np.float32 and t.shape == (N_DRAWS, 8)
        jit, gray, blur, sol = t[:, 4] >= 0, t[:, 5] != 0, t[:, 6] > 0, t[:, 7] < 2.0
        for flag, p in ((jit, aug.jitter_p), (gray, aug.gray_p), (blur, bp), (sol, sp)):
            assert _within(int(flag.sum()), N_DRAWS, p), (name, p, int(flag.sum()))
        assert ((t[:, 0] >= 0.6) & (t[:, 0] <= 1.4)).all() and ((t[:, 1] >= 0.6) & (t[:, 1] <= 1.4)).all()
        assert ((t[:, 2] >= 0.8) & (t[:, 2] <= 1.2)).all() and (np.abs(t[:, 3]) <= 0.1).all()
        assert ((t[blur, 6] >= 0.1) & (t[blur, 6] <= 2.0)).all() and (t[~blur, 6] == 0).all()
        assert (t[sol, 7] == np.float32(128 / 255)).all() and (t[~sol, 7] == 2.0).all()
        assert set(np.unique(t[:, 5]).tolist()) <= {0.0, 1.0} and (t[~jit, 4] == -1).all()
        codes = np.bincount(t[jit, 4].astype(np.int64), minlength=24)
        assert codes.size == 24 and (codes > 0).all()
        assert stats.chisquare(codes).pvalue > 1e-4, (name, codes)
        if name == "global1":
            assert blur.all()
        if name != "global2":
            assert not sol.any()
    a = photometric_params(np.random.default_rng(3), 1000, aug, 0.5, 0.2)
    b = photometric_params(np.random.default_rng(3), 1000, aug, 0.5, 0.2)
    assert np.array_equal(a, b)
