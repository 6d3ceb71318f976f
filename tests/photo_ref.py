"""Plain-torch fp64 restatement of vtp_crop_augment's photometric stages (csrc/data.cu) on one crop, on the CPU or the
GPU (no kernels).  Semantics are torchvision.transforms.v2.functional's on float images in [0, 1]; the stages are exposed
one by one so that tests can compose them, and mutate them.

apply(x01, row, mean, std)   the whole chain on x01 fp64 [3, S, S]: colour jitter (4 ops in the row's order, a clamp to
                             [0, 1] after each) -> grayscale -> 9-tap Gaussian blur (reflect padding) -> solarise ->
                             (x - mean[c]) / std[c].  `row` is one 8-float row of the params table (include/vtp_b200.h).
pre_solarize(x01, row)       the chain up to and including the blur, in [0, 1]: what the solarise threshold is compared against.
"""
import itertools

import torch
import torch.nn.functional as F

ORDERS = list(itertools.permutations(range(4)))   # order code -> (op, op, op, op); 0 brightness 1 contrast 2 saturation 3 hue
GRAY = (0.2989, 0.587, 0.114)
RADIUS = 4                                         # kernel size 9

# Per-pixel bound of tests/test_photometric_gpu.py in [0, 1] units (output error x std): about 1.5x the largest error
# measured on an H100 80GB HBM3 (700 W limit), capped at 5e-5; largest measured 1.75e-6, on 2 048 local crops drawn from
# the DINOv2 recipe (per stage alone: 1.3e-7 solarise to 6.5e-7 saturation; extreme tables 1.3e-6).  Pixels whose fp64 pre-solarise value lies within
# SOLARIZE_BAND of the threshold are left out of the comparison (a last-bit difference flips them to 1 - x).
PHOTO_TOL = 2.7e-6
SOLARIZE_BAND = 1e-5


def gray(x):
    """rgb_to_grayscale, one channel [S, S]"""
    return GRAY[0] * x[0] + GRAY[1] * x[1] + GRAY[2] * x[2]


def _blend(a, b, r):
    return (r * a + (1.0 - r) * b).clamp(0.0, 1.0)


def brightness(x, f):
    return (x * f).clamp(0.0, 1.0)


def contrast(x, f, mean=None):
    """blend towards the scalar grayscale mean of x (or the given `mean`)"""
    return _blend(x, gray(x).mean() if mean is None else mean, f)


def saturation(x, f):
    return _blend(x, gray(x)[None], f)


def rgb_to_hsv(x):
    """torchvision's _rgb_to_hsv: ties resolve to r first, then g"""
    r, g, _ = x
    maxc, minc = x.max(0).values, x.min(0).values
    eqc = maxc == minc
    cr = maxc - minc
    s = cr / torch.where(eqc, torch.ones_like(maxc), maxc)
    rc, gc, bc = (maxc - x) / torch.where(eqc, torch.ones_like(cr), cr)
    h = torch.where(maxc == r, bc - gc, torch.where(maxc == g, 2.0 + rc - bc, 4.0 + gc - rc))
    return torch.fmod(h / 6.0 + 1.0, 1.0), s, maxc


def hsv_to_rgb(h, s, v):
    """torchvision's _hsv_to_rgb: sector floor(6h) taken with a floored remainder(6)"""
    h6 = h * 6.0
    i = torch.floor(h6)
    f = h6 - i
    i = i.long().remainder(6)
    sxf = s * f
    q = ((1.0 - sxf) * v).clamp(0.0, 1.0)
    t = ((sxf + 1.0 - s) * v).clamp(0.0, 1.0)
    p = ((1.0 - s) * v).clamp(0.0, 1.0)
    vpqt = torch.stack((v, p, q, t))
    select = torch.tensor([[0, 2, 1, 1, 3, 0], [3, 0, 0, 2, 1, 1], [1, 1, 3, 0, 0, 2]], device=h.device)
    return vpqt.gather(0, select[:, i])


def hue(x, dh):
    h, s, v = rgb_to_hsv(x)
    return hsv_to_rgb((h + dh).remainder(1.0), s, v)


def jitter(x, row, mean=None):
    """the row's four jitter ops in its order; `mean` overrides contrast's blend target"""
    code = int(row[4])
    if code < 0:
        return x
    for op in ORDERS[code]:
        f = float(row[op])
        if op == 0:
            x = brightness(x, f)
        elif op == 1:
            x = contrast(x, f, mean)
        elif op == 2:
            x = saturation(x, f)
        else:
            x = hue(x, f)
    return x


def grayscale(x):
    return gray(x)[None].expand(3, -1, -1).clone()


def blur_kernel(sigma, radius=RADIUS, dtype=torch.float64, device=None):
    k = torch.arange(-radius, radius + 1, dtype=dtype, device=device)
    w = torch.exp(-k * k / (2.0 * sigma * sigma))
    return w / w.sum()


def blur(x, sigma, radius=RADIUS, mode="reflect"):
    """separable (2 radius + 1)-tap Gaussian, padded with `mode` at the crop border"""
    w = blur_kernel(sigma, radius, x.dtype, x.device)
    y = F.pad(x[None], (radius,) * 4, mode=mode)
    y = F.conv2d(y, w.view(1, 1, 1, -1).expand(3, 1, 1, -1), groups=3)
    return F.conv2d(y, w.view(1, 1, -1, 1).expand(3, 1, -1, 1), groups=3)[0]


def solarize(x, t):
    return torch.where(x >= t, 1.0 - x, x)


def normalize(x, mean, std):
    m = torch.tensor(mean, dtype=x.dtype, device=x.device)[:, None, None]
    s = torch.tensor(std, dtype=x.dtype, device=x.device)[:, None, None]
    return (x - m) / s


def pre_solarize(x01, row):
    x = jitter(x01, row)
    if row[5] != 0:
        x = grayscale(x)
    if row[6] > 0:
        x = blur(x, float(row[6]))
    return x


def apply(x01, row, mean, std):
    return normalize(solarize(pre_solarize(x01, row), float(row[7])), mean, std)
