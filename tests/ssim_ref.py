"""Two restatements of torchmetrics' StructuralSimilarityIndexMeasure(data_range=1.0) per-image values (the reference's
SSIM, tools/test_reconstruction_hf.py:82-86,392).  torchmetrics is not installed here, so these are written from its
algorithm, not checked against the package:

  * `ssim_torchmetrics_form`: reflect pad by 5, one grouped F.conv2d of the 11x11 Gaussian over (x, y, x², y², xy),
    the SSIM map, its 5-pixel border cropped, mean per image.  `round_tf32` rounds every conv operand to TF32 first,
    as cuDNN's default conv precision does on an H100.
  * `ssim_valid_fp64`: the mean over the 11x11 windows wholly inside the image, in fp64.
"""
import torch
import torch.nn.functional as F

SIGMA, K = 1.5, 11
C1, C2 = 0.01 ** 2, 0.03 ** 2


def gaussian_1d(dtype=torch.float32):
    d = torch.arange((1 - K) / 2, (1 + K) / 2, 1, dtype=dtype)
    g = torch.exp(-((d / SIGMA) ** 2) / 2)
    return g / g.sum()


def round_tf32(t: torch.Tensor) -> torch.Tensor:
    """Round fp32 values to TF32 (10 explicit mantissa bits), nearest-even."""
    b = t.float().contiguous().view(torch.int32)
    b = (b + 0x0FFF + ((b >> 13) & 1)) & ~0x1FFF
    return b.view(torch.float32)


def _map(x, y, win, round_ops=None):
    C = x.shape[1]
    r = round_ops or (lambda t: t)
    stack = torch.cat([x, y, x * x, y * y, x * y])
    out = F.conv2d(r(stack), r(win.expand(C, 1, K, K).contiguous()), groups=C)
    B = x.shape[0]
    mx, my, exx, eyy, exy = out.split(B)
    mxx, myy, mxy = mx.pow(2), my.pow(2), mx * my
    vx = torch.clamp(exx - mxx, min=0.0)
    vy = torch.clamp(eyy - myy, min=0.0)
    cxy = exy - mxy
    upper = 2 * cxy + C2
    lower = (vx + vy) + C2
    return ((2 * mxy + C1) * upper) / ((mxx + myy + C1) * lower)


def ssim_torchmetrics_form(x: torch.Tensor, y: torch.Tensor, tf32: bool = False) -> torch.Tensor:
    """x, y [B,C,H,W] fp32 in [0,1] -> per-image SSIM [B] (fp32)."""
    g = gaussian_1d(torch.float32)
    win = (g[:, None] @ g[None, :])[None, None]
    p = (K - 1) // 2
    xp = F.pad(x, (p, p, p, p), mode="reflect")
    yp = F.pad(y, (p, p, p, p), mode="reflect")
    m = _map(xp, yp, win, round_tf32 if tf32 else None)
    m = m[..., p:-p, p:-p]
    return m.reshape(m.shape[0], -1).mean(-1)


def ssim_valid_fp64(x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """The same per-image values as the mean over the windows wholly inside the image, in fp64."""
    g = gaussian_1d(torch.float64)
    win = (g[:, None] @ g[None, :])[None, None]
    m = _map(x.double(), y.double(), win)
    return m.reshape(m.shape[0], -1).mean(-1)
