"""Fréchet Inception Distance on the device: pytorch-fid's `calculate_fid_given_paths(paths, batch_size=50, dims=2048)`
(pytorch-fid 0.3.0), which the reference's reconstruction tool calls for rFID (tools/test_reconstruction_hf.py:98-104)
and its generation script for gFID.

pytorch-fid is not a dependency: this module restates its documented behaviour, and that restatement is not pinned
against the package (it is not installed where this project is tested).
  * images: a directory is read as its files `*.{bmp,jpg,jpeg,pgm,png,ppm,tif,tiff,webp}` (lower-case extensions, not
    recursive, sorted), each `Image.open(p).convert('RGB')`; a path ending in `.npz` holds precomputed `mu` / `sigma`.
  * network input: ToTensor (x / 255), `F.interpolate(x, (299, 299), mode='bilinear', align_corners=False)`, 2x - 1.
  * network: torchvision's Inception3 trunk with pytorch-fid's FID blocks (Mixed_5b-5d, 6b-6e and 7b average-pool with
    count_include_pad=False, Mixed_7c max-pools its pool branch), BasicConv2d = bias-free conv, BatchNorm (eps 0.001,
    eval mode), ReLU; 94 convolutions, stopped at the global average pool (2048 features).  Only dims = 2048.
  * statistics: mu = mean, sigma = np.cov(rowvar=False) (n - 1).  pytorch-fid's mu is fp32 (np.mean of fp32
    activations); here mu and sigma are fp64 throughout.  Saved `.npz` files keep pytorch-fid's keys and dtypes (mu fp32,
    sigma fp64).
  * distance: ||mu1 - mu2||² + tr σ1 + tr σ2 - 2 tr sqrtm(σ1 σ2) on the host in fp64 (`scipy.linalg.sqrtm` called with
    the matrix only: SciPy >= 1.18 has no `disp`), with pytorch-fid's eps retry and imaginary-part check.

On the device (csrc/fid.cu): `vtp_fid_resize` turns the uint8 images into the network input (bit-identical to torch's
CUDA resize); every conv is the wgmma GEMM on bf16x3 operands with fp32 output, the BatchNorm folded into its weights
and bias (in fp64, rounded once to fp32) and the ReLU in its epilogue; 1x1 convs read the activations through
`vtp_split3`, the others through `vtp_fid_im2col3`; each branch writes straight into its channel slice of the block's
concatenated output; `vtp_fid_pool` does the pools and `vtp_fid_moments` the spatial mean and the fp64 sums S1, S2, n.
A forward only enqueues work, so it can be captured in a CUDA graph.

The weights are pytorch-fid's `pt_inception-2015-12-05-6726825d.pth`, which the user supplies (nothing is downloaded);
`random_weights` gives seeded stand-ins in the same layout.

    python -m vtp_b200.fid DIR_OR_NPZ DIR_OR_NPZ --weights pt_inception-2015-12-05-6726825d.pth
"""
from __future__ import annotations

import argparse
import math
import os
import pathlib
from concurrent.futures import ThreadPoolExecutor
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import lib

F32, BF = torch.float32, torch.bfloat16
DIMS = 2048
BN_EPS = 1e-3
IMAGE_EXTENSIONS = ("bmp", "jpg", "jpeg", "pgm", "png", "ppm", "tif", "tiff", "webp")


# ---------------------------------------------------------------------------------------------------------- network
def _a(p, cin, pool):
    return {f"{p}.branch1x1": (cin, 64, 1, 1, 1, 0, 0), f"{p}.branch5x5_1": (cin, 48, 1, 1, 1, 0, 0),
            f"{p}.branch5x5_2": (48, 64, 5, 5, 1, 2, 2), f"{p}.branch3x3dbl_1": (cin, 64, 1, 1, 1, 0, 0),
            f"{p}.branch3x3dbl_2": (64, 96, 3, 3, 1, 1, 1), f"{p}.branch3x3dbl_3": (96, 96, 3, 3, 1, 1, 1),
            f"{p}.branch_pool": (cin, pool, 1, 1, 1, 0, 0)}


def _c(p, c7):
    return {f"{p}.branch1x1": (768, 192, 1, 1, 1, 0, 0), f"{p}.branch7x7_1": (768, c7, 1, 1, 1, 0, 0),
            f"{p}.branch7x7_2": (c7, c7, 1, 7, 1, 0, 3), f"{p}.branch7x7_3": (c7, 192, 7, 1, 1, 3, 0),
            f"{p}.branch7x7dbl_1": (768, c7, 1, 1, 1, 0, 0), f"{p}.branch7x7dbl_2": (c7, c7, 7, 1, 1, 3, 0),
            f"{p}.branch7x7dbl_3": (c7, c7, 1, 7, 1, 0, 3), f"{p}.branch7x7dbl_4": (c7, c7, 7, 1, 1, 3, 0),
            f"{p}.branch7x7dbl_5": (c7, 192, 1, 7, 1, 0, 3), f"{p}.branch_pool": (768, 192, 1, 1, 1, 0, 0)}


def _e(p, cin):
    return {f"{p}.branch1x1": (cin, 320, 1, 1, 1, 0, 0), f"{p}.branch3x3_1": (cin, 384, 1, 1, 1, 0, 0),
            f"{p}.branch3x3_2a": (384, 384, 1, 3, 1, 0, 1), f"{p}.branch3x3_2b": (384, 384, 3, 1, 1, 1, 0),
            f"{p}.branch3x3dbl_1": (cin, 448, 1, 1, 1, 0, 0), f"{p}.branch3x3dbl_2": (448, 384, 3, 3, 1, 1, 1),
            f"{p}.branch3x3dbl_3a": (384, 384, 1, 3, 1, 0, 1), f"{p}.branch3x3dbl_3b": (384, 384, 3, 1, 1, 1, 0),
            f"{p}.branch_pool": (cin, 192, 1, 1, 1, 0, 0)}


# name -> (Cin, Cout, kh, kw, stride, ph, pw) of the 94 BasicConv2d, in torchvision's naming and forward order
CONVS: Dict[str, Tuple[int, ...]] = {
    "Conv2d_1a_3x3": (3, 32, 3, 3, 2, 0, 0), "Conv2d_2a_3x3": (32, 32, 3, 3, 1, 0, 0),
    "Conv2d_2b_3x3": (32, 64, 3, 3, 1, 1, 1), "Conv2d_3b_1x1": (64, 80, 1, 1, 1, 0, 0),
    "Conv2d_4a_3x3": (80, 192, 3, 3, 1, 0, 0),
    **_a("Mixed_5b", 192, 32), **_a("Mixed_5c", 256, 64), **_a("Mixed_5d", 288, 64),
    "Mixed_6a.branch3x3": (288, 384, 3, 3, 2, 0, 0), "Mixed_6a.branch3x3dbl_1": (288, 64, 1, 1, 1, 0, 0),
    "Mixed_6a.branch3x3dbl_2": (64, 96, 3, 3, 1, 1, 1), "Mixed_6a.branch3x3dbl_3": (96, 96, 3, 3, 2, 0, 0),
    **_c("Mixed_6b", 128), **_c("Mixed_6c", 160), **_c("Mixed_6d", 160), **_c("Mixed_6e", 192),
    "Mixed_7a.branch3x3_1": (768, 192, 1, 1, 1, 0, 0), "Mixed_7a.branch3x3_2": (192, 320, 3, 3, 2, 0, 0),
    "Mixed_7a.branch7x7x3_1": (768, 192, 1, 1, 1, 0, 0), "Mixed_7a.branch7x7x3_2": (192, 192, 1, 7, 1, 0, 3),
    "Mixed_7a.branch7x7x3_3": (192, 192, 7, 1, 1, 3, 0), "Mixed_7a.branch7x7x3_4": (192, 192, 3, 3, 2, 0, 0),
    **_e("Mixed_7b", 1280), **_e("Mixed_7c", 2048),
}
assert len(CONVS) == 94


def required_keys() -> List[str]:
    return [f"{n}.{k}" for n in CONVS for k in ("conv.weight", "bn.weight", "bn.bias", "bn.running_mean", "bn.running_var")]


def fold_bn(sd: Dict[str, torch.Tensor], name: str) -> Tuple[torch.Tensor, torch.Tensor]:
    """conv + eval BatchNorm of one BasicConv2d as (weight, bias), folded in fp64 and rounded once to fp32 (CPU)."""
    w = sd[f"{name}.conv.weight"].double()
    g, b = sd[f"{name}.bn.weight"].double(), sd[f"{name}.bn.bias"].double()
    m, v = sd[f"{name}.bn.running_mean"].double(), sd[f"{name}.bn.running_var"].double()
    s = g / torch.sqrt(v + BN_EPS)
    return (w * s[:, None, None, None]).float(), (b - m * s).float()


def load_weight_file(path: str) -> Dict[str, torch.Tensor]:
    """pytorch-fid's FID Inception state dict (torchvision key names; fc.*, AuxLogits.* and num_batches_tracked are not
    used).  Raises KeyError naming every missing key."""
    from .lpips import _load_state

    sd = _load_state(path)
    missing = [k for k in required_keys() if k not in sd]
    if missing:
        raise KeyError(f"{path}: missing FID Inception keys {missing}")
    return {k: sd[k] for k in required_keys()}


def random_weights(seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded stand-ins for pytorch-fid's weights, in its layout.  Rule: each conv filter is drawn N(0, 1), made
    zero-mean over its fan-in and scaled to variance π/(π−1) · 2/fan_in, which keeps the variance of a zero-mean
    pre-activation unchanged through ReLU and the next conv; each BatchNorm gets running_var ~ U(0.5, 2), running_mean
    ~ N(0, 0.1²), weight = sqrt(running_var + eps) · U(0.9, 1.1) and bias = the shift that cancels running_mean plus
    N(0, 0.05²), so the folded conv is the filter times ~1 plus a small bias.  Activations stay O(1) through the 94
    convs (checked on the device by tests/test_fid_gpu.py, which also bounds the share of dead pool3 channels)."""
    g = torch.Generator().manual_seed(5000 + seed)
    sd = {}
    gain = math.pi / (math.pi - 1.0)
    for name, (ci, co, kh, kw, *_r) in CONVS.items():
        w = torch.randn(co, ci, kh, kw, generator=g, dtype=torch.float64)
        w = w - w.mean(dim=(1, 2, 3), keepdim=True)
        w = w / w.std(dim=(1, 2, 3), keepdim=True) * math.sqrt(gain * 2.0 / (ci * kh * kw))
        var = 0.5 + 1.5 * torch.rand(co, generator=g, dtype=torch.float64)
        mean = 0.1 * torch.randn(co, generator=g, dtype=torch.float64)
        gamma = torch.sqrt(var + BN_EPS) * (0.9 + 0.2 * torch.rand(co, generator=g, dtype=torch.float64))
        beta = gamma * mean / torch.sqrt(var + BN_EPS) + 0.05 * torch.randn(co, generator=g, dtype=torch.float64)
        sd[f"{name}.conv.weight"] = w.float()
        sd[f"{name}.bn.weight"], sd[f"{name}.bn.bias"] = gamma.float(), beta.float()
        sd[f"{name}.bn.running_mean"], sd[f"{name}.bn.running_var"] = mean.float(), var.float()
    return sd


class FIDStatistics:
    """Device accumulators of one image set: S2 (fp64 [D, D], upper triangle), S1 (fp64 [D]) and n, in one flat buffer
    so that ranks can sum them with a single all_reduce."""

    def __init__(self, device="cuda", dims: int = DIMS):
        D = self.dims = dims
        self.buf = torch.zeros(D * D + D + 1, dtype=torch.float64, device=device)
        self.S2 = self.buf[:D * D].view(D, D)
        self.S1 = self.buf[D * D:D * D + D]
        self.n = self.buf[D * D + D:]

    def reset(self) -> None:
        self.buf.zero_()

    def all_reduce(self, group=None) -> None:
        import torch.distributed as dist

        dist.all_reduce(self.buf, op=dist.ReduceOp.SUM, group=group)

    def count(self) -> int:
        return int(self.n.item())

    def mu_sigma(self) -> Tuple[np.ndarray, np.ndarray]:
        """(mu, sigma) in fp64 on the host: mu = S1 / n, sigma = (S2 - S1 S1ᵀ / n) / (n - 1)."""
        buf = self.buf.cpu().numpy()
        D = self.dims
        n = buf[-1]
        if n < 2:
            raise ValueError(f"FID statistics need at least 2 images, got {int(n)}")
        S2 = np.triu(buf[:D * D].reshape(D, D))
        S2 = S2 + np.triu(S2, 1).T
        S1 = buf[D * D:D * D + D]
        return S1 / n, (S2 - np.outer(S1, S1) / n) / (n - 1)

    def save_npz(self, path: str) -> None:
        mu, sigma = self.mu_sigma()
        save_stats_npz(path, mu, sigma)


def save_stats_npz(path: str, mu: np.ndarray, sigma: np.ndarray) -> None:
    """pytorch-fid's statistics file: keys mu (fp32) and sigma (fp64)."""
    np.savez_compressed(path, mu=np.asarray(mu, dtype=np.float32), sigma=np.asarray(sigma, dtype=np.float64))


class FIDInception:
    """pytorch-fid's FID Inception network on the sm_90a kernels (see the module docstring).  Images go through the
    network in chunks of `chunk` to bound the im2col workspace (the stem's 3x3 convs need ~37 MB of bf16x3 operand per
    image)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device="cuda", chunk: int = 16):
        self.device, self.chunk = torch.device(device), int(chunk)
        if self.device.type != "cuda":
            raise lib.VtpError("FIDInception runs on the CUDA device only")
        self.w3: Dict[str, torch.Tensor] = {}
        self.bias: Dict[str, torch.Tensor] = {}
        for name, (ci, co, kh, kw, *_r) in CONVS.items():
            w, b = fold_bn(state_dict, name)
            taps = kh * kw
            if ci == 3:  # stem: [Cout, 27 -> 32] (k = tap*3 + c) -> [Cout, 96]
                wf = torch.zeros(co, 32)
                wf[:, :27] = w.permute(0, 2, 3, 1).reshape(co, 27)
                rows, k = co, 32
            else:        # [Cout, taps, Cin] -> [Cout, taps * 3Cin]: per tap [hi|lo|hi] of Cin
                wf = w.permute(0, 2, 3, 1).reshape(co * taps, ci)
                rows, k = co * taps, ci
            wf = wf.to(self.device).contiguous()
            w3 = torch.empty((co, (96 if ci == 3 else taps * 3 * ci)), dtype=BF, device=self.device)
            lib.split3(wf, w3, rows, k, b_side=True)
            self.w3[name], self.bias[name] = w3, b.to(self.device).contiguous()
        self._scratch: Optional[FIDStatistics] = None
        self._rows0: Optional[torch.Tensor] = None

    @classmethod
    def from_file(cls, path: str, device="cuda", chunk: int = 16) -> "FIDInception":
        return cls(load_weight_file(path), device=device, chunk=chunk)

    @classmethod
    def random_init(cls, seed: int = 0, device="cuda", chunk: int = 16) -> "FIDInception":
        return cls(random_weights(seed), device=device, chunk=chunk)

    # ------------------------------------------------------------------ one conv into a channel slice
    def _conv(self, name: str, x: torch.Tensor, out: torch.Tensor, c0: int = 0) -> None:
        ci, co, kh, kw, s, ph, pw = CONVS[name]
        B, H, W, _ = x.shape
        Ho, Wo = lib.fid_conv_out(H, W, kh, kw, s, ph, pw)
        M, ldo = B * Ho * Wo, out.shape[-1]
        if kh == kw == 1 and s == 1:
            K = 3 * ci
            a3 = torch.empty((M, K), dtype=BF, device=x.device)
            lib.split3(x.view(M, ci), a3, M, ci, b_side=False)
        else:
            K = 96 if ci == 3 else kh * kw * 3 * ci
            a3 = torch.empty((M, K), dtype=BF, device=x.device)
            lib.fid_im2col3(x, a3, B, H, W, ci, (kh, kw), s, (ph, pw))
        lib.gemm(a3, self.w3[name], out.view(M, ldo)[:, c0:], M=M, N=co, K=K, lda=K, ldb=K, ldo=ldo,
                 bias=self.bias[name], act=lib.ACT_RELU, round_bf16=False)

    def _new(self, B, H, W, C):
        return torch.empty((B, H, W, C), dtype=F32, device=self.device)

    def _seq(self, names: Sequence[str], x: torch.Tensor, out: torch.Tensor, c0: int) -> None:
        """A chain of convs; the last writes channels c0.. of out."""
        for i, n in enumerate(names):
            if i == len(names) - 1:
                self._conv(n, x, out, c0)
            else:
                ci, co, kh, kw, s, ph, pw = CONVS[n]
                B, H, W, _ = x.shape
                y = self._new(B, *lib.fid_conv_out(H, W, kh, kw, s, ph, pw), co)
                self._conv(n, x, y)
                x = y

    def _pool_conv(self, name: str, x: torch.Tensor, out: torch.Tensor, c0: int, mode: int) -> None:
        B, H, W, C = x.shape
        p = self._new(B, H, W, C)
        lib.fid_pool(x, p, B, H, W, mode)
        self._conv(name, p, out, c0)

    def _block_a(self, p, x):
        B, H, W, _ = x.shape
        pool = CONVS[f"{p}.branch_pool"][1]
        out = self._new(B, H, W, 224 + pool)
        self._conv(f"{p}.branch1x1", x, out, 0)
        self._seq([f"{p}.branch5x5_1", f"{p}.branch5x5_2"], x, out, 64)
        self._seq([f"{p}.branch3x3dbl_{i}" for i in (1, 2, 3)], x, out, 128)
        self._pool_conv(f"{p}.branch_pool", x, out, 224, lib.FID_POOL_AVG1)
        return out

    def _block_c(self, p, x):
        B, H, W, _ = x.shape
        out = self._new(B, H, W, 768)
        self._conv(f"{p}.branch1x1", x, out, 0)
        self._seq([f"{p}.branch7x7_{i}" for i in (1, 2, 3)], x, out, 192)
        self._seq([f"{p}.branch7x7dbl_{i}" for i in (1, 2, 3, 4, 5)], x, out, 384)
        self._pool_conv(f"{p}.branch_pool", x, out, 576, lib.FID_POOL_AVG1)
        return out

    def _block_e(self, p, x, pool_mode, out=None):
        B, H, W, _ = x.shape
        out = self._new(B, H, W, 2048) if out is None else out
        self._conv(f"{p}.branch1x1", x, out, 0)
        t = self._new(B, H, W, 384)
        self._conv(f"{p}.branch3x3_1", x, t)
        self._conv(f"{p}.branch3x3_2a", t, out, 320)
        self._conv(f"{p}.branch3x3_2b", t, out, 704)
        t = self._new(B, H, W, 448)
        self._conv(f"{p}.branch3x3dbl_1", x, t)
        t2 = self._new(B, H, W, 384)
        self._conv(f"{p}.branch3x3dbl_2", t, t2)
        self._conv(f"{p}.branch3x3dbl_3a", t2, out, 1088)
        self._conv(f"{p}.branch3x3dbl_3b", t2, out, 1472)
        self._pool_conv(f"{p}.branch_pool", x, out, 1856, pool_mode)
        return out

    def _maxpool2(self, x, out=None, c0=0):
        B, H, W, C = x.shape
        if out is None:
            out = self._new(B, (H - 3) // 2 + 1, (W - 3) // 2 + 1, C)
        lib.fid_pool(x, out, B, H, W, lib.FID_POOL_MAX2, c0)
        return out

    def trunk(self, u8: torch.Tensor, out: torch.Tensor) -> None:
        """uint8 NHWC [B,H,W,3] -> out fp32 [B, 8, 8, 2048], the output of Mixed_7c."""
        B = u8.shape[0]
        x = self._new(B, lib.FID_SIZE, lib.FID_SIZE, 3)
        lib.fid_resize(u8, x)
        for n in ("Conv2d_1a_3x3", "Conv2d_2a_3x3", "Conv2d_2b_3x3"):
            ci, co, kh, kw, s, ph, pw = CONVS[n]
            y = self._new(B, *lib.fid_conv_out(x.shape[1], x.shape[2], kh, kw, s, ph, pw), co)
            self._conv(n, x, y)
            x = y
        x = self._maxpool2(x)
        for n in ("Conv2d_3b_1x1", "Conv2d_4a_3x3"):
            ci, co, kh, kw, s, ph, pw = CONVS[n]
            y = self._new(B, *lib.fid_conv_out(x.shape[1], x.shape[2], kh, kw, s, ph, pw), co)
            self._conv(n, x, y)
            x = y
        x = self._maxpool2(x)
        for p in ("Mixed_5b", "Mixed_5c", "Mixed_5d"):
            x = self._block_a(p, x)
        y = self._new(B, 17, 17, 768)                                    # Mixed_6a (InceptionB)
        self._conv("Mixed_6a.branch3x3", x, y, 0)
        self._seq([f"Mixed_6a.branch3x3dbl_{i}" for i in (1, 2, 3)], x, y, 384)
        self._maxpool2(x, y, 480)
        x = y
        for p in ("Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e"):
            x = self._block_c(p, x)
        y = self._new(B, 8, 8, 1280)                                     # Mixed_7a (InceptionD)
        self._seq(["Mixed_7a.branch3x3_1", "Mixed_7a.branch3x3_2"], x, y, 0)
        self._seq([f"Mixed_7a.branch7x7x3_{i}" for i in (1, 2, 3, 4)], x, y, 320)
        self._maxpool2(x, y, 512)
        x = self._block_e("Mixed_7b", y, lib.FID_POOL_AVG1)
        self._block_e("Mixed_7c", x, lib.FID_POOL_MAX1, out)

    # ------------------------------------------------------------------ public
    def _forward(self, u8: torch.Tensor, stats: FIDStatistics, rows: torch.Tensor, feat=None) -> None:
        if u8.dim() != 4 or u8.shape[-1] != 3 or u8.dtype != torch.uint8 or not u8.is_cuda:
            raise ValueError(f"FIDInception: uint8 NHWC [B,H,W,3] CUDA images expected, got {u8.dtype} {tuple(u8.shape)}")
        B = u8.shape[0]
        last = torch.empty((B, 8, 8, DIMS), dtype=F32, device=self.device)
        for s in range(0, B, self.chunk):
            e = min(B, s + self.chunk)
            self.trunk(u8[s:e], last[s:e])
        lib.fid_moments(last.view(B, 64, DIMS), rows, stats.S2, stats.S1, stats.n, feat=feat)

    @torch.no_grad()
    def accumulate(self, u8: torch.Tensor, stats: FIDStatistics, rows) -> None:
        """Add the first `rows` images of u8 (uint8 NHWC [B,H,W,3] on the device) to stats.  rows: an int, or a device
        int32 [1] tensor (read by the kernel, so a captured graph can vary it between replays).  Enqueues only."""
        if not isinstance(rows, torch.Tensor):
            rows = torch.full((1,), int(rows), dtype=torch.int32, device=self.device)
        self._forward(u8, stats, rows)

    @torch.no_grad()
    def features(self, u8: torch.Tensor) -> torch.Tensor:
        """fp32 [B, 2048] pool3 features of uint8 NHWC [B,H,W,3] device images."""
        if self._scratch is None:
            self._scratch = FIDStatistics(self.device)
            self._rows0 = torch.zeros(1, dtype=torch.int32, device=self.device)
        feat = torch.empty((u8.shape[0], DIMS), dtype=F32, device=self.device)
        self._forward(u8, self._scratch, self._rows0, feat=feat)
        return feat


# ---------------------------------------------------------------------------------------------------------- distance
def frechet_distance(mu1, sigma1, mu2, sigma2, eps: float = 1e-6) -> float:
    """d² = ||mu1 - mu2||² + tr σ1 + tr σ2 - 2 tr sqrtm(σ1 σ2), in fp64 on the host (pytorch-fid's
    calculate_frechet_distance, with sqrtm called on the matrix alone).  A non-finite square root is retried with eps·I
    added to both covariances; a complex one with a diagonal imaginary part above 1e-3 raises ValueError."""
    from scipy import linalg

    mu1, mu2 = np.atleast_1d(np.asarray(mu1, dtype=np.float64)), np.atleast_1d(np.asarray(mu2, dtype=np.float64))
    sigma1, sigma2 = np.atleast_2d(np.asarray(sigma1, dtype=np.float64)), np.atleast_2d(np.asarray(sigma2, dtype=np.float64))
    if mu1.shape != mu2.shape or sigma1.shape != sigma2.shape:
        raise ValueError("frechet_distance: mean vectors / covariances of different shapes")
    diff = mu1 - mu2
    covmean = linalg.sqrtm(sigma1.dot(sigma2))
    if not np.isfinite(covmean).all():
        print(f"fid calculation produces singular product; adding {eps} to diagonal of cov estimates")
        offset = np.eye(sigma1.shape[0]) * eps
        covmean = linalg.sqrtm((sigma1 + offset).dot(sigma2 + offset))
    if np.iscomplexobj(covmean):
        if not np.allclose(np.diagonal(covmean).imag, 0, atol=1e-3):
            raise ValueError(f"Imaginary component {np.max(np.abs(covmean.imag))}")
        covmean = covmean.real
    return float(diff.dot(diff) + np.trace(sigma1) + np.trace(sigma2) - 2 * np.trace(covmean))


# ---------------------------------------------------------------------------------------------------------- paths
def list_images(path: str) -> List[pathlib.Path]:
    """pytorch-fid's file list: `*.{ext}` for the lower-case extensions, not recursive, sorted."""
    p = pathlib.Path(path)
    return sorted(f for ext in IMAGE_EXTENSIONS for f in p.glob(f"*.{ext}"))


def _decode(f) -> np.ndarray:
    from PIL import Image

    with Image.open(f) as im:
        return np.asarray(im.convert("RGB"))


def statistics_of_path(path: str, model: FIDInception, batch_size: int = 50, num_workers: int = 4,
                       stats: Optional[FIDStatistics] = None) -> Tuple[np.ndarray, np.ndarray]:
    """(mu, sigma) of a directory of images, or those stored in an `.npz` file.  Images are decoded by a pool of
    `num_workers` threads into pinned uint8 batches; consecutive files of one size form a batch of up to batch_size (a
    size change starts a new one)."""
    if path.endswith(".npz"):
        with np.load(path) as f:
            return f["mu"][:], f["sigma"][:]
    files = list_images(path)
    if not files:
        raise ValueError(f"no images found in {path}")
    batch_size = max(1, min(batch_size, len(files)))
    stats = stats if stats is not None else FIDStatistics(model.device)
    stats.reset()
    dev = model.device
    with ThreadPoolExecutor(max_workers=max(1, num_workers)) as pool:
        pending: List[np.ndarray] = []

        def flush():
            if not pending:
                return
            host = torch.from_numpy(np.stack(pending)).pin_memory()
            model.accumulate(host.to(dev, non_blocking=True), stats, len(pending))
            pending.clear()

        for arr in pool.map(_decode, files):
            if pending and (arr.shape != pending[0].shape or len(pending) == batch_size):
                flush()
            pending.append(arr)
        flush()
    return stats.mu_sigma()


def _check_paths(paths: Sequence[str]) -> None:
    for p in paths:
        if not os.path.exists(p):
            raise RuntimeError(f"Invalid path: {p}")


def fid_from_paths(paths: Sequence[str], batch_size: int = 50, device="cuda", dims: int = DIMS, num_workers: int = 4,
                   weights: Optional[str] = None, model: Optional[FIDInception] = None) -> float:
    """pytorch-fid's calculate_fid_given_paths: the FID between two directories / `.npz` statistics files.  The network
    is `model`, or loaded from `weights`."""
    if dims != DIMS:
        raise NotImplementedError(f"dims = {dims}: only the 2048-dimensional pool3 features are supported")
    _check_paths(paths)
    if model is None:
        if weights is None:
            raise ValueError("fid_from_paths: give the FID Inception weights file (weights=) or a model")
        model = FIDInception.from_file(weights, device=device)
    m1, s1 = statistics_of_path(paths[0], model, batch_size, num_workers)
    m2, s2 = statistics_of_path(paths[1], model, batch_size, num_workers)
    return frechet_distance(m1, s1, m2, s2)


def save_fid_stats(paths: Sequence[str], batch_size: int = 50, device="cuda", dims: int = DIMS, num_workers: int = 4,
                   weights: Optional[str] = None, model: Optional[FIDInception] = None) -> None:
    """pytorch-fid's --save-stats: statistics of the directory paths[0] written to paths[1] (which must not exist)."""
    if dims != DIMS:
        raise NotImplementedError(f"dims = {dims}: only the 2048-dimensional pool3 features are supported")
    if not os.path.exists(paths[0]):
        raise RuntimeError(f"Invalid path: {paths[0]}")
    if os.path.exists(paths[1]):
        raise RuntimeError(f"Existing output file: {paths[1]}")
    if model is None:
        model = FIDInception.from_file(weights, device=device)
    m, s = statistics_of_path(paths[0], model, batch_size, num_workers)
    save_stats_npz(paths[1], m, s)


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(description="Fréchet Inception Distance (pytorch-fid's definition) on the H100 path")
    ap.add_argument("path", type=str, nargs=2, help="paths to the generated images or to .npz statistic files")
    ap.add_argument("--weights", type=str, required=True, help="pytorch-fid's pt_inception-2015-12-05-6726825d.pth")
    ap.add_argument("--batch-size", type=int, default=50, help="batch size to use")
    ap.add_argument("--num-workers", type=int, default=None, help="number of image decoding threads")
    ap.add_argument("--device", type=str, default="cuda", help="CUDA device to use")
    ap.add_argument("--dims", type=int, default=DIMS, help="dimensionality of the Inception features (2048 only)")
    ap.add_argument("--save-stats", action="store_true",
                    help="write the statistics of the first path (a directory) to the second (an .npz file)")
    return ap


def main(argv=None):
    args = build_parser().parse_args(argv)
    workers = args.num_workers if args.num_workers is not None else min(8, os.cpu_count() or 1)
    if args.save_stats:
        save_fid_stats(args.path, args.batch_size, args.device, args.dims, workers, weights=args.weights)
        return None
    value = fid_from_paths(args.path, args.batch_size, args.device, args.dims, workers, weights=args.weights)
    print("FID: ", value)
    return value


if __name__ == "__main__":
    main()
