"""LPIPS perceptual loss on the sm_90a kernels: value + gradient w.r.t. the reconstructed image.

Mirrors the reference's metric module vtp/utils/lpips.py:61-171 (ScalingLayer -> VGG16 features, 5 ReLU taps ->
channel unit-normalise -> squared difference -> 1x1 `lin` -> spatial mean -> sum).  The reference downloads the VGG16 /
lin weights at run time (lpips.py:15-17,48-58,130) which is impossible offline: weights are supplied by the caller
(the constructors' tensor lists, or `LPIPSMetric.from_files`) or drawn from a seeded generator (`random_init`, He-normal
convs, positive lin weights) — SURVEY.md §7.

`LPIPSLoss` is the bf16 training loss (value + gradient); `LPIPSMetric` is the fp32-accurate, forward-only evaluation
metric of the reconstruction evaluator (vtp_b200/recon_eval.py).

All 13 3x3 convolutions and their input-gradients run on the wgmma GEMM in implicit-conv mode (4-D TMA over NHWC
bf16 activations, zero fill = padding; bias+ReLU, respectively the ReLU mask, fused in the epilogue); conv1_1 (3 input
channels) goes through a 27->32 im2col.  Images are processed in chunks to bound activation memory.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch

from . import lib

BF, F32 = torch.bfloat16, torch.float32
VGG_CFG = [64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512]
TAPS = (1, 3, 6, 9, 12)  # conv indices whose ReLU output is a tap (relu1_2, 2_2, 3_3, 4_3, 5_3)


def check_shape(H: int, W: int) -> None:
    """Raise ValueError unless the VGG stack can run on H x W images: four 2x2 pools need H % 16 == 0, and the conv
    GEMM needs every feature map's width to be a multiple of 4, so W % 64 == 0."""
    if H % 16 or W % 64:
        raise ValueError(f"LPIPS: {H}x{W} images are not supported (needs H % 16 == 0 and W % 64 == 0)")


def _e(shape, dtype, dev):
    return torch.empty(shape, dtype=dtype, device=dev)


class LPIPSLoss:
    def __init__(self, vgg_w: Sequence[torch.Tensor], vgg_b: Sequence[torch.Tensor], lin_w: Sequence[torch.Tensor],
                 device="cuda", chunk: int = 32):
        """vgg_w[i]: [Cout, Cin, 3, 3], vgg_b[i]: [Cout], lin_w[k]: [1, C_k, 1, 1] (torch layouts, 13 convs, 5 lins)."""
        self.device, self.chunk = torch.device(device), chunk
        dev = self.device
        self.cin = [int(w.shape[1]) for w in vgg_w]
        self.cout = [int(w.shape[0]) for w in vgg_w]
        self.w_fwd, self.w_bwd, self.bias = [], [], []
        for i, (w, b) in enumerate(zip(vgg_w, vgg_b)):
            w = w.to(dev, F32)
            co, ci = w.shape[0], w.shape[1]
            if i == 0:  # [64, 27 -> 32], k = tap*3 + c
                wf = torch.zeros(co, 32, device=dev)
                wf[:, :27] = w.permute(0, 2, 3, 1).reshape(co, 27)
                self.w_fwd.append(wf.to(BF).contiguous())
                self.w_bwd.append(None)  # dgrad of conv1_1 is a plain NN GEMM on w_fwd
            else:
                self.w_fwd.append(w.permute(0, 2, 3, 1).reshape(co, 9 * ci).to(BF).contiguous())  # k = tap*Cin + c
                # dgrad = conv3x3 of dY with the 180-degree rotated kernel and in/out channels swapped
                wb = w.flip(2, 3).permute(1, 2, 3, 0).reshape(ci, 9 * co)                        # k = tap*Cout + co
                self.w_bwd.append(wb.to(BF).contiguous())
            self.bias.append(b.to(dev, BF).to(F32).contiguous())
        self.lin = [l.to(dev, F32).reshape(-1).contiguous() for l in lin_w]

    # ------------------------------------------------------------------ constructors
    @classmethod
    def random_init(cls, seed: int = 0, device="cuda", chunk: int = 32) -> "LPIPSLoss":
        vw, vb, lw = random_weights(seed)
        return cls(vw, vb, lw, device=device, chunk=chunk)

    # ------------------------------------------------------------------ VGG forward on one chunk
    def _features(self, img: torch.Tensor, keep_all: bool):
        """img NCHW (bf16|fp32) -> list of per-conv ReLU outputs NHWC bf16 (all of them if keep_all, else only taps)."""
        dev = self.device
        B, _, H, W = img.shape
        col = _e((B * H * W, 32), BF, dev)
        lib.lpips_prep(img.contiguous(), col, B, H, W)
        acts: List[Optional[torch.Tensor]] = []
        x, h, w, ci = None, H, W, 0
        pooled_in = {}
        for c in VGG_CFG:
            if c == "M":
                y = _e((B, h // 2, w // 2, x.shape[-1]), BF, dev)
                lib.maxpool2_fwd(x, y, B, h, w, x.shape[-1])
                x, h, w = y, h // 2, w // 2
                continue
            co = c
            y = _e((B, h, w, co), BF, dev)
            M = B * h * w
            if ci == 0:
                lib.gemm(col, self.w_fwd[0], y, M=M, N=co, K=32, bias=self.bias[0], act=lib.ACT_RELU, ldo=co)
            else:
                cin = self.cin[ci]
                lib.gemm(x, self.w_fwd[ci], y, M=M, N=co, K=9 * cin, lda=cin, ldb=9 * cin, bias=self.bias[ci],
                         act=lib.ACT_RELU, ldo=co, conv=(cin, h, w))
            acts.append(y if (keep_all or ci in TAPS) else None)
            x = y
            ci += 1
        return acts, col

    # ------------------------------------------------------------------ public
    @torch.no_grad()
    def loss_and_grad(self, rec: torch.Tensor, target: torch.Tensor, coef: float, loss_acc: torch.Tensor) -> torch.Tensor:
        """loss_acc[0] += coef * Σ_images LPIPS(rec_i, target_i);  returns d(that)/d(rec) as fp32 NCHW.
        (coef = weight / batch gives the batch-mean LPIPS term of the reconstruction loss.)"""
        dev = self.device
        B, _, H, W = rec.shape
        check_shape(H, W)
        dimg = _e((B, 3, H, W), F32, dev)
        for s in range(0, B, self.chunk):
            e = min(B, s + self.chunk)
            self._chunk(rec[s:e], target[s:e], coef, loss_acc, dimg[s:e])
        return dimg

    def _chunk(self, rec, tgt, coef, loss_acc, dimg):
        dev = self.device
        B, _, H, W = rec.shape
        a1, _ = self._features(tgt, keep_all=False)
        a0, _ = self._features(rec, keep_all=True)
        # spatial sizes per conv index
        sizes, h, w, ci = [], H, W, 0
        for c in VGG_CFG:
            if c == "M":
                h, w = h // 2, w // 2
            else:
                sizes.append((h, w))
                ci += 1
        # ---- taps: loss + gradient w.r.t. the reconstruction features
        gt = {}
        for k, ti in enumerate(TAPS):
            h, w = sizes[ti]
            C = self.cout[ti]
            g = _e((B, h, w, C), BF, dev)
            lib.lpips_tap(a0[ti], a1[ti], self.lin[k], g, B * h * w, C, coef / (h * w), loss_acc)
            gt[ti] = g
        del a1
        # ---- backward through the VGG stack (dgrad only: the VGG weights are frozen)
        n = len(self.cout)
        dz = gt[n - 1]  # relu5_3: tap gradient already masked by (y > 0)
        for i in range(n - 1, 0, -1):
            h, w = sizes[i]
            co, cin = self.cout[i], self.cin[i]
            hp, wp = sizes[i - 1]
            pooled = (hp, wp) != (h, w)
            dx = _e((B, h, w, cin), BF, dev)
            M = B * h * w
            # dX = conv(dz, rot180(W)^T); when the producer of X is a plain conv+ReLU, its mask (X > 0) is fused here
            lib.gemm(dz, self.w_bwd[i], dx, M=M, N=cin, K=9 * co, lda=co, ldb=9 * co, ldo=cin, conv=(co, h, w),
                     round_bf16=False, mask_pos=None if pooled else a0[i - 1])
            if pooled:
                dzp = _e((B, hp, wp, cin), BF, dev)
                lib.pool_relu_bwd(a0[i - 1], dx, gt.get(i - 1), dzp, B, hp, wp, cin)
                dz = dzp
            else:
                dz = dx
            a0[i] = None
        # conv1_1: d(col) = dz1_1 [M,64] · W1_1 [64,32]
        h, w = sizes[0]
        M = B * h * w
        dcol = _e((M, 32), BF, dev)
        lib.gemm(dz, self.w_fwd[0], dcol, M=M, N=32, K=64, lda=64, ldb=32, b_mn=True, ldo=32, round_bf16=False)
        lib.lpips_img_grad(dcol, dimg, B, h, w)


VGG_FEATURE_INDEX = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)  # torchvision vgg16.features index of each conv


class LPIPSMetric:
    """The reference's LPIPS module as an evaluation metric (tools/test_reconstruction_hf.py:379-388): per-image values,
    forward only, fp32-accurate.  The reference runs the VGG in fp32 (TF32 convolutions under cuDNN's default); here
    every conv is the implicit-conv wgmma GEMM on bf16x3 operands (activations [hi|hi|lo] over 3C channels, weights
    [hi|lo|hi] per tap, fp32 accumulation and output with bias + ReLU), max-pool runs in fp32, and only the five taps
    are kept.  Images are processed in chunks of `chunk` pairs to bound activation memory.  Shapes: see `check_shape`."""

    def __init__(self, vgg_w: Sequence[torch.Tensor], vgg_b: Sequence[torch.Tensor], lin_w: Sequence[torch.Tensor],
                 device="cuda", chunk: int = 8):
        """vgg_w[i]: [Cout, Cin, 3, 3], vgg_b[i]: [Cout], lin_w[k]: [1, C_k, 1, 1] (torch layouts, 13 convs, 5 lins)."""
        if len(vgg_w) != 13 or len(vgg_b) != 13 or len(lin_w) != 5:
            raise ValueError(f"LPIPSMetric: 13 conv weights / biases and 5 lin weights expected, got "
                             f"{len(vgg_w)} / {len(vgg_b)} / {len(lin_w)}")
        self.device, self.chunk = torch.device(device), int(chunk)
        dev = self.device
        self.cin = [int(w.shape[1]) for w in vgg_w]
        self.cout = [int(w.shape[0]) for w in vgg_w]
        self.w3, self.bias = [], []
        for i, (w, b) in enumerate(zip(vgg_w, vgg_b)):
            w = w.to(dev, F32)
            co, ci = w.shape[0], w.shape[1]
            if i == 0:  # [64, 27 -> 32] (k = tap*3 + c) -> [64, 96] = [hi|lo|hi]
                wf = torch.zeros(co, 32, device=dev)
                wf[:, :27] = w.permute(0, 2, 3, 1).reshape(co, 27)
                w3 = _e((co, 96), BF, dev)
                lib.split3(wf, w3, co, 32, b_side=True)
            else:  # [Cout, 9, Cin] -> [Cout, 9 * 3Cin]: per tap [hi|lo|hi] of Cin
                wt = w.permute(0, 2, 3, 1).reshape(co * 9, ci).contiguous()
                w3 = _e((co, 9 * 3 * ci), BF, dev)
                lib.split3(wt, w3, co * 9, ci, b_side=True)
            self.w3.append(w3)
            self.bias.append(b.to(dev, F32).contiguous())
        self.lin = [l.to(dev, F32).reshape(-1).contiguous() for l in lin_w]

    @classmethod
    def random_init(cls, seed: int = 0, device="cuda", chunk: int = 8) -> "LPIPSMetric":
        vw, vb, lw = random_weights(seed)
        return cls(vw, vb, lw, device=device, chunk=chunk)

    @classmethod
    def from_files(cls, vgg16_path: str, lin_path: str, device="cuda", chunk: int = 8) -> "LPIPSMetric":
        """torchvision's VGG16 checkpoint (keys features.{0,2,...,28}.{weight,bias}; the classifier is ignored) and the
        LPIPS lin file (keys lin{0..4}.model.1.weight; other keys are ignored, as the reference's strict=False load)."""
        return cls(*load_weight_files(vgg16_path, lin_path), device=device, chunk=chunk)

    check_shape = staticmethod(check_shape)

    def parts(self, lp: torch.Tensor) -> torch.Tensor:
        """lp fp32 [B, 2, 3, H, W] (the ScalingLayer outputs of each (reference, reconstruction) pair, as
        vtp_recon_pixels writes them) -> fp64 [B, 5 * slices] partials whose row sums are the per-image LPIPS values."""
        B, _, _, H, W = lp.shape
        self.check_shape(H, W)
        part = torch.empty((B, 5 * self.SLICES), dtype=torch.float64, device=lp.device)
        for s in range(0, B, self.chunk):
            e = min(B, s + self.chunk)
            self._chunk(lp[s:e].reshape(2 * (e - s), 3, H, W), part[s:e])
        return part

    SLICES = 32  # pixel slices per (pair, tap) in the partial sums: 32 CTAs per pair keep a chunk's taps spread over the SMs

    def _chunk(self, img: torch.Tensor, part: torch.Tensor) -> None:
        dev = img.device
        N, _, H, W = img.shape
        n = N // 2
        col = _e((N * H * W, 96), BF, dev)
        lib.lpips_prep3(img, col)
        x, h, w, ci, k = None, H, W, 0, 0
        for c in VGG_CFG:
            if c == "M":
                y = _e((N, h // 2, w // 2, x.shape[-1]), F32, dev)
                lib.maxpool2_f32(x, y, N, h, w, x.shape[-1])
                x, h, w = y, h // 2, w // 2
                continue
            y = _e((N, h, w, c), F32, dev)
            M = N * h * w
            if ci == 0:
                lib.gemm(col, self.w3[0], y, M=M, N=c, K=96, bias=self.bias[0], act=lib.ACT_RELU, ldo=c, round_bf16=False)
            else:
                cin = self.cin[ci]
                a3 = _e((M, 3 * cin), BF, dev)
                lib.split3(x.view(M, cin), a3, M, cin, b_side=False)
                lib.gemm(a3, self.w3[ci], y, M=M, N=c, K=27 * cin, lda=3 * cin, ldb=27 * cin, bias=self.bias[ci],
                         act=lib.ACT_RELU, ldo=c, conv=(3 * cin, h, w), round_bf16=False)
            if ci in TAPS:
                lib.lpips_tap_metric(y, self.lin[k], n, h * w, c, part, k * self.SLICES, self.SLICES)
                k += 1
            x = y
            ci += 1


def load_weight_files(vgg16_path: str, lin_path: str):
    """(vgg_w, vgg_b, lin_w) tensor lists from torchvision's VGG16 checkpoint and the LPIPS lin file (CPU tensors).
    Raises KeyError naming every missing key."""
    vgg, lin = _load_state(vgg16_path), _load_state(lin_path)
    need = [f"features.{j}.{p}" for j in VGG_FEATURE_INDEX for p in ("weight", "bias")]
    missing = [k for k in need if k not in vgg]
    if missing:
        raise KeyError(f"{vgg16_path}: missing VGG16 keys {missing}")
    lneed = [f"lin{k}.model.1.weight" for k in range(5)]
    missing = [k for k in lneed if k not in lin]
    if missing:
        raise KeyError(f"{lin_path}: missing LPIPS lin keys {missing}")
    return ([vgg[f"features.{j}.weight"] for j in VGG_FEATURE_INDEX], [vgg[f"features.{j}.bias"] for j in VGG_FEATURE_INDEX],
            [lin[k] for k in lneed])


def _load_state(path: str):
    if path.endswith(".safetensors"):
        from safetensors.torch import load_file

        return load_file(path)
    sd = torch.load(path, map_location="cpu", weights_only=True)
    if isinstance(sd, dict) and "state_dict" in sd and isinstance(sd["state_dict"], dict):
        sd = sd["state_dict"]
    return sd


def random_weights(seed: int = 0):
    """Deterministic stand-ins for the un-downloadable VGG16 / lin weights (same shapes; He-normal convs so that the
    activations keep unit scale through 13 ReLU layers; small positive lin weights like the trained LPIPS ones)."""
    g = torch.Generator().manual_seed(1000 + seed)
    vw, vb = [], []
    cin = 3
    for c in VGG_CFG:
        if c == "M":
            continue
        vw.append(torch.randn(c, cin, 3, 3, generator=g) * (2.0 / (9 * cin)) ** 0.5)
        vb.append(torch.randn(c, generator=g) * 0.05)
        cin = c
    lw = [torch.rand(1, c, 1, 1, generator=g) * (2.0 / c) for c in (64, 128, 256, 512, 512)]
    return vw, vb, lw
