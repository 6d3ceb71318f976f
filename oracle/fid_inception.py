"""Reference network of the FID tests: pytorch-fid's FID Inception (fid_score / inception.py of pytorch-fid 0.3.0,
restated from its documented behaviour) on torchvision's Inception3.

torchvision's `Inception3(num_classes=1008, aux_logits=False, init_weights=False, transform_input=False)` with
pytorch-fid's four FID blocks substituted: InceptionA / InceptionC / InceptionE_1 average-pool their pool branch with
count_include_pad=False, InceptionE_2 (Mixed_7c) max-pools it (3x3, stride 1, pad 1).  The input stage is
F.interpolate(x, (299, 299), bilinear, align_corners=False) then 2x - 1 on ToTensor images in [0, 1]; the output is the
global average pool (2048 features).  Runs in any dtype on CPU or GPU; `round_ops` (e.g. a TF32 rounding) is applied to
both operands of every convolution, which models cuDNN's default TF32 convolutions.
"""
from __future__ import annotations

import types

import torch
import torch.nn.functional as F
from torchvision.models.inception import BasicConv2d, Inception3, InceptionA, InceptionC, InceptionE


class FIDInceptionA(InceptionA):
    def forward(self, x):
        b1 = self.branch1x1(x)
        b5 = self.branch5x5_2(self.branch5x5_1(x))
        b3 = self.branch3x3dbl_3(self.branch3x3dbl_2(self.branch3x3dbl_1(x)))
        bp = self.branch_pool(F.avg_pool2d(x, kernel_size=3, stride=1, padding=1, count_include_pad=False))
        return torch.cat([b1, b5, b3, bp], 1)


class FIDInceptionC(InceptionC):
    def forward(self, x):
        b1 = self.branch1x1(x)
        b7 = self.branch7x7_3(self.branch7x7_2(self.branch7x7_1(x)))
        bd = self.branch7x7dbl_1(x)
        for m in (self.branch7x7dbl_2, self.branch7x7dbl_3, self.branch7x7dbl_4, self.branch7x7dbl_5):
            bd = m(bd)
        bp = self.branch_pool(F.avg_pool2d(x, kernel_size=3, stride=1, padding=1, count_include_pad=False))
        return torch.cat([b1, b7, bd, bp], 1)


class _FIDInceptionE(InceptionE):
    def _pool(self, x):
        raise NotImplementedError

    def forward(self, x):
        b1 = self.branch1x1(x)
        b3 = self.branch3x3_1(x)
        b3 = torch.cat([self.branch3x3_2a(b3), self.branch3x3_2b(b3)], 1)
        bd = self.branch3x3dbl_2(self.branch3x3dbl_1(x))
        bd = torch.cat([self.branch3x3dbl_3a(bd), self.branch3x3dbl_3b(bd)], 1)
        bp = self.branch_pool(self._pool(x))
        return torch.cat([b1, b3, bd, bp], 1)


class FIDInceptionE_1(_FIDInceptionE):
    def _pool(self, x):
        return F.avg_pool2d(x, kernel_size=3, stride=1, padding=1, count_include_pad=False)


class FIDInceptionE_2(_FIDInceptionE):
    def _pool(self, x):
        return F.max_pool2d(x, kernel_size=3, stride=1, padding=1)


def fid_inception(state_dict=None, dtype=torch.float64, device="cpu") -> Inception3:
    """The FID network in eval mode (fc / AuxLogits unused), loaded from a torchvision-layout state dict if given."""
    net = Inception3(num_classes=1008, aux_logits=False, init_weights=False, transform_input=False)
    net.Mixed_5b = FIDInceptionA(192, pool_features=32)
    net.Mixed_5c = FIDInceptionA(256, pool_features=64)
    net.Mixed_5d = FIDInceptionA(288, pool_features=64)
    net.Mixed_6b = FIDInceptionC(768, channels_7x7=128)
    net.Mixed_6c = FIDInceptionC(768, channels_7x7=160)
    net.Mixed_6d = FIDInceptionC(768, channels_7x7=160)
    net.Mixed_6e = FIDInceptionC(768, channels_7x7=192)
    net.Mixed_7b = FIDInceptionE_1(1280)
    net.Mixed_7c = FIDInceptionE_2(2048)
    if state_dict is not None:
        net.load_state_dict(state_dict, strict=False)
    return net.to(device=device, dtype=dtype).eval()


def set_operand_rounding(net: Inception3, round_ops) -> None:
    """Apply round_ops to the input and the weight of every convolution (BatchNorm and ReLU stay in net's dtype)."""
    def fwd(self, x):
        w = self.conv.weight
        return F.relu(self.bn(F.conv2d(round_ops(x), round_ops(w).to(x.dtype), None, self.conv.stride, self.conv.padding)))

    for m in net.modules():
        if isinstance(m, BasicConv2d):
            m.forward = types.MethodType(fwd, m)


def network_input(img01: torch.Tensor) -> torch.Tensor:
    """pytorch-fid's input stage on ToTensor images [B,3,H,W] in [0, 1]."""
    x = F.interpolate(img01, size=(299, 299), mode="bilinear", align_corners=False)
    return 2 * x - 1


def trunk(net: Inception3, x: torch.Tensor) -> torch.Tensor:
    """Network input [B,3,299,299] -> Mixed_7c output [B,2048,8,8]."""
    for n in ("Conv2d_1a_3x3", "Conv2d_2a_3x3", "Conv2d_2b_3x3", "maxpool1", "Conv2d_3b_1x1", "Conv2d_4a_3x3", "maxpool2",
              "Mixed_5b", "Mixed_5c", "Mixed_5d", "Mixed_6a", "Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e", "Mixed_7a",
              "Mixed_7b", "Mixed_7c"):
        x = getattr(net, n)(x)
    return x


@torch.no_grad()
def features(net: Inception3, img01: torch.Tensor, dtype=None) -> torch.Tensor:
    """[B, 2048] pool3 features of ToTensor images, the network input formed in fp32 (as pytorch-fid) and the network run
    in net's dtype."""
    dtype = dtype or next(net.parameters()).dtype
    x = network_input(img01.float()).to(dtype)
    return trunk(net, x).mean(dim=(2, 3))
