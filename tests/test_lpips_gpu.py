"""GPU parity of the LPIPS loss + image gradient (wgmma implicit-conv VGG16) against the CPU oracle restatement of
vtp/utils/lpips.py with identical (seeded random) VGG/lin weights."""
import pytest
import torch

from oracle import vtp_oracle as vo
from tests.util import rel
from vtp_b200 import lib
from vtp_b200.lpips import LPIPSLoss, random_weights

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B,H", [(2, 64), (1, 128)])
def test_lpips_loss_and_grad(B, H):
    vw, vb, lw = random_weights(0)
    g = torch.Generator().manual_seed(3)
    rec = (torch.randn(B, 3, H, H, generator=g) * 0.5).to(torch.bfloat16)
    tgt = torch.randn(B, 3, H, H, generator=g) * 0.5
    r = rec.float().requires_grad_(True)
    val = vo.lpips(r, tgt, vw, vb, lw, mode="bf16")          # [B,1,1,1]
    loss = val.mean()
    loss.backward()
    mod = LPIPSLoss(vw, vb, lw, device="cuda", chunk=1)
    acc = torch.zeros(1, device="cuda")
    dimg = mod.loss_and_grad(rec.cuda(), tgt.cuda(), 1.0 / B, acc)
    torch.cuda.synchronize()
    assert torch.isfinite(dimg).all()
    assert abs(acc.item() - loss.item()) < 3e-2 * abs(loss.item()), (acc.item(), loss.item())
    e = rel(dimg, r.grad)
    assert e < 8e-2, e


def test_conv_mode_gemm_matches_conv2d():
    B, H, W, Ci, Co = 2, 16, 16, 64, 128
    x = (torch.randn(B, H, W, Ci, device="cuda") * 0.5).to(torch.bfloat16)
    w = (torch.randn(Co, Ci, 3, 3, device="cuda") * 0.05).to(torch.bfloat16)
    b = torch.randn(Co, device="cuda") * 0.1
    wk = w.permute(0, 2, 3, 1).reshape(Co, 9 * Ci).contiguous()
    y = torch.empty(B, H, W, Co, device="cuda", dtype=torch.bfloat16)
    lib.gemm(x, wk, y, M=B * H * W, N=Co, K=9 * Ci, lda=Ci, ldb=9 * Ci, bias=b, act=lib.ACT_RELU, ldo=Co, conv=(Ci, H, W))
    ref = torch.relu(torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w.float(), b, padding=1)).permute(0, 2, 3, 1)
    assert rel(y, ref) < 5e-3
    # small feature map (W = 4 -> 4x32 tiles, mostly out of bounds) and the ReLU-mask epilogue
    x2 = (torch.randn(3, 4, 4, 64, device="cuda")).to(torch.bfloat16)
    m2 = torch.randn(3, 4, 4, 128, device="cuda").to(torch.bfloat16)
    y2 = torch.empty(3, 4, 4, Co, device="cuda", dtype=torch.bfloat16)
    lib.gemm(x2, wk, y2, M=48, N=Co, K=9 * Ci, lda=Ci, ldb=9 * Ci, ldo=Co, conv=(Ci, 4, 4), round_bf16=False, mask_pos=m2)
    ref2 = torch.nn.functional.conv2d(x2.float().permute(0, 3, 1, 2), w.float(), None, padding=1).permute(0, 2, 3, 1)
    ref2 = ref2 * (m2.float() > 0)
    assert rel(y2, ref2) < 5e-3


@pytest.mark.parametrize("variant", ["default", "VTP_GEMM_CONV_NO_FAST", "VTP_GEMM_CONV_NO_CLUSTER", "VTP_GEMM_CONV_BRES=0",
                                     "VTP_GEMM_CONV_BRES=1", "VTP_GEMM_CONV_BRES=2", "VTP_GEMM_CONV_HALO=0",
                                     "VTP_GEMM_CONV_HALO=1", "ldo_pad", "ldo_pad_no_fast", "no_relu"])
@pytest.mark.parametrize("B,H,W,Ci,Co,mask", [(1, 24, 16, 64, 64, False), (3, 8, 8, 128, 256, True), (2, 32, 32, 64, 64, True),
                                              (5, 16, 16, 256, 512, False), (1, 8, 8, 512, 512, True),
                                              (3, 40, 24, 64, 64, False), (2, 20, 12, 64, 64, True), (3, 256, 256, 64, 64, False),
                                              (3, 256, 256, 64, 64, True), (2, 32, 32, 64, 128, False), (2, 32, 32, 128, 64, True),
                                              (3, 40, 24, 128, 128, True), (2, 128, 128, 128, 128, False), (1, 24, 16, 256, 128, True),
                                              (2, 128, 128, 128, 64, True), (1, 16, 16, 128, 64, False)])
def test_conv_mode_variants(monkeypatch, variant, B, H, W, Ci, Co, mask):
    """Implicit 3x3 conv GEMM (4-D TMA over NHWC, zero fill = padding) through the TMA-store epilogue (4-D NHWC tensor map)
    and the generic one (VTP_GEMM_CONV_NO_FAST): 64- and 128-wide tiles, 16 / 8 / 4-pixel tile rows, ragged heights, Cout <
    tile width, many tiles per persistent CTA, bias+ReLU forward form, bias-only form and masked dgrad form, and an output
    whose pixel stride is wider than Cout (ldo_pad: the result lands in a channel slice of a wider NHWC buffer).  The
    CONV_NO_CLUSTER / CONV_BRES / CONV_HALO ids named pre-Hopper conv forms; the library no longer reads them and those ids
    run the default kernel."""
    if variant in ("VTP_GEMM_CONV_NO_FAST", "ldo_pad_no_fast"):
        monkeypatch.setenv("VTP_GEMM_CONV_NO_FAST", "1")
    ldo = Co + 64 if variant.startswith("ldo_pad") else Co
    g = torch.Generator(device="cuda").manual_seed(B * 100 + Ci)
    x = (torch.randn(B, H, W, Ci, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    w = (torch.randn(Co, Ci, 3, 3, device="cuda", generator=g) * (2.0 / (9 * Ci)) ** 0.5).to(torch.bfloat16)
    wk = w.permute(0, 2, 3, 1).reshape(Co, 9 * Ci).contiguous()
    ybuf = torch.full((B, H, W, ldo), float("nan"), device="cuda", dtype=torch.bfloat16)
    y = ybuf[..., :Co]
    conv = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w.float(), None, padding=1).permute(0, 2, 3, 1)
    if mask:
        m = torch.randn(B, H, W, Co, device="cuda", generator=g).to(torch.bfloat16)
        lib.gemm(x, wk, ybuf, M=B * H * W, N=Co, K=9 * Ci, lda=Ci, ldb=9 * Ci, ldo=ldo, conv=(Ci, H, W), round_bf16=False,
                 mask_pos=m)
        ref = conv * (m.float() > 0)
    else:
        b = torch.randn(Co, device="cuda", generator=g) * 0.1
        relu = variant != "no_relu"
        lib.gemm(x, wk, ybuf, M=B * H * W, N=Co, K=9 * Ci, lda=Ci, ldb=9 * Ci, bias=b, act=lib.ACT_RELU if relu else lib.ACT_NONE,
                 ldo=ldo, conv=(Ci, H, W))
        ref = torch.relu(conv + b) if relu else conv + b
    torch.cuda.synchronize()
    assert torch.isfinite(y.float()).all()
    assert rel(y, ref) < 5e-3, rel(y, ref)
