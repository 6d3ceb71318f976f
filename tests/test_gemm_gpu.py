"""GPU parity of the wgmma GEMM (vtp_gemm_bf16) against a plain fp32 PyTorch reference of the same op."""
import math

import pytest
import torch

from vtp_b200 import lib

pytestmark = pytest.mark.gpu


def _mk(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, device="cuda", generator=g) * scale).to(torch.bfloat16)


def _ref(A, B, a_mn, b_mn):
    torch.backends.cuda.matmul.allow_tf32 = False
    Af = A.float().t() if a_mn else A.float()
    Bf = B.float().t() if b_mn else B.float()
    return Af @ Bf.t()


def _relerr(x, y):
    return ((x.float() - y.float()).norm() / (y.float().norm() + 1e-30)).item()


@pytest.mark.parametrize("a_mn", [False, True])
@pytest.mark.parametrize("b_mn", [False, True])
@pytest.mark.parametrize("M,N,K", [(300, 384, 384), (1000, 512, 200), (128, 64, 64), (777, 1152, 384), (513, 5472, 1024)])
def test_gemm_majors(a_mn, b_mn, M, N, K):
    r8 = lambda v: (v + 7) // 8 * 8
    A = _mk((K, r8(M)), 1)[:, :M] if a_mn else _mk((M, r8(K)), 1)[:, :K]
    B = _mk((K, r8(N)), 2)[:, :N] if b_mn else _mk((N, r8(K)), 2)[:, :K]
    out = torch.full((M, N), float("nan"), device="cuda", dtype=torch.float32)
    lib.gemm(A, B, out, M=M, N=N, K=K, a_mn=a_mn, b_mn=b_mn, round_bf16=False)
    torch.cuda.synchronize()
    ref = _ref(A, B, a_mn, b_mn)
    assert torch.isfinite(out).all()
    assert _relerr(out, ref) < 2e-5, _relerr(out, ref)


def test_gemm_bias_bf16_out_large():
    M, N, K = 65792, 1152, 384
    A, B = _mk((M, K), 3), _mk((N, K), 4, 0.05)
    bias = torch.randn(N, device="cuda")
    out = torch.empty((M, N), device="cuda", dtype=torch.bfloat16)
    lib.gemm(A, B, out, M=M, N=N, K=K, bias=bias)
    torch.cuda.synchronize()
    ref = (_ref(A, B, False, False) + bias).to(torch.bfloat16)
    assert (out.float() - ref.float()).abs().max().item() <= 2 * 2**-8 * ref.float().abs().max().item()
    assert _relerr(out, ref) < 1e-3


def test_gemm_residual_rowremap_inplace():
    B_, G, D, K = 3, 256, 384, 768
    M = B_ * G
    A, W = _mk((M, K), 5), _mk((D, K), 6, 0.05)
    bias = torch.randn(D, device="cuda")
    x = torch.randn(B_ * (G + 1), D, device="cuda")
    x0 = x.clone()
    lib.gemm(A, W, x, M=M, N=D, K=K, bias=bias, resid=x, rr_group=G, rr_skip=1)
    torch.cuda.synchronize()
    lin = (_ref(A, W, False, False) + bias).to(torch.bfloat16).float().view(B_, G, D)
    exp = x0.view(B_, G + 1, D).clone()
    exp[:, 1:] += lin
    assert torch.equal(x.view(B_, G + 1, D)[:, 0], x0.view(B_, G + 1, D)[:, 0])
    assert _relerr(x.view(B_, G + 1, D), exp) < 1e-3


@pytest.mark.parametrize("M,N,K,split", [(384, 1152, 8200, 16), (384, 1152, 8200, -1), (2048, 384, 20000, -1),
                                         (384, 384, 20000, -1), (1152, 384, 9000, 5), (256, 64, 4100, -1)])
def test_gemm_splitk_accumulate(M, N, K, split):
    """wgrad form: TN GEMM, split-K + fp32 red.add into a pre-filled output; split = -1 lets the library choose
    (192-wide tiles when N % 192 == 0)."""
    A, B = _mk((K, M), 7), _mk((K, N), 8)
    out = torch.ones((M, N), device="cuda")
    lib.gemm(A, B, out, M=M, N=N, K=K, a_mn=True, b_mn=True, accumulate=True, split_k=split, round_bf16=False)
    torch.cuda.synchronize()
    ref = _ref(A, B, True, True) + 1.0
    assert _relerr(out, ref) < 2e-5


def test_gemm_gelu_and_out2():
    M, N, K = 500, 1536, 384
    A, B = _mk((M, K), 9), _mk((N, K), 10, 0.05)
    bias = torch.randn(N, device="cuda") * 0.1
    out = torch.empty((M, N), device="cuda", dtype=torch.bfloat16)
    pre = torch.empty((M, N), device="cuda", dtype=torch.bfloat16)
    lib.gemm(A, B, out, M=M, N=N, K=K, bias=bias, act=lib.ACT_GELU, out2=pre)
    torch.cuda.synchronize()
    ref_pre = (_ref(A, B, False, False) + bias).to(torch.bfloat16)
    ref = torch.nn.functional.gelu(ref_pre.float()).to(torch.bfloat16)
    assert _relerr(pre, ref_pre) < 1e-3
    assert _relerr(out, ref) < 2e-3


def test_gemm_swiglu8():
    M, Hs, K = 300, 1024, 384
    A = _mk((M, K), 11)
    W1, W2 = _mk((Hs, K), 12, 0.05), _mk((Hs, K), 13, 0.05)
    b1, b2 = torch.randn(Hs, device="cuda") * 0.1, torch.randn(Hs, device="cuda") * 0.1
    # 8-interleave: packed rows [16g,16g+8) = w1[8g:8g+8], [16g+8,16g+16) = w2[8g:8g+8]
    Wp = torch.stack([W1.view(Hs // 8, 8, K), W2.view(Hs // 8, 8, K)], dim=1).reshape(2 * Hs, K).contiguous()
    bp = torch.stack([b1.view(-1, 8), b2.view(-1, 8)], dim=1).reshape(-1).contiguous()
    out = torch.empty((M, Hs), device="cuda", dtype=torch.bfloat16)
    lib.gemm(A, Wp, out, M=M, N=2 * Hs, K=K, bias=bp, act=lib.ACT_SWIGLU8, ldo=Hs)
    torch.cuda.synchronize()
    x1 = (A.float() @ W1.float().t() + b1).to(torch.bfloat16)
    x2 = (A.float() @ W2.float().t() + b2).to(torch.bfloat16)
    ref = (torch.nn.functional.silu(x1.float()).to(torch.bfloat16).float() * x2.float()).to(torch.bfloat16)
    assert _relerr(out, ref) < 3e-3


def test_gemm_rope_epilogue():
    Bn, Ntok, prefix, D, K = 2, 257, 1, 384, 384
    H = D // 64
    M = Bn * Ntok
    A, W = _mk((M, K), 14), _mk((3 * D, K), 15, 0.05)
    bias = torch.randn(3 * D, device="cuda") * 0.1
    HW = Ntok - prefix
    ang = torch.rand(HW, 64, device="cuda") * 6.28
    sin, cos = torch.sin(ang).to(torch.bfloat16), torch.cos(ang).to(torch.bfloat16)
    out = torch.empty((M, 3 * D), device="cuda", dtype=torch.bfloat16)
    lib.gemm(A, W, out, M=M, N=3 * D, K=K, bias=bias, act=lib.ACT_ROPE, rope=(sin, cos, Ntok, prefix, 2 * D))
    torch.cuda.synchronize()
    qkv = (_ref(A, W, False, False) + bias).to(torch.bfloat16).view(Bn, Ntok, 3, H, 64)

    def rot(x):  # layers/attention.py:12-23 in bf16
        x1, x2 = x.chunk(2, dim=-1)
        return torch.cat([-x2, x1], dim=-1)

    ref = qkv.clone()
    for i in (0, 1):
        x = qkv[:, prefix:, i]  # [B, HW, H, 64]
        ref[:, prefix:, i] = (x * cos[None, :, None, :]) + (rot(x) * sin[None, :, None, :])
    got = out.view(Bn, Ntok, 3, H, 64)
    assert torch.equal(got[:, :prefix], ref[:, :prefix]) or _relerr(got[:, :prefix], ref[:, :prefix]) < 1e-3
    assert _relerr(got[:, :, 2], ref[:, :, 2]) < 1e-3
    assert _relerr(got[:, :, :2], ref[:, :, :2]) < 3e-3


def test_gemm_pixel_shuffle():
    Bn, g, r, D = 2, 16, 16, 384
    M, N = Bn * g * g, 3 * r * r
    A, W = _mk((M, D), 16), _mk((N, D), 17, 0.05)
    bias = torch.randn(N, device="cuda") * 0.1
    out = torch.empty((Bn, 3, g * r, g * r), device="cuda")
    lib.gemm(A, W, out, M=M, N=N, K=D, bias=bias, pixel_shuffle=(r, g, g, 3), ldo=g * r, round_bf16=False)
    torch.cuda.synchronize()
    y = (_ref(A, W, False, False) + bias).view(Bn, g, g, N).permute(0, 3, 1, 2)
    ref = torch.nn.functional.pixel_shuffle(y, r)
    assert _relerr(out, ref) < 2e-5


@pytest.mark.parametrize("variant", ["default", "VTP_GEMM_G2", "VTP_GEMM_NO_FAST", "VTP_GEMM_NO_CLUSTER", "a_mn", "b_mn"])
@pytest.mark.parametrize("out_f32,resid,relu", [(False, False, False), (False, True, False), (True, False, False),
                                                (True, True, False), (False, False, True)])
@pytest.mark.parametrize("M,N,K", [(1000, 384, 384), (777, 1160, 200), (260, 2048, 1024), (129, 72, 64)])
def test_gemm_fast_epilogue_modes(monkeypatch, variant, out_f32, resid, relu, M, N, K):
    """The lean TMA-store epilogue (bias, rounding point, optional same-dtype residual, ReLU) incl. M / N tails, in place
    and out of place, on the lean and the generic epilogue (VTP_GEMM_NO_FAST), and with an MN-major A or B operand
    (64- and 128-wide tiles: N = 72 runs on 128, N <= 64 elsewhere).  VTP_GEMM_G2 / VTP_GEMM_NO_CLUSTER named the
    pre-Hopper pair-tile and single-CTA forms; the library no longer reads them and those ids run the default kernel."""
    if variant == "VTP_GEMM_NO_FAST":
        monkeypatch.setenv(variant, "1")
    r8 = lambda v: (v + 7) // 8 * 8
    A, W = _mk((M, r8(K)), 11)[:, :K], _mk((N, r8(K)), 12, 0.1)[:, :K]
    opA, opW, kw = A, W, {}
    if variant == "a_mn":   # A stored [K][M] (padded rows of 8)
        opA = torch.zeros(K, r8(M), device="cuda", dtype=torch.bfloat16)
        opA[:, :M] = A.t()
        kw = dict(a_mn=True, lda=r8(M))
    elif variant == "b_mn":
        opW = torch.zeros(K, r8(N), device="cuda", dtype=torch.bfloat16)
        opW[:, :N] = W.t()
        kw = dict(b_mn=True, ldb=r8(N))
    bias = torch.randn(N, device="cuda")
    dt = torch.float32 if out_f32 else torch.bfloat16
    x = torch.randn(M, N, device="cuda").to(dt)
    acc = (_ref(A, W, False, False) + bias).to(torch.bfloat16).float()  # bf16 rounding point of the linear (autocast)
    if relu:
        acc = acc.clamp_min(0)
    ref = (acc + x.float()).to(dt) if resid else acc.to(dt)
    for inplace in ([False, True] if resid else [False]):
        xin = x.clone()
        out = xin if inplace else torch.full((M, N), float("nan"), device="cuda", dtype=dt)
        lib.gemm(opA, opW, out, M=M, N=N, K=K, bias=bias, resid=xin if resid else None,
                 act=lib.ACT_RELU if relu else lib.ACT_NONE, **kw)
        torch.cuda.synchronize()
        assert torch.isfinite(out.float()).all()
        # one bf16 ulp of slack where the fp32 accumulation order flips the rounding point
        assert (out.float() - ref.float()).abs().max().item() <= 2.0 ** -7 * ref.float().abs().max().item() + 1e-6
        assert _relerr(out, ref) < 2e-3


@pytest.mark.parametrize("variant", ["default", "VTP_GEMM_NO_N64_BRES", "VTP_GEMM_NO_FAST"])
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("M,K", [(40000, 32), (38000, 96), (50001, 576), (131072, 32)])
def test_gemm_n64_resident_weights(monkeypatch, variant, relu, M, K):
    """Tall 64-column GEMMs with K <= 576 (the VGG conv1_1 im2col form) on 64-wide tiles, lean and generic epilogue: K shorter
    than a k-block (zero fill), ragged last tile, many tiles per persistent CTA.  VTP_GEMM_NO_N64_BRES named the pre-Hopper
    resident-weight form; the library no longer reads it and that id runs the default kernel."""
    if variant == "VTP_GEMM_NO_FAST":
        monkeypatch.setenv(variant, "1")
    A, W = _mk((M, K), 21, 0.5), _mk((64, K), 22, 0.1)
    bias = torch.randn(64, device="cuda")
    out = torch.full((M, 64), float("nan"), device="cuda", dtype=torch.bfloat16)
    lib.gemm(A, W, out, M=M, N=64, K=K, bias=bias, act=lib.ACT_RELU if relu else lib.ACT_NONE)
    torch.cuda.synchronize()
    ref = (_ref(A, W, False, False) + bias).to(torch.bfloat16).float()
    if relu:
        ref = ref.clamp_min(0)
    assert torch.isfinite(out.float()).all()
    assert (out.float() - ref).abs().max().item() <= 2.0 ** -7 * ref.abs().max().item() + 1e-6
    assert _relerr(out, ref) < 2e-3


@pytest.mark.parametrize("M,Hs,K,with_pre", [(300, 1024, 384, True), (300, 1024, 384, False), (4100, 2736, 1024, True),
                                             (1000, 344, 128, True), (129, 64, 64, True), (2048, 2048, 768, False),
                                             (515, 1368, 384, True)])
def test_gemm_swiglu_fast_epilogue(monkeypatch, M, Hs, K, with_pre):
    """SwiGLU gate in the lean TMA-store epilogue (fast_swiglu_tile, FAST 6 / 7): hidden = round(round(silu(x1)) * x2) and the
    bf16 pre-activation, vs torch and vs the generic epilogue (VTP_GEMM_NO_FAST_SWIGLU=1) — bit-identical to the latter.
    Shapes: 256- and 128-wide tiles, ragged N (2 * 2736 = 21.375 tiles; 2 * 344; 2 * 1368), M tails, one-tile problems."""
    A = _mk((M, K), 41)
    W1, W2 = _mk((Hs, K), 42, 0.05), _mk((Hs, K), 43, 0.05)
    b1, b2 = torch.randn(Hs, device="cuda") * 0.1, torch.randn(Hs, device="cuda") * 0.1
    Wp = torch.stack([W1.view(Hs // 8, 8, K), W2.view(Hs // 8, 8, K)], dim=1).reshape(2 * Hs, K).contiguous()
    bp = torch.stack([b1.view(-1, 8), b2.view(-1, 8)], dim=1).reshape(-1).contiguous()
    res = {}
    for variant in ("fast", "generic"):
        if variant == "generic":
            monkeypatch.setenv("VTP_GEMM_NO_FAST_SWIGLU", "1")
        else:
            monkeypatch.delenv("VTP_GEMM_NO_FAST_SWIGLU", raising=False)
        out = torch.full((M, Hs), float("nan"), device="cuda", dtype=torch.bfloat16)
        pre = torch.full((M, 2 * Hs), float("nan"), device="cuda", dtype=torch.bfloat16) if with_pre else None
        lib.gemm(A, Wp, out, M=M, N=2 * Hs, K=K, bias=bp, act=lib.ACT_SWIGLU8, ldo=Hs, out2=pre)
        torch.cuda.synchronize()
        res[variant] = (out, pre)
    x1 = (A.float() @ W1.float().t() + b1).to(torch.bfloat16)
    x2 = (A.float() @ W2.float().t() + b2).to(torch.bfloat16)
    ref = (torch.nn.functional.silu(x1.float()).to(torch.bfloat16).float() * x2.float()).to(torch.bfloat16)
    out, pre = res["fast"]
    assert torch.isfinite(out.float()).all()
    assert _relerr(out, ref) < 3e-3
    assert torch.equal(out, res["generic"][0])
    if with_pre:
        pre_ref = torch.stack([x1.view(M, Hs // 8, 8), x2.view(M, Hs // 8, 8)], dim=2).reshape(M, 2 * Hs)
        assert torch.isfinite(pre.float()).all()
        assert _relerr(pre, pre_ref) < 3e-3 and torch.equal(pre, res["generic"][1])
