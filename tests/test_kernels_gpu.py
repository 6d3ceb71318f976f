"""GPU parity of the HBM-bound kernels and the wgmma attention against plain fp32 PyTorch references."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

from tests.attn_ref import FWD_ROW_TOL, emulated_fwd, row_err
from vtp_b200 import lib

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def _rel(x, y):
    return ((x.float() - y.float()).norm() / (y.float().norm() + 1e-30)).item()


def test_patchify():
    x = torch.randn(3, 3, 64, 96, device="cuda")
    out = torch.empty(3 * 4 * 6, 768, device="cuda", dtype=BF)
    lib.patchify(x, out, 16)
    ref = F.unfold(x, 16, stride=16).transpose(1, 2).reshape(-1, 768).to(BF)  # k = c*256 + i*16 + j
    assert torch.equal(out, ref)


@pytest.mark.parametrize("D", [384, 768, 1024, 128])
@pytest.mark.parametrize("ln", [False, True])
@pytest.mark.parametrize("in_bf16", [False, True])
def test_norm_fwd(D, ln, in_bf16):
    M = 1000
    x = torch.randn(M, D, device="cuda") * 2 + 0.3
    if in_bf16:
        x = x.to(BF)
    w = torch.randn(D, device="cuda")
    b = torch.randn(D, device="cuda") if ln else None
    eps = 1e-6 if ln else 1e-5
    y32 = torch.empty(M, D, device="cuda")
    y16 = torch.empty(M, D, device="cuda", dtype=BF)
    y3 = torch.empty(M, 3 * D, device="cuda", dtype=BF)
    rstd = torch.empty(M, device="cuda")
    mean = torch.empty(M, device="cuda")
    lib.norm_fwd(x, y32, w, b, eps, M, D, y_mode=lib.OUT_F32, rstd=rstd, mean=mean)
    lib.norm_fwd(x, y16, w, b, eps, M, D, y_mode=lib.OUT_BF16)
    lib.norm_fwd(x, y3, w, b, eps, M, D, y_mode=lib.OUT_SPLIT3)
    xf = x.float()
    if ln:
        ref = F.layer_norm(xf, (D,), w, b, eps)
    else:
        ref = (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)).type_as(x).float() * w
    assert _rel(y32, ref) < 5e-5
    assert _rel(y16, ref.to(BF)) < 2e-3
    hi, hi2, lo = y3[:, :D].float(), y3[:, D:2 * D].float(), y3[:, 2 * D:].float()
    assert torch.equal(hi, hi2)
    assert _rel(hi + lo, ref) < (1e-4 if in_bf16 else 2e-5)


def test_split3_gemm_is_fp32_accurate():
    M, N, K = 512, 384, 768
    A = torch.randn(M, K, device="cuda")
    W = torch.randn(N, K, device="cuda") * 0.05
    A3 = torch.empty(M, 3 * K, device="cuda", dtype=BF)
    W3 = torch.empty(N, 3 * K, device="cuda", dtype=BF)
    lib.split3(A, A3, M, K, b_side=False)
    lib.split3(W, W3, N, K, b_side=True)
    out = torch.empty(M, N, device="cuda")
    lib.gemm(A3, W3, out, M=M, N=N, K=3 * K, round_bf16=False)
    ref = (A.double() @ W.double().t()).float()
    assert _rel(out, ref) < 2e-5, _rel(out, ref)


def test_transpose_and_gather():
    x = torch.randn(5, 256, 64, device="cuda")
    o = torch.empty(5, 64, 256, device="cuda", dtype=BF)
    lib.transpose_batched(x, o, 5, 256, 64)
    assert torch.equal(o, x.transpose(1, 2).to(BF))
    idx = torch.randint(0, 5 * 256, (333,), device="cuda")
    g = torch.empty(333, 64, device="cuda")
    lib.gather_rows(x.view(-1, 64), g, idx, 64)
    assert torch.equal(g, x.view(-1, 64)[idx])


def test_prefix_and_mask_tokens():
    B, T, D = 3, 17, 128
    x = torch.randn(B * T, D, device="cuda")
    x0 = x.clone()
    cls = torch.randn(D, device="cuda")
    mt = torch.randn(D, device="cuda")
    lib.fill_prefix_tokens(x, cls, B, T, 1, D)
    idx = torch.tensor([0, 5, 16 + 3, 47], device="cuda", dtype=torch.long)
    lib.apply_mask_tokens(x, mt, idx, 16, T, 1, D)
    ref = x0.view(B, T, D).clone()
    ref[:, 0] = cls
    flat = ref[:, 1:].reshape(B * 16, D)
    flat[idx] = mt
    ref[:, 1:] = flat.view(B, 16, D)
    assert torch.equal(x.view(B, T, D), ref)


def _sdpa_ref(qkv, B, T, H, causal):
    q, k, v = [t.transpose(1, 2).float() for t in qkv.view(B, T, 3, H, 64).unbind(2)]
    return F.scaled_dot_product_attention(q, k, v, is_causal=causal).transpose(1, 2).reshape(B * T, H * 64)


@pytest.mark.parametrize("B,T,H,prefix,causal", [(3, 257, 6, 1, False), (2, 256, 2, 0, False), (5, 37, 6, 1, False),
                                                  (4, 77, 6, 0, True), (2, 197, 12, 1, False), (2, 130, 2, 2, False),
                                                  (64, 257, 6, 1, False), (7, 50, 2, 0, False), (3, 64, 2, 1, False),
                                                  (100, 37, 6, 1, False), (300, 257, 6, 1, False)])
@pytest.mark.parametrize("variant", ["rows4", "rows8", "pipe", "no_lse", "VTP_ATTN_NO_PACK"])
def test_attention_fwd(B, T, H, prefix, causal, variant, monkeypatch):
    """attn_fwd_kernel<NKT>: one 128-key tile (HW <= 128) or two (128 < HW <= 256), cls / prefix rows on CUDA cores, causal
    text shapes, packed multi-sequence tiles for T <= 64 (VTP_ATTN_NO_PACK=1: one sequence per tile), with and without the
    saved log-sum-exp.  rows4 / rows8 / pipe are the ids of the three pre-Hopper forward kernels (one or two threads per
    query row, persistent ping-pong); the Hopper build has the one kernel above, which all three ids run.  The cls /
    prefix rows, 1/T of the whole-tensor norm, are also checked row by row against the emulated bf16 reference
    (tests/test_attention_rows_gpu.py checks every row)."""
    if variant == "VTP_ATTN_NO_PACK":
        monkeypatch.setenv(variant, "1")
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + T)
    qkv = (torch.randn(B * T, 3 * H * 64, device="cuda", generator=g) * 1.5).to(BF)
    out = torch.full((B * T, H * 64), float("nan"), device="cuda", dtype=BF)
    lse = None if variant == "no_lse" else torch.empty(B, H, T, device="cuda")
    lib.attention_fwd(qkv, out, B, T, H, prefix=prefix, causal=causal, lse=lse)
    torch.cuda.synchronize()
    ref = _sdpa_ref(qkv, B, T, H, causal)
    assert torch.isfinite(out.float()).all()
    assert _rel(out, ref) < 6e-3, _rel(out, ref)
    if prefix:
        e = row_err(out, emulated_fwd(qkv, B, T, H, prefix, causal)[0], (B, T, 1, H))[:, :prefix].max().item()
        assert e <= FWD_ROW_TOL, ("cls rows", e)
    if lse is None:
        return
    q, k, _ = [t.transpose(1, 2).float() for t in qkv.view(B, T, 3, H, 64).unbind(2)]
    s = q @ k.transpose(-1, -2) * 0.125
    if causal:
        s = s + torch.full((T, T), float("-inf"), device="cuda").triu(1)
    assert _rel(lse, torch.logsumexp(s, -1)) < 1e-4


def test_attention_fwd_f32():
    B, T, H = 2, 257, 3
    qkv = torch.randn(B * T, 3 * H * 64, device="cuda")
    out = torch.empty(B * T, H * 64, device="cuda")
    lib.attention_fwd_f32(qkv, out, B, T, H)
    assert _rel(out, _sdpa_ref(qkv, B, T, H, False)) < 1e-5
    lib.attention_fwd_f32(qkv, out, B, T, H, causal=True)
    assert _rel(out, _sdpa_ref(qkv, B, T, H, True)) < 1e-5
