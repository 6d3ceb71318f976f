"""attn_fwd_256_kernel (vtp_attention_fwd with 128 < HW <= 256, not packed) at the training step's sizes, where many
CTAs share each SM and the prefix query rows of one (head, image) are spread over its query tiles and warps.

tests/test_attention_rows_gpu.py checks every row of small launches; this file adds what only the benchmark's sizes
exercise: B = 512 images at T = 257 (encoder, cls prefix) and B = 256 at T = 256 (decoder, no prefix), every
(head, image) with its own inputs, a seeded sample of images checked on every row and every image's prefix rows,
outputs in NaN buffers with sentinel rows, repeat launches bit for bit, and inputs whose row maxima lie in the second
128-key half (found by the kernel's max-only pass) or on the cls key, at logits up to about ±30.
"""
import pytest
import torch

from tests import attn_ref as ar
from tests.test_attention_rows_gpu import run_fwd

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
H = 6
SAMPLE = 12  # images checked on every row (plus the first and the last)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _qkv(B, T, seed, scale=1.2):
    return (torch.randn(B * T, 3 * H * 64, device="cuda", generator=_gen(seed)) * scale).to(BF)


def _check(qkv, out, lse, B, T, prefix, seed):
    """every row of a seeded sample of images, and the prefix rows of all images, against the emulated reference"""
    x = qkv.view(B, T, -1)
    imgs = torch.randperm(B, generator=torch.Generator().manual_seed(seed))[:SAMPLE].tolist()
    imgs = sorted(set(imgs) | {0, B - 1})
    idx = torch.tensor(imgs, device="cuda")
    n = len(imgs)
    sub = x[idx].reshape(n * T, -1)
    em, _ = ar.emulated_fwd(sub, n, T, H, prefix)
    _, lse_ex = ar.exact_fwd(sub, n, T, H, prefix)
    got = out.view(B, T, -1)[idx].reshape(n * T, -1)
    e = ar.row_err(got, em, (n, T, 1, H)).max().item()
    e_lse = ((lse[idx].double() - lse_ex).abs() / lse_ex.abs().clamp(min=1.0)).max().item()
    print(f"ROWSTAT sample_rows B={B} T={T} {e:.3e} lse {e_lse:.3e}")
    assert e <= ar.FWD_ROW_TOL, e
    assert e_lse <= 1e-4, e_lse
    if prefix:
        q, k, v = ar.heads(qkv, B, T, H, 3)
        o_pre, _ = ar.fwd_core(q[:, :, :prefix], k, v, ar.visible(T, False, q.device)[:prefix])
        em_pre = ar.merge(o_pre)  # [B * prefix, H * 64]
        got_pre = out.view(B, T, -1)[:, :prefix].reshape(B * prefix, -1)
        e_pre = ar.row_err(got_pre, em_pre, (B, prefix, 1, H)).max().item()
        s = (q[:, :, :prefix] @ k.transpose(-1, -2)) * ar.SCALE
        lse_pre_ex = torch.logsumexp(s, -1)
        e_lse_pre = ((lse[:, :, :prefix].double() - lse_pre_ex).abs() / lse_pre_ex.abs().clamp(min=1.0)).max().item()
        print(f"ROWSTAT prefix_rows B={B} T={T} {e_pre:.3e} lse {e_lse_pre:.3e}")
        assert e_pre <= ar.FWD_ROW_TOL, e_pre
        assert e_lse_pre <= 1e-4, e_lse_pre


@pytest.mark.parametrize("B,T,prefix", [(512, 257, 1), (256, 256, 0)])
def test_fwd_short_benchmark_size(B, T, prefix):
    qkv = _qkv(B, T, seed=T)
    out, lse = run_fwd(qkv, B, T, H, prefix, False)
    _check(qkv, out, lse, B, T, prefix, seed=B)
    out2, lse2 = run_fwd(qkv, B, T, H, prefix, False)
    assert torch.equal(out, out2) and torch.equal(lse, lse2)


def _stress(kind, B, T, prefix, seed):
    x = _qkv(B, T, seed, scale=3.0).float().view(B, T, 3, H, 64)
    if kind == "second_half_max":
        # q·k / 8 ~ N(0, 9²); keys 128.. gain a² / 8 = 18 logits, so every row's maximum lies in the second half and the
        # first half's numerators are up to ~40 logits below it
        a = 12.0
        x[:, :, 0, :, 0] += a
        x[:, prefix + 128:, 1, :, 0] += a
    else:
        # cls_dominant: the cls key leads by ~20 logits for the odd tokens, so their max is the prefix column and both
        # halves' numerators are tiny
        a = 160 ** 0.5  # a * a / 8 = 20
        x[:, 1::2, 0, :, 1] += a
        x[:, 0, 1, :, 1] = a
    return x.reshape(B * T, -1).to(BF)


@pytest.mark.parametrize("kind", ["second_half_max", "cls_dominant"])
def test_fwd_short_row_max_placement(kind):
    B, T, prefix = 64, 257, 1
    qkv = _stress(kind, B, T, prefix, seed=7)
    out, lse = run_fwd(qkv, B, T, H, prefix, False)
    _check(qkv, out, lse, B, T, prefix, seed=3)
