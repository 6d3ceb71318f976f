"""The references of tests/step_ref.py and its two checkers, proved without a GPU.

- each reference equals fp64 autograd of a plain torch restatement of its operation (norm, SwiGLU, GELU, softmax
  cross-entropy, DINO / iBOT, L1, AdamW, max-pool, LPIPS tap, im2col / col2im);
- elem_k / col_k reject a set of seeded kernel bugs, each built from a reference output, by at least 2x the bounds the
  GPU tests apply (each test prints its margin).
"""
import math

import pytest
import torch
import torch.nn.functional as F

from tests import step_ref as sr

D64 = torch.float64


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _close(a, b, tol=1e-12):
    a, b = a.double(), b.double()
    assert ((a - b).abs().max() / (b.abs().max() + 1e-300)).item() < tol


def _rejects(name, k, bound):
    print(f"{name}: k = {k:.3g}, bound {bound:g}, margin {k / bound:.3g}x")
    assert k >= 2 * bound, (name, k, bound)


# ------------------------------------------------------------------------------------------------- vs fp64 autograd

@pytest.mark.parametrize("ln,xbf", [(False, False), (True, False), (False, True), (True, True)])
def test_norm_matches_autograd(ln, xbf):
    M, D = 37, 200
    g = _g(1)
    x = torch.randn(M, D, generator=g, dtype=D64) * 1.5 + 0.2
    if xbf:
        x = x.to(torch.bfloat16)
    w, b = torch.randn(D, generator=g, dtype=D64), (torch.randn(D, generator=g, dtype=D64) if ln else None)
    dy = torch.randn(M, D, generator=g).to(torch.bfloat16)
    g0 = torch.randn(M, D, generator=g, dtype=D64)
    eps = 1e-6 if ln else 1e-5
    y, rstd, mean, _ = sr.norm_fwd(x, w, b, eps)
    ref = sr.norm_bwd(x, rstd, mean if ln else None, w, dy, g0)
    xr, wr = x.double().requires_grad_(True), w.clone().requires_grad_(True)
    br = b.clone().requires_grad_(True) if ln else None
    if ln:
        yr = F.layer_norm(xr, (D,), wr, br, sr.f32(eps))
    else:
        xh = xr * torch.rsqrt(xr.pow(2).mean(-1, keepdim=True) + sr.f32(eps))
        if xbf:  # .type_as(x): a rounding whose gradient is the identity
            xh = xh + (sr.bf16((x.float() * rstd.float()[:, None]).double()) - xh).detach()
        yr = xh * wr
    _close(yr, y, 1e-12 if not (xbf and not ln) else 1e-6)
    yr.backward(dy.double())
    _close(wr.grad, ref["dw"])
    if ln:
        _close(br.grad, ref["db"])
    if xbf and not ln:
        # the kernel's x̂·m2 correction uses the rounded x̂, autograd the unrounded one (step_ref.norm_bwd)
        xh_r = sr.bf16((x.float() * rstd.float()[:, None]).double())
        dxw = dy.double() * w
        bound = 2.0 ** -8 * rstd[:, None] * (xh_r.abs() * (dxw * xh_r).mean(1, keepdim=True).abs()
                                              + (dxw * xh_r).abs().mean(1, keepdim=True))
        assert ((ref["g"] - g0 - xr.grad).abs() <= bound).all()
    else:
        _close(ref["g"] - g0, xr.grad, 1e-11)


def test_swiglu_gelu_match_autograd():
    M, Hs = 29, 48
    g = _g(2)
    pre = (torch.randn(M, 2 * Hs, generator=g) * 2).to(torch.bfloat16)
    dh = torch.randn(M, Hs, generator=g).to(torch.bfloat16)
    x1, x2 = [t.double().requires_grad_(True) for t in sr.split8(pre, Hs)]
    (F.silu(x1) * x2).backward(dh.double())
    dpre, _, db, _ = sr.swiglu_bwd(pre, dh, Hs)
    _close(dpre, sr.join8(x1.grad, x2.grad))
    _close(db, sr.join8(x1.grad, x2.grad).sum(0))
    hid, alt, _ = sr.swiglu_fwd(pre, Hs)
    assert torch.equal(hid, sr.bf16(sr.bf16(F.silu(x1.detach())) * x2.detach()))
    assert (alt != hid).double().mean() < 0.05         # the other rounding is admitted only next to a midpoint
    p = (torch.randn(M, Hs, generator=g) * 2).to(torch.bfloat16)
    pr = p.double().requires_grad_(True)
    F.gelu(pr).backward(dh.double())
    d, _, db, _ = sr.gelu_bwd(p, dh)
    _close(d, pr.grad)
    _close(db, pr.grad.sum(0))


@pytest.mark.parametrize("log_scale", [None, math.log(100.0)])
def test_softmax_ce_matches_autograd(log_scale):
    R, C, ld, label0, coef = 8, 40, 48, 16, 0.5 / 8
    lg = torch.randn(R, ld, generator=_g(3), dtype=D64) * 0.3
    ref = sr.softmax_ce(lg, C, label0, coef, log_scale)
    x = lg[:, :C].clone().requires_grad_(True)
    ls = torch.tensor(sr.f32(log_scale) if log_scale is not None else 0.0, dtype=D64, requires_grad=True)
    loss = coef * F.cross_entropy(ls.exp() * x, label0 + torch.arange(R), reduction="sum")
    loss.backward()
    _close(ref["loss"], loss.detach())
    _close(ref["G"], x.grad)
    _close(ref["dscale"], ls.grad)


def test_dino_matches_autograd():
    K, Rt, Rs, temp, ttemp = 64, 5, 9, 0.1, 0.04
    g = _g(4)
    t = torch.randn(Rt, K, generator=g, dtype=D64) * 0.5
    c = torch.randn(K, generator=g, dtype=D64) * 0.1
    tp, _ = sr.dino_teacher(t, c, ttemp)
    _close(tp, F.softmax((t - c) / sr.f32(ttemp), -1))
    s = torch.randn(Rs, K, generator=g, dtype=D64)
    t0 = torch.tensor([0, 1, 2, -1, 4, -1, 0, 3, 1], dtype=torch.int32)
    t1 = torch.tensor([1, -1, 3, 2, -1, -1, 4, 0, 1], dtype=torch.int32)
    w = torch.rand(Rs, generator=g, dtype=D64)
    ref = sr.dino_student(s, tp, t0, t1, w, temp)
    sg = s.clone().requires_grad_(True)
    lsm = F.log_softmax(sg / sr.f32(temp), -1)
    loss = 0
    for r in range(Rs):
        for i in (int(t0[r]), int(t1[r])):
            if i >= 0:
                loss = loss - w[r] * (tp[i] * lsm[r]).sum()
    loss.backward()
    _close(ref["loss"], loss.detach())
    _close(ref["ds"], sg.grad)
    assert (ref["ds"][5] == 0).all()                     # a row without teachers: no gradient
    one = sr.dino_student(s[3:4], tp, torch.tensor([2], dtype=torch.int32), None, w[3:4], temp)
    _close(one["ds"], ref["ds"][3:4])                   # t0 = −1, t1 = 2 is the row with teacher 2 alone


def test_recon_l1_matches_autograd():
    B, C, gh, gw, r = 2, 3, 2, 3, 4
    g = _g(5)
    rec = torch.randn(B, C, gh * r, gw * r, generator=g).to(torch.bfloat16)
    tgt = rec.double().clone()
    tgt[:, :, ::3] += torch.randn(B, C, (gh * r + 2) // 3, gw * r, generator=g, dtype=D64)
    dlp = torch.randn(B, C, gh * r, gw * r, generator=g, dtype=D64) * 1e-3
    coef = 1.0 / rec.numel()
    out, loss, _ = sr.recon_l1(rec, tgt, dlp, coef, r)
    rr = rec.double().requires_grad_(True)
    (coef * (rr - tgt).abs().sum()).backward()       # torch: d|x|/dx = sign(x), 0 at 0 — as the kernel
    _close(loss, coef * (rec.double() - tgt).abs().sum())
    _close(out, F.pixel_unshuffle(rr.grad + dlp, r).permute(0, 2, 3, 1).reshape(B * gh * gw, C * r * r))


def test_adamw_matches_torch():
    n, steps = 64, 5
    g = _g(6)
    p = torch.randn(n, generator=g, dtype=D64)
    m, v = torch.zeros(n, dtype=D64), torch.zeros(n, dtype=D64)
    pr = p.clone().requires_grad_(True)
    hp = dict(lr=sr.f32(1e-3), b1=sr.f32(0.9), b2=sr.f32(0.999), eps=sr.f32(1e-8), wd=sr.f32(0.04))
    opt = torch.optim.AdamW([pr], lr=hp["lr"], betas=(hp["b1"], hp["b2"]), eps=hp["eps"], weight_decay=hp["wd"])
    t, t_ref, mom = p.clone() + 0.1, p.clone() + 0.1, sr.f32(0.99)
    for step in range(1, steps + 1):
        gr = torch.randn(n, generator=g, dtype=D64)
        pr.grad = gr * 0.25
        opt.step()
        t_ref = mom * t_ref + (1 - mom) * pr.detach()
        o = sr.adamw(p, m, v, gr, **hp, step=step, grad_scale=0.25, teacher=t, mom=0.99)
        p, m, v, t = o["p"], o["m"], o["v"], o["teacher"]
    _close(t, t_ref, 1e-12)
    _close(p, pr.detach(), 1e-12)
    _close(m, opt.state[pr]["exp_avg"])
    _close(v, opt.state[pr]["exp_avg_sq"])


def test_maxpool_and_pool_relu_match_autograd():
    B, H, W, C = 2, 6, 4, 8
    g = _g(7)
    y = F.relu(torch.randn(B, H, W, C, generator=g, dtype=D64))
    y = y + torch.rand(B, H, W, C, generator=g, dtype=D64) * 1e-3 * (y > 0)   # distinct maxima
    yr = y.clone().requires_grad_(True)
    pooled = F.max_pool2d(yr.permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)
    assert torch.equal(sr.maxpool2(y), pooled.detach())
    dpool = torch.randn(B, H // 2, W // 2, C, generator=g, dtype=D64)
    gtap = torch.randn(B, H, W, C, generator=g, dtype=D64)
    z = yr  # y is the ReLU output: the kernel's mask y > 0 is relu'(z)
    ((pooled * dpool).sum() + (F.relu(z) * gtap).sum()).backward()
    _close(sr.pool_relu_bwd(y, dpool, gtap), yr.grad * (y > 0))
    # ties: the first maximum in row-major window order takes the pooled gradient
    t = torch.zeros(1, 2, 2, 1, dtype=D64)
    t[0, 0, 1, 0] = t[0, 1, 1, 0] = 2.0
    out = sr.pool_relu_bwd(t, torch.ones(1, 1, 1, 1, dtype=D64), None)
    assert out.flatten().tolist() == [0.0, 1.0, 0.0, 0.0]


def test_lpips_tap_matches_autograd():
    P, C, coef = 11, 64, 0.37
    g = _g(8)
    f0 = F.relu(torch.randn(P, C, generator=g, dtype=D64))
    f1 = F.relu(torch.randn(P, C, generator=g, dtype=D64))
    f1[3] = 0                                                # a dead target pixel
    w = torch.rand(C, generator=g, dtype=D64)
    ref = sr.lpips_tap(f0, f1, w, coef)
    a = f0.clone().requires_grad_(True)
    eps = sr.f32(1e-10)
    n0 = a / (a.norm(dim=1, keepdim=True) + eps)
    n1 = f1 / (f1.norm(dim=1, keepdim=True) + eps)
    loss = coef * (w * (n0 - n1) ** 2).sum()
    loss.backward()
    _close(ref["loss"], loss.detach())
    _close(ref["g0"], a.grad * (f0 > 0), 1e-10)


def test_im2col_col2im_match_autograd():
    B, H, W = 2, 5, 7
    g = _g(9)
    img = torch.rand(B, 3, H, W, generator=g, dtype=D64).requires_grad_(True)
    sh = torch.tensor([sr.f32(v) for v in sr.LP_SHIFT], dtype=D64).view(1, 3, 1, 1)
    sc = torch.tensor([sr.f32(v) for v in sr.LP_SCALE], dtype=D64).view(1, 3, 1, 1)
    u = F.unfold((img - sh) / sc, 3, padding=1)                       # [B, c*9 + tap, H*W]
    u = u.view(B, 3, 9, H * W).permute(0, 3, 2, 1).reshape(B * H * W, 27)  # k = tap*3 + c
    col = sr.lpips_prep(img.detach())
    _close(col[:, :27], u.detach())
    assert (col[:, 27:] == 0).all()
    dcol = torch.randn(B * H * W, 32, generator=g, dtype=D64)
    (u * dcol[:, :27]).sum().backward()
    dimg, _ = sr.lpips_img_grad(dcol, B, H, W)
    _close(dimg, img.grad)


# ------------------------------------------------------------------------------------------------- seeded mutations

def _norm_case(M, D, seed):
    g = _g(seed)
    x = torch.randn(M, D, generator=g, dtype=D64) + 0.2
    w = torch.randn(D, generator=g, dtype=D64)
    dy = torch.randn(M, D, generator=g).to(torch.bfloat16)
    _, rstd, _, _ = sr.norm_fwd(x, w, None, 1e-5)
    return x, rstd, w, dy


def test_dw_missing_strip_rejected():
    """the persistent strip loop ends one strip early: dw misses 32 rows, at the benchmark's M"""
    M, D = 131584, 8
    x, rstd, w, dy = _norm_case(M, D, 10)
    ref = sr.norm_bwd(x, rstd, None, w, dy, torch.zeros(1, D, dtype=D64))
    xh = x * rstd[:, None]
    r0 = 32 * 2000
    mut = ref["dw"] - (dy.double()[r0:r0 + 32] * xh[r0:r0 + 32]).sum(0)
    _rejects("dw without one 32-row strip", sr.col_k(mut, ref["dw"], ref["dw_abs"]), sr.COL_K)


def test_colsum_doubled_strip_rejected():
    """one 64-row strip of cast_colsum counted twice (a strip walked by two blocks)"""
    M, N = 131584, 8
    x = torch.randn(M, N, generator=_g(11), dtype=D64)
    ref, absum = x.sum(0), x.abs().sum(0)
    mut = ref + x[64 * 700:64 * 701].sum(0)
    _rejects("column sum with a 64-row strip twice", sr.col_k(mut, ref, absum), sr.COL_K)


def test_swiglu_swapped_group_rejected():
    """x1 / x2 halves of one 8-group of dpre exchanged"""
    M, Hs = 16, 64
    g = _g(12)
    pre = torch.randn(M, 2 * Hs, generator=g).to(torch.bfloat16)
    dh = torch.randn(M, Hs, generator=g).to(torch.bfloat16)
    dpre, scale, _, _ = sr.swiglu_bwd(pre, dh, Hs)
    ref = sr.bf16(dpre)
    mut = ref.clone().view(M, Hs // 8, 2, 8)
    mut[5, 3] = mut[5, 3].flip(0)
    _rejects("dpre with one swapped 8-group", sr.elem_k(mut.view(M, 2 * Hs), dpre, scale), sr.ACT_K)


def test_dino_lone_second_teacher_rejected():
    """the row t0 = −1, t1 ≥ 0 computed the way the kernel did before the fix: n = 1 but no teacher term"""
    K, temp = 256, 0.1
    g = _g(13)
    tp = F.softmax(torch.randn(3, K, generator=g, dtype=D64) / 0.04, -1)
    s = torch.randn(1, K, generator=g, dtype=D64)
    w = torch.tensor([0.7], dtype=D64)
    ref = sr.dino_student(s, tp, torch.tensor([-1], dtype=torch.int32), torch.tensor([2], dtype=torch.int32), w, temp)
    z = s / sr.f32(temp)
    mut_ds = w * (1 / sr.f32(temp)) * torch.softmax(z, -1)
    mut_loss = w * torch.logsumexp(z, -1)
    _rejects("ds of the lone-t1 row", sr.elem_k(sr.bf16(mut_ds), ref["ds"], ref["ds_scale"]), sr.DINO_K)
    _rejects("loss of the lone-t1 row", sr.col_k(mut_loss.sum(), ref["loss"], ref["loss_abs"]), sr.DINO_K)


def test_pool_ties_to_last_rejected():
    """a window tie routed to the LAST maximum"""
    g = _g(14)
    y = sr.bf16(F.relu(torch.randn(1, 4, 4, 8, generator=g, dtype=D64)) + 0.5)
    y[0, 0, 0, :] = y[0, 1, 1, :] = 3.0                    # window (0, 0): (0,0) and (1,1) tie in every channel
    dpool = torch.randn(1, 2, 2, 8, generator=g).to(torch.bfloat16).double()
    gtap = torch.randn(1, 4, 4, 8, generator=g).to(torch.bfloat16).double()
    ref = sr.pool_relu_bwd(y, dpool, gtap)
    mut = ref.clone()
    mut[0, 0, 0] -= dpool[0, 0, 0]
    mut[0, 1, 1] += dpool[0, 0, 0]
    scale = gtap.abs() + dpool.abs().repeat_interleave(2, 1).repeat_interleave(2, 2)
    _rejects("ties routed to the last maximum", sr.elem_k(sr.bf16(mut), ref, scale), sr.LPIPS_K)


def test_col2im_flipped_tap_rejected():
    """col2im reading h + dy − 1 instead of h − dy + 1 (= the reference applied to the taps in reverse order)"""
    B, H, W = 1, 6, 9
    dcol = torch.randn(B * H * W, 32, generator=_g(15)).to(torch.bfloat16).double()
    ref, absum = sr.lpips_img_grad(dcol, B, H, W)
    rev = dcol.clone()
    rev[:, :27] = dcol[:, :27].view(-1, 9, 3).flip(1).reshape(-1, 27)
    mut, _ = sr.lpips_img_grad(rev, B, H, W)
    _rejects("col2im with a flipped tap", sr.elem_k(mut, ref, absum, ulps=0), sr.LPIPS_K)


def test_adam_bias_correction_off_by_one_rejected():
    n = 4096
    g = _g(16)
    p = torch.randn(n, generator=g, dtype=D64)
    m = torch.randn(n, generator=g, dtype=D64) * 1e-2
    v = torch.rand(n, generator=g, dtype=D64) * 1e-4
    gr = torch.randn(n, generator=g, dtype=D64) * 1e-2
    hp = dict(lr=1e-3, b1=0.9, b2=0.999, eps=1e-8, wd=0.04, grad_scale=1.0)
    ref = sr.adamw(p, m, v, gr, step=3, **hp)
    mut = sr.adamw(p, m, v, gr, step=4, **hp)
    _rejects("AdamW bias correction one step off", sr.elem_k(mut["p"], ref["p"], ref["p_scale"], ulps=0), sr.ADAM_K)


def test_softmax_ce_label0_ignored_rejected():
    R, C = 32, 96
    lg = torch.randn(R, C, generator=_g(17), dtype=D64) * 0.3
    ref = sr.softmax_ce(lg, C, 32, 1.0 / 64, math.log(100.0))
    mut = sr.softmax_ce(lg, C, 0, 1.0 / 64, math.log(100.0))
    _rejects("softmax_ce with label0 ignored", sr.elem_k(sr.bf16(mut["G"]), ref["G"], ref["G_scale"]), sr.CE_K)
    _rejects("softmax_ce loss with label0 ignored", sr.col_k(mut["loss"], ref["loss"], ref["loss_abs"]), sr.CE_SUM_K)


def test_checkers_accept_their_own_rounding():
    """a correctly rounded bf16 result passes at k = 0; one ulp more does not"""
    ref = torch.randn(1000, generator=_g(18), dtype=D64)
    assert sr.elem_k(sr.bf16(ref), ref, 0.0) == 0.0
    bumped = sr.bf16(ref) + 2 * sr.ulp_bf16(ref)
    assert sr.elem_k(bumped, ref, ref.abs()) > 1e4
    assert sr.elem_k(torch.full_like(ref, float("nan")), ref, 1.0) == math.inf
    assert sr.col_k(ref, ref, ref.abs()) == 0.0


def _trunc_bf16(x):
    """bf16 by truncation (round toward zero) instead of round-to-nearest"""
    b = x.float().view(torch.int32) & -65536
    return b.view(torch.float32).double()


@pytest.mark.parametrize("mutation", ["no inner rounding", "truncation instead of round-to-nearest"])
def test_swiglu_fwd_rounding_mutations_rejected(mutation):
    """swiglu_fwd output without the inner round(silu(x1)), or rounded by truncation, compared the way the GPU test
    compares (the nearer of hid / alt, no ulp of slack)"""
    M, Hs = 4000, 1024
    pre = (torch.randn(M, 2 * Hs, generator=_g(19)) * 2).to(torch.bfloat16)
    x1, x2 = [t.double() for t in sr.split8(pre, Hs)]
    silu = x1 * torch.sigmoid(x1)
    mut = sr.bf16(silu * x2) if mutation == "no inner rounding" else _trunc_bf16(_trunc_bf16(silu) * x2)
    hid, alt, scale = sr.swiglu_fwd(pre, Hs)
    ref = torch.where((mut - alt).abs() < (mut - hid).abs(), alt, hid)
    _rejects(f"swiglu_fwd with {mutation}", sr.elem_k(mut, ref, scale, ulps=0), sr.ACT_K)
