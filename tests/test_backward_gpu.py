"""GPU parity of the training-step kernels against PyTorch autograd (fp32) on the same inputs.  The attention backward
is checked row by row in tests/test_attention_rows_gpu.py."""
import pytest
import torch
import torch.nn.functional as F

from vtp_b200 import lib

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def _rel(x, y):
    return ((x.float() - y.float()).norm() / (y.float().norm() + 1e-30)).item()


@pytest.mark.parametrize("D,ln,xbf", [(384, False, False), (768, True, True), (1024, True, False), (128, False, False)])
def test_norm_bwd(D, ln, xbf):
    M = 777
    x = (torch.randn(M, D, device="cuda") * 1.5 + 0.2)
    if xbf:
        x = x.to(BF)
    w = torch.randn(D, device="cuda")
    b = torch.randn(D, device="cuda") if ln else None
    eps = 1e-6 if ln else 1e-5
    dy = torch.randn(M, D, device="cuda").to(BF)
    g0 = torch.randn(M, D, device="cuda")
    y = torch.empty(M, D, device="cuda", dtype=BF)
    rstd = torch.empty(M, device="cuda")
    mean = torch.empty(M, device="cuda") if ln else None
    lib.norm_fwd(x, y, w, b, eps, M, D, y_mode=lib.OUT_BF16, rstd=rstd, mean=mean)
    g = g0.clone()
    dw = torch.zeros(D, device="cuda")
    db = torch.zeros(D, device="cuda") if ln else None
    gb = torch.empty(M, D, device="cuda", dtype=BF)
    gs = torch.zeros(D, device="cuda")
    lib.norm_bwd(x, rstd, mean, w, dy, g, dw, db, M, D, gb_out=gb, g_colsum=gs)
    assert torch.equal(gb, g.to(BF)) and _rel(gs, g.sum(0)) < 1e-4
    xr = x.float().requires_grad_(True)
    wr = w.clone().requires_grad_(True)
    if ln:
        br = b.clone().requires_grad_(True)
        yr = F.layer_norm(xr, (D,), wr, br, eps)
    else:
        yr = xr * torch.rsqrt(xr.pow(2).mean(-1, keepdim=True) + eps) * wr
    yr.backward(dy.float())
    assert _rel(g - g0, xr.grad) < 2e-3
    assert _rel(dw, wr.grad) < 2e-3
    if ln:
        assert _rel(db, br.grad) < 2e-3


def test_swiglu_gelu_bwd():
    M, Hs = 300, 512
    x1 = torch.randn(M, Hs, device="cuda").to(BF)
    x2 = torch.randn(M, Hs, device="cuda").to(BF)
    dh = torch.randn(M, Hs, device="cuda").to(BF)
    pre = torch.stack([x1.view(M, Hs // 8, 8), x2.view(M, Hs // 8, 8)], dim=2).reshape(M, 2 * Hs).contiguous()
    dpre = torch.empty_like(pre)
    dbias = torch.zeros(2 * Hs, device="cuda")
    lib.swiglu_bwd(pre, dh, dpre, dbias, M, Hs)
    a, b = x1.float().requires_grad_(True), x2.float().requires_grad_(True)
    (F.silu(a) * b).backward(dh.float())
    d1 = dpre.view(M, Hs // 8, 2, 8)[:, :, 0].reshape(M, Hs)
    d2 = dpre.view(M, Hs // 8, 2, 8)[:, :, 1].reshape(M, Hs)
    assert _rel(d1, a.grad) < 5e-3 and _rel(d2, b.grad) < 5e-3
    assert _rel(dbias.view(Hs // 8, 2, 8)[:, 0].reshape(-1), a.grad.sum(0)) < 5e-3
    p = torch.randn(M, Hs, device="cuda").to(BF)
    dp = torch.empty_like(p)
    db = torch.zeros(Hs, device="cuda")
    lib.gelu_bwd(p, dh, dp, db, M, Hs)
    pr = p.float().requires_grad_(True)
    F.gelu(pr).backward(dh.float())
    assert _rel(dp, pr.grad) < 5e-3 and _rel(db, pr.grad.sum(0)) < 5e-3


def test_cast_colsum_l2norm_scatter_strip():
    M, N = 500, 384
    x = torch.randn(M, N, device="cuda")
    y = torch.empty(M, N, device="cuda", dtype=BF)
    cs = torch.zeros(N, device="cuda")
    lib.cast_colsum(x, y, cs, M, N)
    assert torch.equal(y, x.to(BF)) and _rel(cs, x.sum(0)) < 1e-5
    f = torch.randn(64, 256, device="cuda")
    yn = torch.empty(64, 256, device="cuda", dtype=BF)
    nrm = torch.empty(64, device="cuda")
    lib.l2norm_fwd(f, yn, 64, 256, 1e-12, norm_out=nrm)
    dy = torch.randn(64, 256, device="cuda")
    dx = torch.empty(64, 256, device="cuda")
    lib.l2norm_bwd(yn, nrm, dy, dx, 64, 256)
    fr = f.clone().requires_grad_(True)
    F.normalize(fr, dim=-1).backward(dy)
    assert _rel(dx, fr.grad) < 5e-3
    idx = torch.randint(0, 50, (200,), device="cuda")
    dst = torch.zeros(50, 64, device="cuda")
    src = torch.randn(200, 64, device="cuda")
    lib.scatter_add_rows(src, dst, idx, 64)
    assert _rel(dst, torch.zeros(50, 64, device="cuda").index_add_(0, idx, src)) < 1e-5
    B, T, D = 3, 17, 128
    g = torch.randn(B * T, D, device="cuda")
    out = torch.empty(B * 16, D, device="cuda", dtype=BF)
    dcls = torch.zeros(D, device="cuda")
    lib.strip_prefix(g, out, dcls, B, T, 1, D)
    assert torch.equal(out.view(B, 16, D), g.view(B, T, D)[:, 1:].to(BF))
    assert _rel(dcls, g.view(B, T, D)[:, 0].sum(0)) < 1e-5


def test_gemm_row_compaction():
    B, T, D, N = 3, 17, 128, 64
    A = torch.randn(B * T, D, device="cuda").to(BF)
    W = torch.randn(N, D, device="cuda").to(BF)
    out = torch.empty(B * 16, N, device="cuda", dtype=BF)
    lib.gemm(A, W, out, M=B * T, N=N, K=D, rr_group=T, rr_skip=-1)
    ref = (A.float() @ W.float().t()).view(B, T, N)[:, 1:].reshape(B * 16, N).to(BF)
    assert _rel(out, ref) < 2e-3


def test_softmax_ce_and_dino_losses():
    R, Cn = 48, 96
    logits = torch.randn(R, Cn, device="cuda") * 3
    G = torch.empty(R, Cn, device="cuda", dtype=BF)
    loss = torch.zeros(1, device="cuda")
    dsc = torch.zeros(1, device="cuda")
    lib.softmax_ce(logits, R, Cn, 16, G, 0.5 / R, loss, dsc)
    lr = logits.clone().requires_grad_(True)
    ref = 0.5 * F.cross_entropy(lr, torch.arange(16, 16 + R, device="cuda"))
    ref.backward()
    assert abs(loss.item() - ref.item()) < 1e-4 * abs(ref.item()) + 1e-6
    assert _rel(G, lr.grad) < 5e-3
    assert abs(dsc.item() - (lr.grad * logits).sum().item()) < 1e-3 * abs((lr.grad * logits).sum().item()) + 1e-5
    K, Rt, Rs = 4096, 20, 30
    t = (torch.randn(Rt, K, device="cuda") * 2).to(BF)
    center = torch.randn(K, device="cuda") * 0.1
    tp = t.clone()
    lib.dino_teacher_probs(tp, center, Rt, K, 0.07)
    tref = F.softmax((t.float() - center) / 0.07, dim=-1)
    assert _rel(tp, tref) < 5e-3
    s = (torch.randn(Rs, K, device="cuda") * 2).to(BF)
    t0 = torch.randint(0, Rt, (Rs,), device="cuda", dtype=torch.int32)
    t1 = torch.randint(0, Rt, (Rs,), device="cuda", dtype=torch.int32)
    t1[::3] = -1
    w = torch.rand(Rs, device="cuda")
    sg = s.clone()
    l2 = torch.zeros(1, device="cuda")
    lib.dino_student_ce(sg, tp, t0, t1, w, Rs, K, 0.1, l2)
    sr = s.float().requires_grad_(True)
    lsm = F.log_softmax(sr / 0.1, dim=-1)
    tpf = tp.float()
    tot = -(tpf[t0.long()] * lsm).sum(-1)
    m1 = (t1 >= 0)
    tot = tot - torch.where(m1[:, None], tpf[t1.clamp(min=0).long()] * lsm, torch.zeros_like(lsm)).sum(-1)
    refl = (tot * w).sum()
    refl.backward()
    assert abs(l2.item() - refl.item()) < 2e-3 * abs(refl.item())
    assert _rel(sg, sr.grad) < 1e-2


def test_adamw_weightnorm_recon():
    n = 10008
    p = torch.randn(n, device="cuda")
    g = torch.randn(n, device="cuda")
    m = torch.zeros(n, device="cuda")
    v = torch.zeros(n, device="cuda")
    pb = torch.empty(n, device="cuda", dtype=BF)
    tch = p.clone() + 0.1
    tb = torch.empty(n, device="cuda", dtype=BF)
    pr = p.clone().requires_grad_(True)
    opt = torch.optim.AdamW([pr], lr=1e-2, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.05)
    t_ref = tch.clone()
    for step in (1, 2, 3):
        gi = torch.randn(n, device="cuda")
        g.copy_(gi * 4.0)  # grad_scale 0.25 below
        pr.grad = gi.clone()
        opt.step()
        lib.adamw_step(p, g, m, v, pb, tch, tb, n, lr=1e-2, beta1=0.9, beta2=0.95, eps=1e-8, wd=0.05, step=step,
                       grad_scale=0.25, ema_momentum=0.99)
        t_ref = 0.99 * t_ref + 0.01 * pr.detach()
    assert _rel(p, pr.detach()) < 1e-5 and torch.equal(pb, p.to(BF)) and float(g.abs().sum()) == 0.0
    assert _rel(tch, t_ref) < 1e-5 and torch.equal(tb, tch.to(BF))
    K, D = 300, 256
    vv = torch.randn(K, D, device="cuda")
    gg = torch.rand(K, device="cuda") + 0.5
    w = torch.empty(K, D, device="cuda", dtype=BF)
    vn = torch.empty(K, device="cuda")
    lib.weight_norm_fwd(vv, gg, w, vn, K, D)
    vr, gr = vv.clone().requires_grad_(True), gg.clone().requires_grad_(True)
    wr = gr[:, None] * vr / vr.norm(dim=1, keepdim=True)
    assert _rel(w, wr) < 5e-3
    dW = torch.randn(K, D, device="cuda")
    wr.backward(dW)
    dv = torch.zeros(K, D, device="cuda")
    dg = torch.zeros(K, device="cuda")
    lib.weight_norm_bwd(vv, gg, vn, dW, dv, dg, K, D)
    assert _rel(dv, vr.grad) < 1e-4 and _rel(dg, gr.grad) < 1e-4
    B, gh, gw, r = 2, 4, 4, 16
    rec = torch.randn(B, 3, gh * r, gw * r, device="cuda").to(BF)
    tgt = torch.randn(B, 3, gh * r, gw * r, device="cuda")
    out = torch.empty(B * gh * gw, 3 * r * r, device="cuda", dtype=BF)
    la = torch.zeros(1, device="cuda")
    coef = 1.0 / rec.numel()
    lib.recon_l1_grad(rec, tgt, None, out, la, B, 3, gh, gw, r, coef)
    rr = rec.float().requires_grad_(True)
    lref = (rr - tgt).abs().mean()
    lref.backward()
    assert abs(la.item() - lref.item()) < 1e-4 * lref.item()
    gref = F.pixel_unshuffle(rr.grad, r).permute(0, 2, 3, 1).reshape(B * gh * gw, 3 * r * r)
    assert _rel(out, gref) < 5e-3
