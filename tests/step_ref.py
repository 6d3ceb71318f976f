"""Plain-torch fp64 references for the memory-bound and loss kernels of the training step, on the CPU or the GPU (no
kernels, nothing from oracle/), and the two checkers the GPU tests apply to them.

Each reference is the exact maths its kernel implements, computed in fp64 from the very values the kernel receives
(bf16 operands upcast), with a rounding only where the kernel itself rounds: bf16 outputs, the RMSNorm `.type_as(x)`
rounding of x̂ for bf16 x, swiglu_fwd's round(round(silu(x1))·x2), and pool_relu_bwd's first-maximum rule.

elem_k  elementwise: the smallest k with |got − ref| ≤ u·ulp_bf16(ref) + k·2⁻²⁴·scale, where u = 1 for bf16 outputs (a
        correct bf16 result is within one ulp of the fp64 value) and 0 for fp32 ones, and `scale` is the magnitude of
        the terms the kernel sums or cancels in fp32 (not the result).
col_k   reductions (bias / weight gradients, column sums, loss scalars): the smallest k with
        |got − ref| ≤ k·2⁻²⁴·Σ|terms| for every column.

The GPU tests (tests/test_step_kernels_gpu.py) assert k ≤ the bounds below; tests/test_step_ref_cpu.py proves the
references against fp64 autograd and shows each bound rejecting a seeded kernel bug with at least 2x margin.

Bounds: 1.8x to 2.3x the largest k measured over every case of the GPU file on an H100 80GB HBM3 (700 W power limit),
two launches per reduction, over three runs (the atomic accumulators vary from run to run):
    bound        value  measured maxima
    NORM_FWD_K   6      rstd 3.08 (rsqrtf), y fp32 1.46, y bf16 0.03, mean 0.03
    NORM_G_K     0.6    norm_bwd g 0.29
    COL_K        5      dbias 2.29 (swiglu) / 1.78 (gelu), norm_bwd dw 0.59, g_colsum 0.44, cast_colsum 0.27
    ACT_K        0.5    recon_l1 out 0.24, gelu dpre 0.23, swiglu dpre 0; swiglu_fwd 0 with no ulp of slack (bit-exact)
    CE_K         1      softmax_ce G 0.52
    CE_SUM_K     3.5    softmax_ce loss 1.74, dscale 0.11
    DINO_K       2      teacher probs 0.99, student ds 0.98, student loss 0.86
    LOSS_K       32     recon_l1 loss 17.6, lpips_tap loss 13.3
    LPIPS_K      2      lpips_img_grad 0.86, lpips_tap g0 0.20, lpips_prep and pool_relu_bwd 0
    ADAM_K       20     p 9.6, v 0.99, m 0.98, teacher 0.96
Three effects of the kernels' fp32 arithmetic are part of the scales below, not bugs: gelu_bwd forms Φ(x) as
0.5 (1 + erf(x/√2)), which cancels for x < 0 (absolute error ~2⁻²⁵|dy|); the DINO kernels' ex2.approx.ftz returns 0
below 2⁻¹²⁶; and hyper_tick's 1 − β2^step cancels in fp32, so the AdamW reference reads the bias corrections from
`hyper` as the kernel does (hyper_tick is checked on its own).
"""
import math

import torch

U24 = 2.0 ** -24

NORM_FWD_K = 6.0     # norm_fwd y, rstd, mean
NORM_G_K = 0.6       # norm_bwd g
COL_K = 5.0          # per-column sums: dw, g_colsum, dbias, cast_colsum
ACT_K = 0.5          # swiglu / gelu dpre, swiglu_fwd, recon_l1 out
CE_K = 1.0           # softmax_ce G
CE_SUM_K = 3.5       # softmax_ce loss and dscale accumulators
DINO_K = 2.0         # teacher probs, student ds and loss
LOSS_K = 32.0        # recon_l1 and lpips_tap loss: about a thousand same-sign fp32 atomics into one scalar
LPIPS_K = 2.0        # lpips_prep, pool_relu_bwd, lpips_tap g0, lpips_img_grad
ADAM_K = 20.0        # AdamW p, m, v, teacher

LP_SHIFT = (-0.030, -0.088, -0.188)   # lpips.cu LP_SHIFT / LP_SCALE, stored as fp32 constants
LP_SCALE = (0.458, 0.448, 0.450)


def f32(v):
    """a Python float as the fp32 value the kernel holds, back in fp64"""
    return float(torch.tensor(v, dtype=torch.float32))


def bf16(x):
    """round to the nearest bf16 (ties to even, as __float2bfloat16_rn), keeping x's dtype"""
    return x.to(torch.bfloat16).to(x.dtype)


def ulp_bf16(x):
    """spacing of bf16 numbers at |x| (2^(e−7) for 2^e ≤ |x| < 2^(e+1)); the subnormal spacing at 0"""
    a = x.double().abs().clamp(min=2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 7)


# ---------------------------------------------------------------------------------------------------------- checkers

def elem_k(got, ref, scale, ulps=1.0):
    """max over elements of the k needed for |got − ref| ≤ ulps·ulp_bf16(ref) + k·2⁻²⁴·scale; inf if any got is not
    finite or an error remains where scale is 0"""
    got, ref = got.double(), ref.double()
    if not torch.isfinite(got).all():
        return math.inf
    excess = ((got - ref).abs() - ulps * ulp_bf16(ref) * (ulps > 0)).clamp(min=0)
    if ulps > 0:
        excess = torch.where(ref == 0, (got - ref).abs(), excess)
    s = torch.as_tensor(scale, dtype=torch.float64, device=got.device).expand_as(got)
    k = torch.where(excess == 0, torch.zeros_like(excess), excess / (U24 * s))
    return k.max().item() if k.numel() else 0.0


def col_k(got, ref, abs_sum):
    """max over columns of |got − ref| / (2⁻²⁴ Σ|terms|); inf if a got value is not finite"""
    got, ref = got.double(), ref.double()
    if not torch.isfinite(got).all():
        return math.inf
    d = (got - ref).abs()
    s = torch.as_tensor(abs_sum, dtype=torch.float64, device=got.device).expand_as(d)
    k = torch.where(d == 0, torch.zeros_like(d), d / (U24 * s))
    return k.max().item() if k.numel() else 0.0


# ------------------------------------------------------------------------------------------------------------ norms

def norm_fwd(x, w, b, eps, rstd_kernel=None):
    """RMSNorm (b None) or LayerNorm of x [M, D] -> (y, rstd, mean, scale_y).  For bf16 x, RMSNorm rounds x̂ = x·rstd to
    bf16 before the weight multiply (.type_as(x)); the kernel forms x·rstd in fp32 with its own rstd, so that product is
    taken from rstd_kernel when given (a rounding decision cannot be reproduced from an rstd that differs in the last
    bit)."""
    xd = x.double()
    D = x.shape[1]
    if b is None:
        mean = torch.zeros_like(xd[:, 0])
        rstd = torch.rsqrt(xd.pow(2).mean(1) + f32(eps))
    else:
        mean = xd.mean(1)
        rstd = torch.rsqrt((xd - mean[:, None]).pow(2).mean(1) + f32(eps))
    xh = (xd - mean[:, None]) * rstd[:, None]
    if b is None and x.dtype == torch.bfloat16:
        r = rstd if rstd_kernel is None else rstd_kernel.double()
        xh = bf16((x.float() * r.float()[:, None]).double())
    y = xh * w.double() + (0 if b is None else b.double())
    scale = (xh.abs() * w.double().abs() + (0 if b is None else b.double().abs())) * D ** 0.5
    return y, rstd, mean, scale


def norm_bwd(x, rstd, mean, w, dy, g0):
    """norm_bwd_kernel's maths, from the forward's rstd / mean (mean None: RMSNorm):
        x̂ = (x − mean)·rstd   (bf16 x under RMSNorm: x̂ = bf16(fp32(x·rstd)), the forward's .type_as(x) value)
        g = g0 + rstd (dy·w − m1 − x̂·m2),  m1 = mean(dy·w) (LayerNorm only), m2 = mean(dy·w·x̂)
        dw = Σ_rows dy·x̂, db = Σ_rows dy
    The bf16-x RMSNorm case uses the rounded x̂ in m2 and in the x̂·m2 term, where autograd of the forward (which sees
    .type_as as an identity) uses the unrounded one: the two differ by at most 2⁻⁸·rstd·(|x̂·m2| + mean|dy·w·x̂|) per
    element (|bf16(x̂) − x̂| ≤ 2⁻⁹|x̂|), which tests/test_step_ref_cpu.py checks.
    -> dict(g, dw, db, g_scale, dw_abs, db_abs)"""
    is_ln = mean is not None
    xd, r, wd, dyd = x.double(), rstd.double()[:, None], w.double(), dy.double()
    if is_ln:
        xh = (xd - mean.double()[:, None]) * r
    elif x.dtype == torch.bfloat16:
        xh = bf16((x.float() * rstd.float()[:, None]).double())
    else:
        xh = xd * r
    dxw = dyd * wd
    D = x.shape[1]
    m1 = dxw.mean(1, keepdim=True) if is_ln else torch.zeros_like(r)
    m2 = (dxw * xh).mean(1, keepdim=True)
    g = g0.double() + r * (dxw - m1 - xh * m2)
    g_scale = g0.double().abs() + r * (dxw.abs() + dxw.abs().mean(1, keepdim=True)
                                       + xh.abs() * (dxw * xh).abs().mean(1, keepdim=True)) * D ** 0.5
    return dict(g=g, dw=(dyd * xh).sum(0), db=dyd.sum(0), g_scale=g_scale, dw_abs=(dyd * xh).abs().sum(0),
                db_abs=dyd.abs().sum(0))


# ---------------------------------------------------------------------------------------------------------- SwiGLU

def split8(pre, Hs):
    """8-interleaved [M, 2Hs] (x1 | x2 in groups of 8) -> x1, x2 [M, Hs]"""
    v = pre.reshape(pre.shape[0], Hs // 8, 2, 8)
    return v[:, :, 0].reshape(-1, Hs), v[:, :, 1].reshape(-1, Hs)


def join8(a, b):
    """inverse of split8"""
    M, Hs = a.shape
    return torch.stack([a.reshape(M, Hs // 8, 8), b.reshape(M, Hs // 8, 8)], 2).reshape(M, 2 * Hs)


def swiglu_fwd(pre, Hs):
    """hid = round(round(silu(x1))·x2) -> (hid, alt, scale).  Where silu(x1) lies within 2⁻¹⁶ (relative) of a bf16
    rounding midpoint, the kernel's fp32 silu may round the other way: alt holds the result for that other neighbour
    there and equals hid everywhere else."""
    x1, x2 = [t.double() for t in split8(pre, Hs)]
    silu = x1 * torch.sigmoid(x1)
    s = bf16(silu)
    d = silu - s
    near = ((d.abs() - 0.5 * ulp_bf16(silu)).abs() <= 2.0 ** -16 * silu.abs()) & (d != 0)
    other = torch.where(near, s + torch.sign(d) * ulp_bf16(silu), s)
    return bf16(s * x2), bf16(other * x2), s.abs() * (1 + x1.abs()) * x2.abs()


def swiglu_bwd(pre, dhid, Hs):
    """dpre = (d1 | d2) 8-interleaved, d1 = dh·x2·σ(1 + x1(1 − σ)), d2 = dh·x1·σ; dbias = colsum(dpre) of the unrounded
    values -> (dpre, scale, dbias, dbias_abs)"""
    x1, x2 = [t.double() for t in split8(pre, Hs)]
    dh = dhid.double()
    sg = torch.sigmoid(x1)
    d1 = dh * x2 * sg * (1 + x1 * (1 - sg))
    d2 = dh * x1 * sg
    a = 1 + x1.abs()
    s1 = (dh * x2 * sg).abs() * a * a
    s2 = (dh * x1 * sg).abs() * a
    dpre = join8(d1, d2)
    return dpre, join8(s1, s2), dpre.sum(0), dpre.abs().sum(0)


def gelu_bwd(pre, dhid):
    """dpre = dh·(Φ(x) + x·φ(x)) (exact erf GELU) -> (dpre, scale, dbias, dbias_abs)"""
    x, dh = pre.double(), dhid.double()
    cdf = 0.5 * (1 + torch.erf(x / math.sqrt(2)))
    pdf = torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)
    d = dh * (cdf + x * pdf)
    scale = dh.abs() * (1 + x.abs() * pdf * (1 + x * x))  # 1 + erf cancels in fp32 for x < 0
    return d, scale, d.sum(0), d.abs().sum(0)


# ------------------------------------------------------------------------------------------------------------ losses

def softmax_ce(logits, C, label0, coef, log_scale=None):
    """softmax_ce_kernel on the first C columns of logits [R, ld]: s = exp(log_scale) (1 without), x = s·logits,
    label(r) = label0 + r, g = coef (softmax(x) − onehot)
    -> dict(G = s·g [R, C], loss = coef Σ_r (lse_r − x[r, label]), dscale = Σ g·x, and the scales)"""
    R = logits.shape[0]
    sc = math.exp(f32(log_scale)) if log_scale is not None else 1.0
    x = sc * logits[:, :C].double()
    lse = torch.logsumexp(x, 1)
    p = torch.exp(x - lse[:, None])
    oh = torch.zeros_like(p)
    oh[torch.arange(R), label0 + torch.arange(R)] = 1.0
    g = coef * (p - oh)
    xl = x[torch.arange(R), label0 + torch.arange(R)]
    m = x.abs().amax(1)
    spread = 1 + (x - lse[:, None]).abs() + m[:, None]
    return dict(G=sc * g, G_scale=abs(sc * coef) * (p + oh) * spread,
                loss=(coef * (lse - xl)).sum(), loss_abs=(abs(coef) * (lse.abs() + xl.abs() + m)).sum(),
                dscale=(g * x).sum(), dscale_abs=(abs(coef) * (p + oh) * x.abs() * spread).sum())


FTZ = 2.0 ** -126 / U24   # ex2.approx.ftz returns 0 below 2^-126: an absolute allowance of that size, in scale units


def dino_teacher(t, center, temp):
    """softmax((t − center) / temp) per row -> (probs, scale)"""
    z = (t.double() - center.double()) / f32(temp)
    lse = torch.logsumexp(z, 1, keepdim=True)
    p = torch.exp(z - lse)
    return p, p * (1 + z.abs() + lse.abs()) + FTZ


def dino_student(s, tprobs, t0, t1, w, temp):
    """dino_student_kernel: z = s/τ, the teacher rows of row r are those of t0[r], t1[r] that are ≥ 0 (t1 None: none),
    n = their count, T = their sum:  ds = (w/τ)(n·softmax(z) − T),  loss = Σ_r w (n·lse(z) − T·z)
    -> dict(ds, ds_scale, loss, loss_abs)"""
    it = 1.0 / f32(temp)
    z = s.double() * it
    tp = tprobs.double()
    R = s.shape[0]
    T = torch.zeros_like(z)
    n = torch.zeros(R, 1, dtype=torch.float64, device=z.device)
    for idx in (t0, t1):
        if idx is None:
            continue
        idx = idx.long()
        have = (idx >= 0)[:, None]
        T = T + torch.where(have, tp[idx.clamp(min=0)], torch.zeros_like(T))
        n = n + have.double()
    lse = torch.logsumexp(z, 1, keepdim=True)
    p = torch.exp(z - lse)
    wr = w.double()[:, None]
    ds = wr * it * (n * p - T)
    ds_scale = (wr * it).abs() * (n * (p * (1 + z.abs() + lse.abs()) + FTZ) + T)
    loss = (wr * (n * lse - (T * z).sum(1, keepdim=True))).sum()
    loss_abs = (wr.abs() * (n * (lse.abs() + z.abs().amax(1, keepdim=True)) + (T * z).abs().sum(1, keepdim=True))).sum()
    return dict(ds=ds, ds_scale=ds_scale, loss=loss, loss_abs=loss_abs)


def recon_l1(rec, tgt, dlp, coef, r):
    """L1 gradient coef·sign(rec − tgt) (+ dlp), pixel-unshuffled to [B·gh·gw, C·r·r], and the loss coef Σ|rec − tgt|
    -> (out, loss, loss_abs)"""
    d = rec.double() - tgt.double()
    g = coef * torch.sign(d) + (0 if dlp is None else dlp.double())
    B, C, H, W = rec.shape
    out = torch.nn.functional.pixel_unshuffle(g, r).permute(0, 2, 3, 1).reshape(B * (H // r) * (W // r), C * r * r)
    return out, coef * d.abs().sum(), abs(coef) * d.abs().sum()


# ------------------------------------------------------------------------------------------------------------- LPIPS

def _lp(c, dev):
    sh = torch.tensor([f32(v) for v in LP_SHIFT], dtype=torch.float64, device=dev)
    sc = torch.tensor([f32(v) for v in LP_SCALE], dtype=torch.float64, device=dev)
    return sh.view(1, 3, 1, 1), sc.view(1, 3, 1, 1)


def lpips_prep(img):
    """ScalingLayer then the 3x3 im2col of NCHW img: out [B·H·W, 32], k = tap·3 + c (tap = 3·dy + dx over the window
    rows dy, columns dx around the pixel, zero outside the image), columns 27..31 zero"""
    B, _, H, W = img.shape
    sh, sc = _lp(3, img.device)
    v = (img.double() - sh) / sc
    vp = torch.nn.functional.pad(v, (1, 1, 1, 1))
    out = torch.zeros(B, H, W, 32, dtype=torch.float64, device=img.device)
    for tap in range(9):
        dy, dx = divmod(tap, 3)
        out[..., tap * 3:tap * 3 + 3] = vp[:, :, dy:dy + H, dx:dx + W].permute(0, 2, 3, 1)
    return out.reshape(B * H * W, 32)


def maxpool2(x):
    """2x2 max pool of NHWC x [B, H, W, C]"""
    B, H, W, C = x.shape
    return x.double().reshape(B, H // 2, 2, W // 2, 2, C).amax((2, 4))


def pool_relu_bwd(y, dpool, gtap):
    """dz = (gtap + [this position is the FIRST maximum of its 2x2 window in row-major order (0,0), (0,1), (1,0), (1,1)]
    · dpool) · [y > 0], NHWC; the first maximum is the position k with y_k > y_j for every j < k and y_k ≥ y_j for every
    j > k"""
    B, H, W, C = y.shape
    win = y.double().reshape(B, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 5, 2, 4).reshape(B, H // 2, W // 2, C, 4)
    arg = torch.zeros(win.shape[:-1], dtype=torch.long, device=y.device)
    best = win[..., 0]
    for k in range(1, 4):
        take = win[..., k] > best            # strictly greater: a tie keeps the earlier position
        arg = torch.where(take, k, arg)
        best = torch.where(take, win[..., k], best)
    route = torch.nn.functional.one_hot(arg, 4).double() * dpool.double()[..., None]
    route = route.reshape(B, H // 2, W // 2, C, 2, 2).permute(0, 1, 4, 2, 5, 3).reshape(B, H, W, C)
    g = route + (0 if gtap is None else gtap.double())
    return torch.where(y.double() > 0, g, torch.zeros_like(g))


def lpips_tap(f0, f1, w, coef):
    """per pixel p: n = f / (‖f‖ + 1e-10), d_p = Σ_c w_c (n0_c − n1_c)²; loss = coef Σ_p d_p, g0 = coef ∂d/∂f0 masked by
    f0 > 0 (f0 is a ReLU output): g0 = gn/(r+ε) − f0 (gn·f0)/(r (r+ε)²), gn = 2 coef w (n0 − n1)
    -> dict(g0, g0_scale, loss, loss_abs)"""
    a, b, wd = f0.double(), f1.double(), w.double()
    r0, r1 = a.norm(dim=1, keepdim=True), b.norm(dim=1, keepdim=True)
    i0, i1 = 1 / (r0 + f32(1e-10)), 1 / (r1 + f32(1e-10))
    n0, n1 = a * i0, b * i1
    diff = n0 - n1
    d = (wd * diff * diff).sum(1)
    gn = 2 * coef * wd * diff
    dot = (gn * a).sum(1, keepdim=True)
    k2 = dot * i0 * i0 / r0.clamp(min=f32(1e-20))
    g = torch.where(a > 0, gn * i0 - a * k2, torch.zeros_like(a))
    scale = (gn.abs() * i0 + a.abs() * (gn * a).abs().sum(1, keepdim=True) * i0 * i0 / r0.clamp(min=f32(1e-20))) \
        * (1 + a.shape[1] ** 0.5)
    return dict(g0=g, g0_scale=scale, loss=coef * d.sum(),
                loss_abs=abs(coef) * (wd.abs() * (n0.abs() + n1.abs()) ** 2).sum())


def lpips_img_grad(dcol, B, H, W):
    """col2im of dcol [B·H·W, 32] (k = tap·3 + c) divided by the ScalingLayer scale -> (dimg NCHW [B, 3, H, W], scale):
    dimg[b, c, h, w] = Σ_tap dcol[b, h − dy + 1, w − dx + 1, tap·3 + c] / scale_c (the output pixel (h', w') read input
    (h' + dy − 1, w' + dx − 1) with tap (dy, dx))"""
    cols = dcol.double().reshape(B, H, W, 32)
    acc = torch.zeros(B, H + 2, W + 2, 3, dtype=torch.float64, device=dcol.device)
    aab = torch.zeros_like(acc)
    for tap in range(9):
        dy, dx = divmod(tap, 3)
        acc[:, dy:dy + H, dx:dx + W] += cols[..., tap * 3:tap * 3 + 3]
        aab[:, dy:dy + H, dx:dx + W] += cols[..., tap * 3:tap * 3 + 3].abs()
    _, sc = _lp(3, dcol.device)
    crop = lambda t: t[:, 1:H + 1, 1:W + 1].permute(0, 3, 1, 2) / sc
    return crop(acc), crop(aab)


# ------------------------------------------------------------------------------------------------------------- AdamW

def adamw(p, m, v, g, *, lr, b1, b2, eps, wd, step, grad_scale, teacher=None, mom=None, bc=None):
    """one adamw_kernel step in fp64 from the fp32 state; bias corrections 1 − β^step, or bc = (bc1, bc2) as the kernel
    reads them from `hyper` (hyper_tick forms 1 − β2^step in fp32, which cancels: ~2^-24 absolute against 1 − β2^step of
    order 1e-3 at β2 = 0.999, so the kernel's input differs from the fp64 value by up to ~3e-5 relative):
        ĝ = grad_scale·g,  m = β1 m + (1 − β1) ĝ,  v = β2 v + (1 − β2) ĝ²
        p = p − lr (m/(1 − β1^step) / (sqrt(v/(1 − β2^step)) + eps) + wd·p),  teacher = mom·teacher + (1 − mom)·p
    -> dict(p, m, v, teacher, p_scale, t_scale)"""
    b1, b2, lr, eps, wd = f32(b1), f32(b2), f32(lr), f32(eps), f32(wd)
    gh = f32(grad_scale) * g.double()
    m = b1 * m.double() + (1 - b1) * gh
    v = b2 * v.double() + (1 - b2) * gh * gh
    bc1, bc2 = bc if bc is not None else (1 - b1 ** step, 1 - b2 ** step)
    u = (m / bc1) / (torch.sqrt(v / bc2) + eps)
    p0 = p.double()
    p = p0 - lr * (u + wd * p0)
    out = dict(p=p, m=m, v=v, p_scale=p0.abs() + lr * (u.abs() + wd * p0.abs()), m_scale=m.abs() + gh.abs(),
               v_scale=v.abs() + gh * gh)
    if teacher is not None:
        mom = f32(mom)
        out["teacher"] = mom * teacher.double() + (1 - mom) * p
        out["t_scale"] = teacher.double().abs() + p.abs()
    return out
