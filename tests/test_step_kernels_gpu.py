"""The training step's memory-bound and loss kernels against the fp64 references of tests/step_ref.py, at the
benchmark's shapes and on every branch of their host dispatch.  Each case names the branch it exists for.

- Outputs go into NaN-filled buffers with sentinel rows (and, where the kernel takes a row stride, sentinel columns)
  on both sides; bias-gradient / column-sum vectors are zeroed slices of a NaN buffer, so a float4 atomic of an
  inactive column group, or any stray write, shows up as a changed sentinel.
- Integer-valued inputs make every fp32 sum exact in any order: cast_colsum, norm_bwd's db, scatter_add_rows,
  scatter_add_images, gather_images and strip_prefix must then match bit for bit, which is what catches a dropped or
  doubled strip at M = 131 584.
- Row counts that cross a persistent-grid boundary are computed from the device's SM count.
- Every reduction is launched twice: the non-atomic outputs must be bit-identical, the atomic ones (column sums, loss
  accumulators) are reported against their bound.

Bounds are tests/step_ref.py's; its header lists the maxima measured on an H100 behind each of them.  Runtime on one
H100 80GB HBM3 (700 W): 21 s for the 74 cases.
"""
import math

import pytest
import torch

from tests import step_ref as sr
from vtp_b200 import lib

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
NAN = float("nan")
S = 3  # sentinel rows / columns on each side


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


class Checks:
    """collects every measured k of a case, prints it against its bound, and fails at the end if any is over"""

    def __init__(self, case):
        self.case, self.bad = case, []

    def k(self, name, k, bound):
        print(f"[{self.case}] {name}: k = {k:.3g} (bound {bound:g})")
        if not k <= bound:
            self.bad.append((name, k, bound))

    def exact(self, name, got, ref):
        ok = torch.equal(got, ref)
        print(f"[{self.case}] {name}: {'bit-exact' if ok else 'DIFFERS'}")
        if not ok:
            self.bad.append((name, "not bit-exact", None))

    def done(self):
        assert not self.bad, (self.case, self.bad)


def _rows(M, N, dtype, init=None):
    """(buffer with S NaN sentinel rows above and below, contiguous view of the M inner rows)"""
    buf = torch.full((M + 2 * S, N), NAN, device="cuda", dtype=dtype)
    inner = buf[S:S + M]
    if init is not None:
        inner.copy_(init)
    return buf, inner


def _rows_intact(buf):
    return bool(torch.isnan(buf[:S].float()).all() and torch.isnan(buf[-S:].float()).all())


def _vec(n):
    """(NaN buffer, zeroed 16-byte-aligned slice of n floats inside it)"""
    buf = torch.full((n + 8,), NAN, device="cuda")
    buf[4:4 + n] = 0
    return buf, buf[4:4 + n]


def _vec_intact(buf):
    return bool(torch.isnan(buf[:4]).all() and torch.isnan(buf[-4:]).all())


def _ints(shape, lo, hi, g, dtype=torch.float32):
    return torch.randint(lo, hi + 1, shape, device="cuda", generator=g).to(dtype)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# ----------------------------------------------------------------------------------------------------- norm backward

NORM_CASES = {  # name: (M as a function of the SM count n, D, LayerNorm, bf16 x)
    "persistent two strips per block, MAXV 3": (lambda n: 32 * 3 * n + 1, 384, False, False),
    "MAXV 4 (384 < D <= 512), LayerNorm, bf16 x": (lambda n: 32 * 3 * n + 1, 512, True, True),
    "MAXV 16 (D > 1024), two strips per block": (lambda n: 32 * n + 1, 1536, False, False),
    "RMSNorm on bf16 x, D not a multiple of 128": (lambda n: 2000, 200, False, True),
    "benchmark global crops (M 131584, D 384)": (lambda n: 131584, 384, True, False),
    "benchmark local crops (M 75776, D 384), RMSNorm bf16 x": (lambda n: 75776, 384, False, True),
}


@pytest.mark.parametrize("case", list(NORM_CASES))
def test_norm_bwd(case):
    rows, D, ln, xbf = NORM_CASES[case]
    M = rows(_sms())
    g = _gen(M + D)
    x = torch.randn(M, D, device="cuda", generator=g) * 1.5 + 0.2
    x = x.to(BF) if xbf else x
    w = torch.randn(D, device="cuda", generator=g)
    b = torch.randn(D, device="cuda", generator=g) if ln else None
    # LayerNorm: integer-valued dy, so that db = Σ dy is exact in any summation order
    dy = (_ints((M, D), -4, 4, g) if ln else torch.randn(M, D, device="cuda", generator=g)).to(BF)
    g0 = torch.randn(M, D, device="cuda", generator=g)
    rstd = torch.empty(M, device="cuda")
    mean = torch.empty(M, device="cuda") if ln else None
    y = torch.empty(M, D, device="cuda", dtype=BF)
    lib.norm_fwd(x, y, w, b, 1e-6 if ln else 1e-5, M, D, y_mode=lib.OUT_BF16, rstd=rstd, mean=mean)
    ref = sr.norm_bwd(x, rstd, mean, w, dy, g0)
    chk = Checks(case)
    first = None
    for rep in range(2):
        gbuf, gin = _rows(M, D, torch.float32, g0)
        bbuf, gb = _rows(M, D, BF)
        dwb, dw = _vec(D)
        dbb, db = _vec(D) if ln else (None, None)
        gsb, gs = _vec(D)
        lib.norm_bwd(x, rstd, mean, w, dy, gin, dw, db, M, D, gb_out=gb, g_colsum=gs)
        torch.cuda.synchronize()
        assert _rows_intact(gbuf) and _rows_intact(bbuf) and _vec_intact(dwb) and _vec_intact(gsb)
        assert not ln or _vec_intact(dbb)
        chk.k(f"g (rep {rep})", sr.elem_k(gin, ref["g"], ref["g_scale"], ulps=0), sr.NORM_G_K)
        chk.exact(f"g_bf16_out (rep {rep})", gb, gin.to(BF))
        chk.k(f"dw (rep {rep})", sr.col_k(dw, ref["dw"], ref["dw_abs"]), sr.COL_K)
        chk.k(f"g_colsum (rep {rep})", sr.col_k(gs, gin.double().sum(0), gin.double().abs().sum(0)), sr.COL_K)
        if ln:
            chk.exact(f"db (rep {rep})", db, ref["db"].float())
        if first is None:
            first = gin.clone()
        else:
            chk.exact("g repeat", gin, first)
    chk.done()


# ------------------------------------------------------------------------------------------------------ norm forward

@pytest.mark.parametrize("D,ln,xbf,ldx", [(1536, False, False, 1536 + 64), (1536, True, True, 1536), (1536, False, True, 1600),
                                         (384, True, False, 392), (200, False, True, 256)])
def test_norm_fwd(D, ln, xbf, ldx):
    """MAXV 16 (D > 1024) and a row stride ldx != D (NaN in the pad columns), both output modes"""
    M = 3000
    g = _gen(D + ldx)
    xs = torch.full((M, ldx), NAN, device="cuda")
    xs[:, :D] = torch.randn(M, D, device="cuda", generator=g) * 2 + 0.3
    xs = xs.to(BF) if xbf else xs
    x = xs[:, :D]
    w = torch.randn(D, device="cuda", generator=g)
    b = torch.randn(D, device="cuda", generator=g) if ln else None
    eps = 1e-6 if ln else 1e-5
    chk = Checks(f"norm_fwd D={D} ln={ln} bf16x={xbf} ldx={ldx}")
    rstd, mean = torch.empty(M, device="cuda"), torch.empty(M, device="cuda")
    y32b, y32 = _rows(M, D, torch.float32)
    lib.norm_fwd(xs, y32, w, b, eps, M, D, y_mode=lib.OUT_F32, ldx=ldx, rstd=rstd, mean=mean)
    y16b, y16 = _rows(M, D, BF)
    lib.norm_fwd(xs, y16, w, b, eps, M, D, y_mode=lib.OUT_BF16, ldx=ldx)
    y16r = torch.empty_like(y16)
    lib.norm_fwd(xs, y16r, w, b, eps, M, D, y_mode=lib.OUT_BF16, ldx=ldx)
    torch.cuda.synchronize()
    assert _rows_intact(y32b) and _rows_intact(y16b)
    ref, rstd_ref, mean_ref, scale = sr.norm_fwd(x, w, b, eps, rstd_kernel=rstd)
    chk.k("rstd", sr.elem_k(rstd, rstd_ref, rstd_ref, ulps=0), sr.NORM_FWD_K)
    if ln:
        chk.k("mean", sr.elem_k(mean, mean_ref, x.double().abs().mean(1) * D ** 0.5, ulps=0), sr.NORM_FWD_K)
    chk.k("y fp32", sr.elem_k(y32, ref, scale, ulps=0), sr.NORM_FWD_K)
    chk.k("y bf16", sr.elem_k(y16, ref, scale), sr.NORM_FWD_K)
    chk.exact("y bf16 repeat", y16r, y16)
    chk.done()


# -------------------------------------------------------------------------------------------------- SwiGLU / GELU

ACT_CASES = {  # name: (kind, M as a function of the SM count n, width, dbias); gy_cap = 2n / column blocks
    "swiglu Hs 2048: two column blocks, several row passes": ("swiglu", lambda n: 8 * 4 * n + 3, 2048, True),
    "swiglu Hs 2736: ragged last column block": ("swiglu", lambda n: 4 * n + 7, 2736, True),
    "swiglu benchmark (M 131584, Hs 1024)": ("swiglu", lambda n: 131584, 1024, True),
    "swiglu dbias NULL": ("swiglu", lambda n: 1000, 1024, False),
    "gelu DINO head N 2048: two column blocks, several row passes": ("gelu", lambda n: 8 * 4 * n + 3, 2048, True),
    "gelu N 1000: one ragged column block": ("gelu", lambda n: 4 * n + 1, 1000, True),
    "gelu dbias NULL": ("gelu", lambda n: 999, 768, False),
}


@pytest.mark.parametrize("case", list(ACT_CASES))
def test_swiglu_gelu(case):
    kind, rows, Wd, with_db = ACT_CASES[case]
    M = rows(_sms())
    g = _gen(M + Wd)
    Np = 2 * Wd if kind == "swiglu" else Wd
    pre = (torch.randn(M, Np, device="cuda", generator=g) * 2).to(BF)
    dh = torch.randn(M, Wd, device="cuda", generator=g).to(BF)
    if kind == "swiglu":
        ref, scale, dbr, dba = sr.swiglu_bwd(pre, dh, Wd)
    else:
        ref, scale, dbr, dba = sr.gelu_bwd(pre, dh)
    chk = Checks(case)
    first = None
    for rep in range(2):
        ob, out = _rows(M, Np, BF)
        vb, dbias = _vec(Np) if with_db else (None, None)
        (lib.swiglu_bwd if kind == "swiglu" else lib.gelu_bwd)(pre, dh, out, dbias, M, Wd)
        torch.cuda.synchronize()
        assert _rows_intact(ob)
        chk.k(f"dpre (rep {rep})", sr.elem_k(out, ref, scale), sr.ACT_K)
        if with_db:
            assert _vec_intact(vb)
            chk.k(f"dbias (rep {rep})", sr.col_k(dbias, dbr, dba), sr.COL_K)
        if first is None:
            first = out.clone()
        else:
            chk.exact("dpre repeat", out, first)
    if kind == "swiglu":
        hb, hid = _rows(M, Wd, BF)
        lib.swiglu_fwd(pre, hid, M, Wd)
        hid2 = torch.empty_like(hid)
        lib.swiglu_fwd(pre, hid2, M, Wd)
        torch.cuda.synchronize()
        assert _rows_intact(hb)
        href, halt, hscale = sr.swiglu_fwd(pre, Wd)
        href = torch.where((hid.double() - halt).abs() < (hid.double() - href).abs(), halt, href)
        # the reference is already rounded twice, as the kernel rounds, and the kernel's product of two bf16 values
        # is exact in fp32: no ulp of slack, so a missing or non-nearest rounding shows up
        chk.k("swiglu_fwd hid", sr.elem_k(hid, href, hscale, ulps=0), sr.ACT_K)
        chk.exact("swiglu_fwd repeat", hid2, hid)
    chk.done()


# ------------------------------------------------------------------------------------------------------ cast_colsum

def _cc_cap(n, N):
    """vtp_cast_colsum's gy_cap: about 4 resident blocks per SM over the column blocks of 128 x 4 columns"""
    gx = -(-(N // 4) // 128)
    return -(-4 * n // gx)


CC_CASES = {  # name: (M as a function of the SM count n, N, dtype, ldx, with y, integer inputs)
    "fp32, more strips than gy_cap, ldx > N": (lambda n: 64 * _cc_cap(n, 384) + 65, 384, torch.float32, 392, True, True),
    "bf16 K 65536 teacher-centre sums, y NULL, more strips than gy_cap":
        (lambda n: 64 * _cc_cap(n, 65536) + 64, 65536, BF, 65536, False, True),
    "bf16 with y, ldx > N": (lambda n: 1000, 768, BF, 800, True, True),
    "benchmark decoder (M 65536, N 768) fp32": (lambda n: 65536, 768, torch.float32, 768, True, True),
    "fp32 non-integer inputs": (lambda n: 20000, 1152, torch.float32, 1152, True, False),
}


@pytest.mark.parametrize("case", list(CC_CASES))
def test_cast_colsum(case):
    rows, N, dt, ldx, with_y, exact = CC_CASES[case]
    M = rows(_sms())
    g = _gen(M + N)
    xs = torch.full((M, ldx), NAN, device="cuda")
    xs[:, :N] = _ints((M, N), -8, 8, g) if exact else torch.randn(M, N, device="cuda", generator=g)
    xs = xs.to(dt)
    x = xs[:, :N]
    chk = Checks(case)
    for rep in range(2):
        yb, y = _rows(M, N, BF) if with_y else (None, None)
        vb, cs = _vec(N)
        lib.cast_colsum(xs, y, cs, M, N, ldx=ldx)
        torch.cuda.synchronize()
        assert _vec_intact(vb)
        if with_y:
            assert _rows_intact(yb)
            chk.exact(f"y (rep {rep})", y, x.to(BF))
        if exact:
            chk.exact(f"colsum (rep {rep})", cs, x.double().sum(0).float())
        else:
            chk.k(f"colsum (rep {rep})", sr.col_k(cs, x.double().sum(0), x.double().abs().sum(0)), sr.COL_K)
    chk.done()


# ----------------------------------------------------------------------------------- scatter / gather / strip_prefix

@pytest.mark.parametrize("src_dt", [torch.float32, BF])
def test_scatter_add_rows_exact(src_dt):
    """duplicate indices, ld_src and ld_dst wider than D (pad columns NaN and untouched); launched twice"""
    n, D, rows, lds, ldd = 5000, 384, 300, 400, 392
    g = _gen(7)
    src = torch.full((n, lds), NAN, device="cuda")
    src[:, :D] = _ints((n, D), -16, 16, g)
    src = src.to(src_dt)
    dst0 = torch.full((rows, ldd), NAN, device="cuda")
    dst0[:, :D] = _ints((rows, D), -100, 100, g)
    idx = torch.randint(0, rows // 3, (n,), device="cuda", generator=g)   # every target row hit many times
    ref = dst0[:, :D].double().index_add(0, idx, src[:, :D].double())
    for _ in range(2):
        dst = dst0.clone()
        lib.scatter_add_rows(src, dst, idx, D, ld_src=lds, ld_dst=ldd)
        torch.cuda.synchronize()
        assert torch.equal(dst[:, :D], ref.float()) and torch.isnan(dst[:, D:]).all()


@pytest.mark.parametrize("src_dt", [torch.float32, BF])
def test_scatter_gather_images_exact(src_dt):
    """stochastic-depth image subsets at the benchmark's token shape (T 257, D 384), alpha 1 and a power of two"""
    B, T, D, n = 64, 257, 384, 37
    g = _gen(8)
    x = _ints((B * T, D), -50, 50, g)
    idx = torch.randperm(B, device="cuda", generator=g)[:n]
    for alpha in (1.0, 0.5):
        ob, out = _rows(n * T, D, torch.float32)
        lib.gather_images(x, out, idx, T, D, alpha)
        torch.cuda.synchronize()
        assert _rows_intact(ob)
        assert torch.equal(out, alpha * x.view(B, T, D)[idx].reshape(n * T, D))
    src = _ints((n * T, D), -50, 50, g).to(src_dt)
    ref = x.view(B, T, D).double().index_add(0, idx, src.view(n, T, D).double()).reshape(B * T, D)
    for _ in range(2):
        db, dst = _rows(B * T, D, torch.float32, x)
        lib.scatter_add_images(src, dst, idx, T, D, 1.0)
        torch.cuda.synchronize()
        assert _rows_intact(db) and torch.equal(dst, ref.float())


@pytest.mark.parametrize("prefix", [1, 4])
def test_strip_prefix_exact(prefix):
    B, HW, D = 256, 256, 384
    T = HW + prefix
    g = _gen(prefix)
    gr = _ints((B * T, D), -64, 64, g)
    v = gr.view(B, T, D)
    for _ in range(2):  # dcls is an atomic column sum, exact in any order on integer-valued input
        ob, out = _rows(B * HW, D, BF)
        vb, dcls = _vec(prefix * D)
        lib.strip_prefix(gr, out, dcls, B, T, prefix, D)
        torch.cuda.synchronize()
        assert _rows_intact(ob) and _vec_intact(vb)
        assert torch.equal(out, v[:, prefix:].reshape(B * HW, D).to(BF))
        assert torch.equal(dcls.view(prefix, D), v[:, :prefix].double().sum(0).float())


# ---------------------------------------------------------------------------------------------------- softmax_ce

@pytest.mark.parametrize("C,log_scale", [(96, True), (96, False), (256, True), (2048, True)])
def test_softmax_ce(C, log_scale):
    """the contrastive loss as train.py calls it: log_scale = log 100, label0 = rank·B of a world of 4, padded ld / ldg
    (pad columns NaN in the logits and untouched in G), C up to 8x the 256-thread block"""
    world, rank = 4, 2
    R, label0 = C // world, rank * (C // world)
    ld, ldg = C + 8, C + 16
    g = _gen(C)
    lg = torch.full((R, ld), NAN, device="cuda")
    lg[:, :C] = (torch.randn(R, C, device="cuda", generator=g) * 0.3).clamp(-1, 1)
    lg[torch.arange(R), label0 + torch.arange(R)] += 0.5
    ls = torch.tensor([math.log(100.0)], device="cuda") if log_scale else None
    coef = 0.5 / C
    ref = sr.softmax_ce(lg, C, label0, coef, ls.item() if log_scale else None)
    chk = Checks(f"softmax_ce C={C} log_scale={log_scale}")
    first = None
    for rep in range(2):
        Gb = torch.full((R + 2 * S, ldg), NAN, device="cuda", dtype=BF)
        G = Gb[S:S + R]
        acc = torch.zeros(2, device="cuda")
        lib.softmax_ce(lg, R, C, label0, G, coef, acc[0:1], acc[1:2], log_scale=ls)
        torch.cuda.synchronize()
        assert _rows_intact(Gb) and torch.isnan(G[:, C:].float()).all()
        chk.k(f"G (rep {rep})", sr.elem_k(G[:, :C], ref["G"], ref["G_scale"]), sr.CE_K)
        chk.k(f"loss (rep {rep})", sr.col_k(acc[0], ref["loss"], ref["loss_abs"]), sr.CE_SUM_K)
        chk.k(f"dscale (rep {rep})", sr.col_k(acc[1], ref["dscale"], ref["dscale_abs"]), sr.CE_SUM_K)
        if first is None:
            first = G.clone()
        else:
            chk.exact("G repeat", G[:, :C], first[:, :C])
    chk.done()


# --------------------------------------------------------------------------------------------------------- DINO / iBOT

def _teacher(K, R, temp, g):
    t = (torch.randn(R, K, device="cuda", generator=g) * 10).clamp(-30, 30).to(BF)
    center = torch.randn(K, device="cuda", generator=g) * 0.5
    tb, tin = _rows(R, K, BF, t)
    lib.dino_teacher_probs(tin, center, R, K, temp)
    torch.cuda.synchronize()
    assert _rows_intact(tb)
    return t, center, tin


@pytest.mark.parametrize("K", [8, 1000, 4096, 65536, 112640])
@pytest.mark.parametrize("temp", [0.04, 0.07])
def test_dino_teacher(K, temp):
    """K = 65 536 is the benchmark's smem-resident row, 112 640 the largest the 220 KB check admits; logits to ±30"""
    g = _gen(K)
    t, center, tp = _teacher(K, 6, temp, g)
    p, scale = sr.dino_teacher(t, center, temp)
    chk = Checks(f"dino_teacher K={K} temp={temp}")
    chk.k("probs", sr.elem_k(tp, p, scale), sr.DINO_K)
    again = t.clone()
    lib.dino_teacher_probs(again, center, 6, K, temp)
    chk.exact("probs repeat", again, tp)
    chk.done()


def _student_run(s, tp, t0, t1, w, K, temp):
    R = s.shape[0]
    sb, sin = _rows(R, K, BF, s)
    acc = torch.zeros(1, device="cuda")
    lib.dino_student_ce(sin, tp, t0, t1, w, R, K, temp, acc)
    torch.cuda.synchronize()
    assert _rows_intact(sb)
    return sin, acc[0]


@pytest.mark.parametrize("K", [8, 1000, 4096, 65536, 112640])
@pytest.mark.parametrize("with_t1", [True, False])
def test_dino_student(K, with_t1):
    """rows with two teachers, one (t0 only), none (t0 = t1 = −1: zero loss and gradient); t1 = NULL"""
    g = _gen(K + 1)
    _, _, tp = _teacher(K, 5, 0.04, g)
    R = 12
    s = (torch.randn(R, K, device="cuda", generator=g) * 5).to(BF)
    t0 = torch.tensor([0, 1, 2, 3, 4, -1, 0, 1, -1, 2, 3, 4], device="cuda", dtype=torch.int32)
    t1 = torch.tensor([1, -1, 3, 4, 0, -1, 2, -1, -1, 1, -1, 3], device="cuda", dtype=torch.int32) if with_t1 else None
    w = torch.rand(R, device="cuda", generator=g) + 0.1
    ref = sr.dino_student(s, tp, t0, t1, w, 0.1)
    chk = Checks(f"dino_student K={K} t1={'set' if with_t1 else 'NULL'}")
    ds, loss = _student_run(s, tp, t0, t1, w, K, 0.1)
    chk.k("ds", sr.elem_k(ds, ref["ds"], ref["ds_scale"]), sr.DINO_K)
    chk.k("loss", sr.col_k(loss, ref["loss"], ref["loss_abs"]), sr.DINO_K)
    ds2, loss2 = _student_run(s, tp, t0, t1, w, K, 0.1)
    chk.exact("ds repeat", ds2, ds)
    chk.k("loss repeat", sr.col_k(loss2, ref["loss"], ref["loss_abs"]), sr.DINO_K)
    assert (ds[5] == 0).all() and (ds[8] == 0).all()
    chk.done()


@pytest.mark.parametrize("K", [4096, 65536])
def test_dino_student_lone_second_teacher(K):
    """t0 = −1, t1 ≥ 0: the row learns from teacher t1 alone, as if that index were in t0"""
    g = _gen(K + 2)
    _, _, tp = _teacher(K, 3, 0.04, g)
    s = (torch.randn(4, K, device="cuda", generator=g) * 5).to(BF)
    t0 = torch.tensor([-1, 0, -1, 2], device="cuda", dtype=torch.int32)
    t1 = torch.tensor([2, -1, 1, 1], device="cuda", dtype=torch.int32)
    w = torch.rand(4, device="cuda", generator=g) + 0.1
    ref = sr.dino_student(s, tp, t0, t1, w, 0.1)
    chk = Checks(f"dino_student lone t1 K={K}")
    ds, loss = _student_run(s, tp, t0, t1, w, K, 0.1)
    chk.k("ds", sr.elem_k(ds, ref["ds"], ref["ds_scale"]), sr.DINO_K)
    chk.k("loss", sr.col_k(loss, ref["loss"], ref["loss_abs"]), sr.DINO_K)
    chk.done()


def test_dino_smem_limit():
    """K = 112 648 needs more than the 220 KB smem-resident row: both kernels refuse it on the host"""
    K = 112648
    t = torch.zeros(1, K, device="cuda", dtype=BF)
    c = torch.zeros(K, device="cuda")
    i = torch.zeros(1, device="cuda", dtype=torch.int32)
    with pytest.raises(lib.VtpError, match="too large"):
        lib.dino_teacher_probs(t, c, 1, K, 0.04)
    with pytest.raises(lib.VtpError, match="too large"):
        lib.dino_student_ce(t, t, i, None, c[:1], 1, K, 0.1, c[:1])


# ------------------------------------------------------------------------------------------------------- recon L1

@pytest.mark.parametrize("rec_dt,with_dlp,B", [(BF, True, 2), (torch.float32, False, 2), (torch.float32, True, 3),
                                               (BF, True, 256)])
def test_recon_l1(rec_dt, with_dlp, B):
    """pixels with rec == tgt (sign 0), both rec dtypes, the LPIPS gradient dlp; B 256 = the benchmark's 65 536
    decoder rows of N 768"""
    C, gh, gw, r = 3, 16, 16, 16
    g = _gen(B)
    rec = torch.randn(B, C, gh * r, gw * r, device="cuda", generator=g).to(rec_dt)
    tgt = rec.float().clone()
    tgt[:, :, 1::2] += torch.randn(B, C, gh * r // 2, gw * r, device="cuda", generator=g)
    dlp = torch.randn(B, C, gh * r, gw * r, device="cuda", generator=g) * 1e-6 if with_dlp else None
    coef = 1.0 / rec.numel()
    ref, lref, labs = sr.recon_l1(rec, tgt, dlp, coef, r)
    chk = Checks(f"recon_l1 {rec_dt} dlp={with_dlp} B={B}")
    scale = coef
    if dlp is not None:  # the fp32 sum coef·sign + dlp: terms |coef| + |dlp|, in the output's pixel-unshuffled order
        scale = coef + torch.nn.functional.pixel_unshuffle(dlp.double().abs(), r).permute(0, 2, 3, 1).reshape(ref.shape)
    first = None
    for rep in range(2):
        ob, out = _rows(B * gh * gw, C * r * r, BF)
        acc = torch.zeros(1, device="cuda")
        lib.recon_l1_grad(rec, tgt, dlp, out, acc, B, C, gh, gw, r, coef)
        torch.cuda.synchronize()
        assert _rows_intact(ob)
        chk.k(f"out (rep {rep})", sr.elem_k(out, ref, scale), sr.ACT_K)
        chk.k(f"loss (rep {rep})", sr.col_k(acc[0], lref, labs), sr.LOSS_K)
        if first is None:
            first = out.clone()
        else:
            chk.exact("out repeat", out, first)
    if dlp is None:
        zero = sr.recon_l1(rec, tgt, None, 1.0, r)[0] == 0
        assert zero.any() and (out[zero] == 0).all()
    chk.done()


# ------------------------------------------------------------------------------------------------------------ LPIPS

@pytest.mark.parametrize("img_dt", [torch.float32, BF])
def test_lpips_prep(img_dt):
    """ScalingLayer + 3x3 im2col with zero borders on a non-square image, fp32 and bf16 input"""
    B, H, W = 3, 20, 33
    img = (torch.rand(B, 3, H, W, device="cuda", generator=_gen(1)) * 2 - 1).to(img_dt)
    ob, out = _rows(B * H * W, 32, BF)
    lib.lpips_prep(img, out, B, H, W)
    torch.cuda.synchronize()
    assert _rows_intact(ob)
    ref = sr.lpips_prep(img)
    chk = Checks(f"lpips_prep {img_dt}")
    chk.k("im2col", sr.elem_k(out, ref, ref.abs()), sr.LPIPS_K)
    chk.done()


def test_maxpool2_exact():
    B, H, W, C = 2, 24, 18, 64
    x = torch.randn(B, H, W, C, device="cuda", generator=_gen(2)).to(BF)
    ob, y = _rows(B * (H // 2) * (W // 2), C, BF)
    lib.maxpool2_fwd(x, y, B, H, W, C)
    torch.cuda.synchronize()
    assert _rows_intact(ob) and torch.equal(y, sr.maxpool2(x).to(BF).reshape(-1, C))


@pytest.mark.parametrize("with_gtap", [True, False])
@pytest.mark.parametrize("C", [64, 128])
def test_pool_relu_bwd_ties(with_gtap, C):
    """bf16 activations drawn from a few values, so that most 2x2 windows hold tied maxima (and zero / negative ones
    the ReLU masks): the pooled gradient goes to the first maximum in row-major order"""
    B, H, W = 2, 16, 12
    g = _gen(C)
    y = (torch.randint(-2, 4, (B, H, W, C), device="cuda", generator=g).float() * 0.5).to(BF)
    dpool = torch.randn(B, H // 2, W // 2, C, device="cuda", generator=g).to(BF)
    gtap = torch.randn(B, H, W, C, device="cuda", generator=g).to(BF) if with_gtap else None
    ob, dz = _rows(B * H * W, C, BF)
    lib.pool_relu_bwd(y, dpool, gtap, dz, B, H, W, C)
    torch.cuda.synchronize()
    assert _rows_intact(ob)
    ref = sr.pool_relu_bwd(y, dpool, gtap).reshape(-1, C)
    scale = (dpool.double().abs().repeat_interleave(2, 1).repeat_interleave(2, 2)
             + (0 if gtap is None else gtap.double().abs())).reshape(-1, C)
    chk = Checks(f"pool_relu_bwd C={C} gtap={with_gtap}")
    chk.k("dz", sr.elem_k(dz, ref, scale), sr.LPIPS_K)
    chk.done()


@pytest.mark.parametrize("C", [64, 128, 256, 512])
def test_lpips_tap(C):
    """every channel count (pixels per warp 4, 2, 1, 1), P not a multiple of the pixels per warp, dead (all-zero)
    pixels in f0 and in f1"""
    P = 64 * 48 * 2 + 3
    g = _gen(C)
    f0 = torch.relu(torch.randn(P, C, device="cuda", generator=g)).to(BF)
    f1 = torch.relu(torch.randn(P, C, device="cuda", generator=g)).to(BF)
    f0[5::97] = 0
    f1[7::89] = 0
    f1[5] = 0
    w = torch.rand(C, device="cuda", generator=g) * 0.1
    coef = 1.0 / (2 * 64 * 48)
    ref = sr.lpips_tap(f0, f1, w, coef)
    chk = Checks(f"lpips_tap C={C}")
    first = None
    for rep in range(2):
        ob, g0 = _rows(P, C, BF)
        acc = torch.zeros(1, device="cuda")
        lib.lpips_tap(f0, f1, w, g0, P, C, coef, acc)
        torch.cuda.synchronize()
        assert _rows_intact(ob)
        chk.k(f"g0 (rep {rep})", sr.elem_k(g0, ref["g0"], ref["g0_scale"]), sr.LPIPS_K)
        chk.k(f"loss (rep {rep})", sr.col_k(acc[0], ref["loss"], ref["loss_abs"]), sr.LOSS_K)
        assert (g0[5::97] == 0).all()
        if first is None:
            first = g0.clone()
        else:
            chk.exact("g0 repeat", g0, first)
    chk.done()


def test_lpips_img_grad():
    """col2im + ScalingLayer backward with borders on a non-square image; dcol's pad columns 27..31 are not read"""
    B, H, W = 3, 20, 33
    dcol = torch.randn(B * H * W, 32, device="cuda", generator=_gen(3)).to(BF)
    ref, scale = sr.lpips_img_grad(dcol, B, H, W)
    chk = Checks("lpips_img_grad")
    first = None
    for rep in range(2):
        buf = torch.full((B + 2, 3, H, W), NAN, device="cuda")
        lib.lpips_img_grad(dcol, buf[1:B + 1], B, H, W)
        torch.cuda.synchronize()
        assert torch.isnan(buf[0]).all() and torch.isnan(buf[-1]).all()
        chk.k(f"dimg (rep {rep})", sr.elem_k(buf[1:B + 1], ref, scale, ulps=0), sr.LPIPS_K)
        if first is None:
            first = buf.clone()
        else:
            chk.exact("dimg repeat", buf[1:B + 1], first[1:B + 1])
    chk.done()


# ------------------------------------------------------------------------------------------------------------ AdamW

def test_adamw_hyper_schedule_ema():
    """six steps of the graph-captured form: hyper_tick reads lr / wd / momentum tables of length 3 (so steps 4-6 hold
    the last entry), adamw_step takes them from `hyper` for a decayed region and an undecayed one (wd = 0 stays 0), with
    grad_scale and the EMA teacher; every step is checked against fp64 from the kernel's own previous state"""
    n_dec, n_nod, steps = 1 << 20, 4096, 6
    b1, b2, eps, gsc = 0.9, 0.999, 1e-8, 0.25
    g = _gen(9)
    lr_tab = torch.tensor([1e-3, 2e-3, 5e-4], device="cuda")
    wd_tab = torch.tensor([0.04, 0.1, 0.2], device="cuda")
    mom_tab = torch.tensor([0.99, 0.995, 0.999], device="cuda")
    hyper = torch.zeros(6, device="cuda")
    regions = []
    for n, wd in ((n_dec, 1.0), (n_nod, 0.0)):
        p = torch.randn(n, device="cuda", generator=g)
        regions.append(dict(n=n, wd=wd, p=p, m=torch.zeros(n, device="cuda"), v=torch.zeros(n, device="cuda"),
                            t=p + 0.01 * torch.randn(n, device="cuda", generator=g), gr=torch.zeros(n, device="cuda"),
                            pb=torch.empty(n, device="cuda", dtype=BF), tb=torch.empty(n, device="cuda", dtype=BF)))
    chk = Checks("adamw hyper")
    for step in range(1, steps + 1):
        lib.hyper_tick(hyper, b1, b2, lr_tab, wd_tab, mom_tab, 3)
        it = min(step, 3) - 1
        bc = (hyper[1].item(), hyper[2].item())   # what adamw_kernel reads; hyper_tick itself is checked below
        for r in regions:
            r["gr"].copy_(torch.randn(r["n"], device="cuda", generator=g) * 1e-2)
            before = {k: r[k].clone() for k in ("p", "m", "v", "t", "gr")}
            lib.adamw_step(r["p"], r["gr"], r["m"], r["v"], r["pb"], r["t"], r["tb"], r["n"], lr=0.0, beta1=b1,
                           beta2=b2, eps=eps, wd=r["wd"], step=0, grad_scale=gsc, ema_momentum=0.0, hyper=hyper)
            torch.cuda.synchronize()
            wd = wd_tab[it].item() if r["wd"] else 0.0
            ref = sr.adamw(before["p"], before["m"], before["v"], before["gr"], lr=lr_tab[it].item(), b1=b1, b2=b2,
                           eps=eps, wd=wd, step=step, grad_scale=gsc, teacher=before["t"], mom=mom_tab[it].item(), bc=bc)
            tag = f"step {step} wd={'sched' if r['wd'] else 0}"
            chk.k(f"p {tag}", sr.elem_k(r["p"], ref["p"], ref["p_scale"], ulps=0), sr.ADAM_K)
            chk.k(f"m {tag}", sr.elem_k(r["m"], ref["m"], ref["m_scale"], ulps=0), sr.ADAM_K)
            chk.k(f"v {tag}", sr.elem_k(r["v"], ref["v"], ref["v_scale"], ulps=0), sr.ADAM_K)
            chk.k(f"teacher {tag}", sr.elem_k(r["t"], ref["teacher"], ref["t_scale"], ulps=0), sr.ADAM_K)
            assert torch.equal(r["pb"], r["p"].to(BF)) and torch.equal(r["tb"], r["t"].to(BF))
            assert (r["gr"] == 0).all()
        h = hyper.tolist()
        assert h[0] == step and h[3] == lr_tab[it].item() and h[4] == wd_tab[it].item() and h[5] == mom_tab[it].item()
        assert abs(h[1] - (1 - b1 ** step)) < 1e-6 and abs(h[2] - (1 - b2 ** step)) < 1e-6
    chk.done()


def test_adamw_host_scalars():
    """the eager form: bias corrections from the host step count, no teacher"""
    n = 65536
    g = _gen(10)
    p = torch.randn(n, device="cuda", generator=g)
    m, v = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    pb = torch.empty(n, device="cuda", dtype=BF)
    chk = Checks("adamw host")
    for step in (1, 2, 3):
        gr = torch.randn(n, device="cuda", generator=g) * 4
        before = (p.clone(), m.clone(), v.clone(), gr.clone())
        lib.adamw_step(p, gr, m, v, pb, None, None, n, lr=1e-2, beta1=0.9, beta2=0.95, eps=1e-8, wd=0.05, step=step,
                       grad_scale=0.25)
        torch.cuda.synchronize()
        ref = sr.adamw(*before, lr=1e-2, b1=0.9, b2=0.95, eps=1e-8, wd=0.05, step=step, grad_scale=0.25)
        chk.k(f"p step {step}", sr.elem_k(p, ref["p"], ref["p_scale"], ulps=0), sr.ADAM_K)
        assert torch.equal(pb, p.to(BF)) and (gr == 0).all()
    chk.done()
