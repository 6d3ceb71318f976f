"""The references of tests/stage_ref.py proved without a GPU: gemm_ref against F.conv2d (and its input gradient through
w_bwd), F.pixel_shuffle, explicit rr_skip row maps, operand majors, ldo and accumulate; the composed LPIPS chain
against fp64 autograd of the LPIPS value; the SSL row lists against their definition.
"""
import pytest
import torch
import torch.nn.functional as F

from tests import stage_ref as st
from tests import step_ref as sr

D64 = torch.float64


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _close(a, b, tol=1e-12):
    a, b = a.double(), b.double()
    assert ((a - b).abs().max() / (b.abs().max() + 1e-300)).item() < tol


def _run(call):
    """gemm_ref over every row, scattered into a copy of `out` as the kernel would store it"""
    rows = torch.arange(call["M"])
    rows = rows[rows % call["rr_group"] >= -call["rr_skip"]] if call.get("rr_skip", 0) < 0 else rows
    out = call["out"].clone().double()
    idx = st.out_index(call, rows)
    out.reshape(-1)[idx.reshape(-1)] = st.gemm_ref(call, rows, call["out"])["out"][0].reshape(-1)
    return out


# ---------------------------------------------------------------------------------------------------------- GEMM

@pytest.mark.parametrize("act", [st.ACT_NONE, st.ACT_RELU])
def test_conv_matches_conv2d(act):
    g = _g(1)
    B, C, Co, H, W = 2, 5, 7, 6, 9
    x = torch.randn(B, C, H, W, generator=g, dtype=D64)
    w = torch.randn(Co, C, 3, 3, generator=g, dtype=D64)
    b = torch.randn(Co, generator=g, dtype=D64)
    ref = F.conv2d(x, w, b, padding=1)
    ref = ref.clamp(min=0) if act == st.ACT_RELU else ref
    out = torch.zeros(B * H * W, Co, dtype=D64)
    call = dict(A=x.permute(0, 2, 3, 1).contiguous(), B=st.w_fwd(w).contiguous(), out=out, M=B * H * W, N=Co,
                K=9 * C, lda=C, bias=b, act=act, conv=(C, H, W))
    _close(_run(call), ref.permute(0, 2, 3, 1).reshape(-1, Co))


def test_conv1_1_im2col_matches_conv2d():
    """lpips_prep's 32-column im2col against w_fwd of a 3-channel kernel is the padded conv of the scaled image"""
    g = _g(2)
    img = torch.rand(2, 3, 8, 12, generator=g, dtype=D64)
    w = torch.randn(64, 3, 3, 3, generator=g, dtype=D64)
    sh, sc = sr._lp(3, "cpu")
    ref = F.conv2d((img - sh) / sc, w, padding=1).permute(0, 2, 3, 1).reshape(-1, 64)
    col = sr.lpips_prep(img)
    call = dict(A=col, B=st.w_fwd(w).contiguous(), out=torch.zeros(col.shape[0], 64, dtype=D64), M=col.shape[0],
                N=64, K=32)
    _close(_run(call), ref)


@pytest.mark.parametrize("masked", [False, True])
def test_conv_dgrad_through_w_bwd_matches_autograd(masked):
    """the conv GEMM of dY with w_bwd (lpips.py's rotated, in / out swapped kernel) is conv2d's input gradient, and
    mask_pos keeps it where the mask is > 0; w_bwd without the 180° rotation is not"""
    g = _g(3)
    B, C, Co, H, W = 2, 4, 6, 5, 8
    x = torch.randn(B, C, H, W, generator=g, dtype=D64, requires_grad=True)
    w = torch.randn(Co, C, 3, 3, generator=g, dtype=D64)
    dy = torch.randn(B, Co, H, W, generator=g, dtype=D64)
    F.conv2d(x, w, padding=1).backward(dy)
    ref = x.grad.permute(0, 2, 3, 1).reshape(-1, C)
    mask = torch.randn(B * H * W, C, generator=g, dtype=D64) if masked else None
    if masked:
        ref = ref * (mask > 0)
    call = dict(A=dy.permute(0, 2, 3, 1).contiguous(), B=st.w_bwd(w).contiguous(), out=torch.zeros(B * H * W, C,
                dtype=D64), M=B * H * W, N=C, K=9 * Co, lda=Co, conv=(Co, H, W), mask_pos=mask)
    _close(_run(call), ref)
    unflipped = w.permute(1, 2, 3, 0).reshape(C, 9 * Co).contiguous()
    assert not torch.allclose(_run(dict(call, B=unflipped)), ref)


def test_pixel_shuffle_store():
    g = _g(4)
    B, gh, gw, r, cout, K = 2, 3, 4, 4, 3, 8
    N = cout * r * r
    a = torch.randn(B * gh * gw, K, generator=g, dtype=D64)
    w = torch.randn(N, K, generator=g, dtype=D64)
    b = torch.randn(N, generator=g, dtype=D64)
    y = (a @ w.t() + b).reshape(B, gh, gw, N).permute(0, 3, 1, 2)
    out = torch.zeros(B, cout, gh * r, gw * r, dtype=D64)
    call = dict(A=a, B=w, out=out, M=B * gh * gw, N=N, K=K, bias=b, pixel_shuffle=(r, gh, gw, cout), ldo=gw * r)
    _close(_run(call), F.pixel_shuffle(y, r))


def test_row_maps():
    """rr_skip = −1 drops the cls row of every T rows (bottleneck write); rr_skip = +1 re-expands HW rows to T = HW + 1
    leaving every cls row as it was (proj_in dgrad)"""
    g = _g(5)
    B, T, K, N = 3, 5, 6, 4
    a = torch.randn(B * T, K, generator=g, dtype=D64)
    w = torch.randn(N, K, generator=g, dtype=D64)
    y = a @ w.t()
    out = torch.full((B * (T - 1), N), 7.0, dtype=D64)
    got = _run(dict(A=a, B=w, out=out, M=B * T, N=N, K=K, rr_group=T, rr_skip=-1))
    _close(got, y.reshape(B, T, N)[:, 1:].reshape(-1, N))
    HW = T - 1
    a2 = torch.randn(B * HW, K, generator=g, dtype=D64)
    out2 = torch.full((B * T, N), 7.0, dtype=D64)
    got2 = _run(dict(A=a2, B=w, out=out2, M=B * HW, N=N, K=K, rr_group=HW, rr_skip=1)).reshape(B, T, N)
    _close(got2[:, 1:].reshape(-1, N), a2 @ w.t())
    assert (got2[:, 0] == 7.0).all()


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (True, False), (False, True), (True, True)])
def test_majors_ldo_accumulate(a_mn, b_mn):
    """A / B read in either major with padded leading dimensions; ldo wider than N leaves the other columns alone;
    accumulate adds onto the prefilled output"""
    g = _g(6)
    M, N, K = 7, 5, 9
    a = torch.randn(M, K, generator=g, dtype=D64)
    b = torch.randn(N, K, generator=g, dtype=D64)
    A = torch.zeros(K, M + 3, dtype=D64) if a_mn else torch.zeros(M, K + 3, dtype=D64)
    Bm = torch.zeros(K, N + 2, dtype=D64) if b_mn else torch.zeros(N, K + 2, dtype=D64)
    (A[:, :M] if a_mn else A[:, :K]).copy_(a.t() if a_mn else a)
    (Bm[:, :N] if b_mn else Bm[:, :K]).copy_(b.t() if b_mn else b)
    out = torch.randn(M, N + 3, generator=g, dtype=D64)
    call = dict(A=A, B=Bm, out=out, M=M, N=N, K=K, lda=A.shape[1], ldb=Bm.shape[1], ldo=N + 3, a_mn=a_mn, b_mn=b_mn,
                accumulate=True)
    got = _run(call)
    _close(got[:, :N], out[:, :N] + a @ b.t())
    assert torch.equal(got[:, N:], out[:, N:])
    assert st.untouched(call, out) and not st.untouched(call, out + 1)


def test_gelu_epilogue_and_refusals():
    g = _g(7)
    a, w = torch.randn(4, 8, generator=g, dtype=D64), torch.randn(6, 8, generator=g, dtype=D64)
    pre = a @ w.t()
    r = st.gemm_ref(dict(A=a, B=w, out=torch.zeros(4, 6, dtype=D64), M=4, N=6, K=8, act=st.ACT_GELU,
                         out2=torch.zeros(4, 6, dtype=D64)), torch.arange(4))
    _close(r["out2"][0], pre)
    _close(r["out"][0], F.gelu(pre))
    for act in (st.ACT_SWIGLU8, st.ACT_ROPE):
        with pytest.raises(NotImplementedError):
            st.gemm_ref(dict(A=a, B=w, out=None, M=4, N=6, K=8, act=act), torch.arange(4))


# --------------------------------------------------------------------------------------------------------- LPIPS

def _lpips_autograd(rec, tgt, vw, vb, lin, coef):
    sh, sc = sr._lp(3, "cpu")
    feats = []
    for img in (rec, tgt):
        x, ci, fs = (img - sh) / sc, 0, []
        for c in st.VGG_CFG:
            if c == "M":
                x = F.max_pool2d(x, 2)
                continue
            x = F.relu(F.conv2d(x, vw[ci], vb[ci], padding=1))
            if ci in st.TAPS:
                fs.append(x)
            ci += 1
        feats.append(fs)
    eps = sr.f32(1e-10)
    total = 0.0
    for k, (f0, f1) in enumerate(zip(*feats)):
        n0 = f0 / (f0.norm(dim=1, keepdim=True) + eps)
        n1 = f1 / (f1.norm(dim=1, keepdim=True) + eps)
        d = (lin[k].reshape(1, -1, 1, 1) * (n0 - n1) ** 2).sum(1)
        total = total + coef * d.mean((1, 2)).sum()
    return total


def test_lpips_chain_is_the_chain_rule():
    """LPIPSLoss._chunk's composition (prep, 13 convs, 4 pools, 5 taps, 12 dgrads with their masks and pool routing,
    the N = 32 GEMM, img_grad) in fp64 equals the LPIPS value and its image gradient by autograd"""
    from vtp_b200.lpips import random_weights

    vw, vb, lw = random_weights(3)
    vw, vb, lw = [w.double() for w in vw], [b.double() for b in vb], [l.double() for l in lw]
    g = _g(8)
    rec = torch.rand(2, 3, 32, 64, generator=g, dtype=D64, requires_grad=True)
    tgt = torch.rand(2, 3, 32, 64, generator=g, dtype=D64)
    coef = 0.37
    loss = _lpips_autograd(rec, tgt, vw, vb, lw, coef)
    loss.backward()
    got = st.lpips_chain(rec.detach(), tgt, vw, vb, lw, coef, rounding=False)
    _close(got["loss"], loss.detach(), 1e-11)
    _close(got["dimg"], rec.grad, 1e-9)


def test_lpips_shape_check():
    from vtp_b200.lpips import LPIPSMetric, check_shape

    for H, W in ((336, 528), (200, 200), (256, 96)):
        with pytest.raises(ValueError, match="LPIPS"):
            check_shape(H, W)
    check_shape(256, 256)
    assert LPIPSMetric.check_shape is check_shape


# ---------------------------------------------------------------------------------------------- SSL, reconstruction

def test_ssl_lists():
    """every student global cls row is held to the teacher row of the other view of its image; local crop (c, b) to
    both views of image b; masked patch i of global crop j to the teacher row of that same patch"""
    B, n_loc, gh = 3, 2, 4
    HW, T = gh * gh, gh * gh + 1
    masks = torch.zeros(2 * B, HW, dtype=torch.bool)
    masks[0, [1, 5, 15]] = True
    masks[4, [0, 3]] = True
    mi = masks.flatten().nonzero().flatten()
    mw = (1.0 / masks.sum(-1).clamp(min=1).float())[:, None].expand_as(masks)[masks]
    L = st.ssl_lists(B, n_loc, T, HW, mi, mw, 2.0, 5)
    tr, sr_ = L["teacher_rows"], L["student_rows"]
    img_of = lambda row: row // T
    for j in range(2 * B):
        assert img_of(sr_[j]) == j and sr_[j] % T == 0
        t = tr[L["t0"][n_loc * B + j]]
        assert img_of(t) == (j + B) % (2 * B) and t % T == 0
    for c in range(n_loc):
        for b in range(B):
            r = c * B + b
            assert {img_of(tr[L["t0"][r]]).item(), img_of(tr[L["t1"][r]]).item()} == {b, B + b}
    for i, m in enumerate(mi.tolist()):
        srow = sr_[2 * B + i]
        assert srow == (m // HW) * T + 1 + m % HW
        assert tr[L["t0"][n_loc * B + 2 * B + i]] == srow and L["t1"][n_loc * B + 2 * B + i] == -1
    assert torch.allclose(L["wrow"][:n_loc * B + 2 * B], torch.full((n_loc * B + 2 * B,), 2.0 / (5 * (2 + 2 * n_loc)),
                                                                     dtype=D64))
    _close(L["wrow"][n_loc * B + 2 * B:], mw.double() * 2.0 / 5)
