"""The GEMM's epilogue warps finish tile t while the MMA warps already run tile t+1, with one shared accumulator tile
between them.  A broken hand-off writes a tile from another tile's accumulators (or from a half-dumped one), so these
tests launch many tiles per persistent CTA (tiles >> 132 SMs), give every 128 x 128 tile its own scale (A rows scaled by
their row block, B rows by their column block), and check every output row against an fp32 product of the same bf16
inputs, on every epilogue family: the lean TMA-store epilogue (FAST 1-5), the SwiGLU gate (FAST 6 / 7), the generic
epilogue (GELU + pre-activation output, RoPE, row remap, PixelShuffle), implicit conv and split-K.  K = 64 is a single
k-block per tile, so the epilogue is longer than the mainloop and the MMA warps wait for the accumulator tile to be
released; K = 384 is the recurring short-K shape of the training step.  Repeat launches must be bit-identical."""
import pytest
import torch
import torch.nn.functional as F

from vtp_b200 import lib

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
ULP = 2.0 ** -7  # one bf16 ulp relative to the row's largest value: where fp32 accumulation order flips a rounding point


def _tiled(rows, K, seed, scale=1.0):
    """[rows, K] bf16 operand whose 128-row blocks carry distinct scales (tile-distinct products)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    blk = torch.arange(rows, device="cuda") // 128
    s = scale * (0.5 + (blk % 7).float() / 4 + (blk % 3).float() / 16)
    return (torch.randn(rows, K, device="cuda", generator=g) * s[:, None]).to(BF)


def _ref(A, W):
    torch.backends.cuda.matmul.allow_tf32 = False
    return A.float() @ W.float().t()


def _nan(shape, dt=BF):
    return torch.full(shape, float("nan"), device="cuda", dtype=dt)


def _check_rows(out, ref, rel, what=""):
    """Every row of out within rel * (largest |ref| of the row); reports the failing rows and their 128-row tiles."""
    o = out.float().reshape(out.shape[0], -1)
    r = ref.float().reshape(ref.shape[0], -1)
    assert o.shape == r.shape
    assert torch.isfinite(o).all(), f"{what}: non-finite output"
    err = (o - r).abs().amax(1)
    lim = rel * r.abs().amax(1) + 1e-6
    bad = (err > lim).nonzero().flatten()
    assert bad.numel() == 0, (f"{what}: {bad.numel()} bad rows, first {bad[:6].tolist()} (row tiles "
                              f"{sorted(set((bad[:64] // 128).tolist()))[:6]}), err {err[bad[:3]].tolist()} lim {lim[bad[:3]].tolist()}")


def _twice(run):
    """run() -> output tensor(s) of a fresh launch; returns the first, asserting the second is bit-identical."""
    a, b = run(), run()
    torch.cuda.synchronize()
    for x, y in zip(a if isinstance(a, tuple) else (a,), b if isinstance(b, tuple) else (b,)):
        assert torch.equal(x, y), "repeat launch differs"
    return a


# (M, N, K): many tiles per CTA at K = 64 and K = 384, and ragged M / N tails (M % 128 != 0, N % 128 != 0)
SHAPES = [(20480, 1024, 64), (20480, 1024, 384), (20037, 1000, 64), (16411, 1160, 384)]


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("mode", ["bf16", "bf16_resid", "f32", "f32_resid", "bf16_relu", "f32_relu"])
def test_fast_epilogue_tiles(M, N, K, mode):
    """FAST 1-4 (bf16 / fp32 out, with and without a same-dtype residual) and their ReLU forms."""
    A, W = _tiled(M, K, 1), _tiled(N, K, 2, 0.1)
    bias = torch.randn(N, device="cuda")
    dt = torch.float32 if mode.startswith("f32") else BF
    resid = torch.randn(M, N, device="cuda").to(dt) if mode.endswith("resid") else None
    relu = mode.endswith("relu")
    acc = (_ref(A, W) + bias).to(BF).float()
    if relu:
        acc = acc.clamp_min(0)
    ref = acc + resid.float() if resid is not None else acc

    def run():
        out = _nan((M, N), dt)
        lib.gemm(A, W, out, M=M, N=N, K=K, bias=bias, resid=resid, act=lib.ACT_RELU if relu else lib.ACT_NONE)
        return out

    _check_rows(_twice(run), ref, 2 * ULP if resid is not None and dt == BF else ULP, mode)


@pytest.mark.parametrize("M,N,K", SHAPES[:2])
def test_fast_epilogue_mn_major_b(M, N, K):
    """dgrad form (weight read untransposed: MN-major B) through the lean epilogue."""
    A, W = _tiled(M, K, 3), _tiled(N, K, 4, 0.1)
    Wt = W.t().contiguous()
    ref = _ref(A, W).to(BF).float()

    def run():
        out = _nan((M, N))
        lib.gemm(A, Wt, out, M=M, N=N, K=K, b_mn=True)
        return out

    _check_rows(_twice(run), ref, ULP)


@pytest.mark.parametrize("M,Hs,K,with_pre", [(20480, 1024, 64, True), (20037, 1000, 384, True), (20480, 1024, 384, False),
                                             (16411, 504, 64, False)])
def test_swiglu_tiles(M, Hs, K, with_pre):
    """FAST 6 (hidden + pre-activation) and FAST 7 (hidden only)."""
    A = _tiled(M, K, 5)
    W1, W2 = _tiled(Hs, K, 6, 0.05), _tiled(Hs, K, 7, 0.05)
    b1, b2 = torch.randn(Hs, device="cuda") * 0.1, torch.randn(Hs, device="cuda") * 0.1
    Wp = torch.stack([W1.view(Hs // 8, 8, K), W2.view(Hs // 8, 8, K)], dim=1).reshape(2 * Hs, K).contiguous()
    bp = torch.stack([b1.view(-1, 8), b2.view(-1, 8)], dim=1).reshape(-1).contiguous()
    x1, x2 = (_ref(A, W1) + b1).to(BF), (_ref(A, W2) + b2).to(BF)
    ref = F.silu(x1.float()).to(BF).float() * x2.float()

    def run():
        out = _nan((M, Hs))
        pre = _nan((M, 2 * Hs)) if with_pre else None
        lib.gemm(A, Wp, out, M=M, N=2 * Hs, K=K, bias=bp, act=lib.ACT_SWIGLU8, ldo=Hs, out2=pre)
        return (out, pre) if with_pre else (out,)

    res = _twice(run)
    _check_rows(res[0], ref, 2 * ULP, "hidden")
    if with_pre:
        pre_ref = torch.stack([x1.view(M, Hs // 8, 8), x2.view(M, Hs // 8, 8)], dim=2).reshape(M, 2 * Hs)
        _check_rows(res[1], pre_ref, ULP, "pre-activation")


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_generic_gelu_out2_tiles(M, N, K):
    """Generic epilogue: GELU with the bf16 pre-activation as a second output."""
    A, W = _tiled(M, K, 8), _tiled(N, K, 9, 0.05)
    bias = torch.randn(N, device="cuda") * 0.1
    pre_ref = (_ref(A, W) + bias).to(BF)
    ref = F.gelu(pre_ref.float())

    def run():
        out, pre = _nan((M, N)), _nan((M, N))
        lib.gemm(A, W, out, M=M, N=N, K=K, bias=bias, act=lib.ACT_GELU, out2=pre)
        return out, pre

    out, pre = _twice(run)
    _check_rows(pre, pre_ref, ULP, "pre-activation")
    _check_rows(out, ref, 2 * ULP, "gelu")


@pytest.mark.parametrize("K", [64, 384])
def test_generic_rope_tiles(K):
    """Generic epilogue: bias + axial RoPE on the q / k columns of a qkv projection (VTP-Small width, 80 images)."""
    Bn, Ntok, prefix, D = 80, 257, 1, 384
    H, M = D // 64, Bn * Ntok
    A, W = _tiled(M, K, 10), _tiled(3 * D, K, 11, 0.05)
    bias = torch.randn(3 * D, device="cuda") * 0.1
    ang = torch.rand(Ntok - prefix, 64, device="cuda") * 6.28
    sin, cos = torch.sin(ang).to(BF), torch.cos(ang).to(BF)
    qkv = (_ref(A, W) + bias).to(BF).view(Bn, Ntok, 3, H, 64)
    ref = qkv.clone()
    for i in (0, 1):  # layers/attention.py:12-23 in bf16
        x = qkv[:, prefix:, i]
        x1, x2 = x.chunk(2, dim=-1)
        ref[:, prefix:, i] = (x * cos[None, :, None, :]) + (torch.cat([-x2, x1], dim=-1) * sin[None, :, None, :])

    def run():
        out = _nan((M, 3 * D))
        lib.gemm(A, W, out, M=M, N=3 * D, K=K, bias=bias, act=lib.ACT_ROPE, rope=(sin, cos, Ntok, prefix, 2 * D))
        return out

    _check_rows(_twice(run), ref.view(M, 3 * D), 4 * ULP, "rope")


@pytest.mark.parametrize("K", [64, 384])
def test_generic_row_remap_tiles(K):
    """Generic epilogue: fp32 residual stream in place, rows written behind a cls slot per image (row remap)."""
    Bn, G, D = 80, 256, 384
    M = Bn * G
    A, W = _tiled(M, K, 12), _tiled(D, K, 13, 0.05)
    bias = torch.randn(D, device="cuda")
    x0 = torch.randn(Bn * (G + 1), D, device="cuda")
    exp = x0.view(Bn, G + 1, D).clone()
    exp[:, 1:] += (_ref(A, W) + bias).to(BF).float().view(Bn, G, D)

    def run():
        x = x0.clone()
        lib.gemm(A, W, x, M=M, N=D, K=K, bias=bias, resid=x, rr_group=G, rr_skip=1)
        return x

    x = _twice(run).view(Bn, G + 1, D)
    assert torch.equal(x[:, 0], x0.view(Bn, G + 1, D)[:, 0])
    _check_rows(x.reshape(-1, D), exp.reshape(-1, D), ULP, "row remap")


def test_generic_pixel_shuffle_tiles():
    """Generic epilogue: PixelShuffle NCHW store of the pixel decoder (16 x 16 grid, r = 16, 3 channels; 60 images)."""
    Bn, g, r, D = 60, 16, 16, 384
    M, N = Bn * g * g, 3 * r * r
    A, W = _tiled(M, D, 14), _tiled(N, D, 15, 0.05)
    bias = torch.randn(N, device="cuda") * 0.1
    ref = F.pixel_shuffle((_ref(A, W) + bias).view(Bn, g, g, N).permute(0, 3, 1, 2), r)

    def run():
        out = _nan((Bn, 3, g * r, g * r), torch.float32)
        lib.gemm(A, W, out, M=M, N=N, K=D, bias=bias, pixel_shuffle=(r, g, g, 3), ldo=g * r, round_bf16=False)
        return out

    out = _twice(run)
    _check_rows(out.permute(0, 2, 1, 3).reshape(Bn * g * r, -1), ref.permute(0, 2, 1, 3).reshape(Bn * g * r, -1), 1e-5,
                "pixel shuffle")


def _conv_operands(Bn, hw, cin, cout, seed):
    torch.backends.cudnn.allow_tf32 = False
    g = torch.Generator(device="cuda").manual_seed(seed)
    img = torch.arange(Bn, device="cuda").float()
    x = (torch.randn(Bn, hw, hw, cin, device="cuda", generator=g) * (0.5 + img % 5 / 4)[:, None, None, None]).to(BF)
    w = (torch.randn(cout, 3, 3, cin, device="cuda", generator=g) * 0.05).to(BF)  # K index = (ky * 3 + kx) * cin + c
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), padding=1).permute(0, 2, 3, 1)
    return x, w.reshape(cout, 9 * cin), ref


@pytest.mark.parametrize("Bn,hw,cin,cout", [(8, 128, 64, 64), (8, 64, 64, 128), (16, 56, 128, 128)])
def test_conv_forward_tiles(Bn, hw, cin, cout):
    """Implicit 3x3 conv (LPIPS conv1_2 / conv2_1 forms, and a height that leaves the last tile row partly empty), bias + ReLU."""
    x, w, ref = _conv_operands(Bn, hw, cin, cout, 16)
    bias = torch.randn(cout, device="cuda") * 0.1
    ref = (ref + bias).to(BF).float().clamp_min(0)
    M = Bn * hw * hw

    def run():
        y = _nan((Bn, hw, hw, cout))
        lib.gemm(x, w, y, M=M, N=cout, K=9 * cin, lda=cin, ldb=9 * cin, bias=bias, act=lib.ACT_RELU, ldo=cout,
                 conv=(cin, hw, hw))
        return y

    _check_rows(_twice(run).reshape(M, cout), ref.reshape(M, cout), ULP, "conv")


@pytest.mark.parametrize("Bn,hw,cin,cout", [(8, 128, 64, 64), (8, 64, 128, 64)])
def test_conv_dgrad_relu_mask_tiles(Bn, hw, cin, cout):
    """LPIPS dgrad: implicit conv whose output is masked by (forward activation > 0) in the epilogue (FAST 5)."""
    dz, w, ref = _conv_operands(Bn, hw, cin, cout, 17)
    g = torch.Generator(device="cuda").manual_seed(18)
    act = torch.randn(Bn, hw, hw, cout, device="cuda", generator=g).to(BF)
    act[..., ::7] = 0  # exact zeros are masked too
    ref = torch.where(act.float() > 0, ref.to(BF).float(), torch.zeros_like(ref))
    M = Bn * hw * hw

    def run():
        dx = _nan((Bn, hw, hw, cout))
        lib.gemm(dz, w, dx, M=M, N=cout, K=9 * cin, lda=cin, ldb=9 * cin, ldo=cout, conv=(cin, hw, hw),
                 mask_pos=act.view(M, cout))
        return dx

    _check_rows(_twice(run).reshape(M, cout), ref.reshape(M, cout), ULP, "masked conv")


@pytest.mark.parametrize("M,N,K,split", [(2048, 1024, 4096, 4), (1152, 1536, 8192, -1), (2056, 1000, 2048, 3)])
def test_splitk_tiles(M, N, K, split):
    """wgrad form (TN) with split-K: fp32 red.add of several k-ranges into a pre-filled output."""
    A, B = _tiled(M, K, 19).t().contiguous(), _tiled(N, K, 20).t().contiguous()  # stored [K][M], [K][N]
    out = torch.ones((M, N), device="cuda")
    lib.gemm(A, B, out, M=M, N=N, K=K, a_mn=True, b_mn=True, accumulate=True, split_k=split, round_bf16=False)
    torch.cuda.synchronize()
    # fp32 sums of up to 8192 products in an unfixed order: ~1e-5 of the row scale; a misplaced tile is off by O(1)
    _check_rows(out, A.float().t() @ B.float() + 1.0, 1e-4, "split-K")
