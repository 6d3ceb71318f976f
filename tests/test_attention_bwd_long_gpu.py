"""The streaming attention backward (vtp_attention_bwd_long, csrc/attention_bwd_long.cu) row by row against the fp64
references of tests/attn_ref.py, and against the single-pass vtp_attention_bwd where both apply.

Contract, as for the single-pass kernel (tests/test_attention_rows_gpu.py): every (token, head, q|k|v) row of 64 values
within BWD_ROW_TOL of emulated_bwd(packed=False) (the kernels' bf16 rounding points: P and dS bf16 where they enter a
patch-key GEMM, the cls row and column fp32), the whole tensor within 5.5e-3 of exact_bwd, outputs written into
NaN-filled buffers with sentinel rows on both sides, o and lse from lib.attention_fwd.  The δ workspace is checked too.
"""
import pytest
import torch

from tests import attn_ref as ar
from tests import test_attention_rows_gpu as rows
from vtp_b200 import lib

pytestmark = pytest.mark.gpu
BF = torch.bfloat16

# name -> (B, T, H, prefix): the branch each shape exists for.  The kernels tile the HW = T - prefix patch tokens in
# 128-row query tiles (dq kernel) and 128-row key tiles (dkdv kernel), each split into 64-row halves, with a 2-stage
# K/V (Q/dO) ring; the cls token goes to attn_bwd_prefix_kernel.
LONG_CASES = {
    "HW1": (3, 2, 2, 1),            # one patch token: 127 masked rows and columns, second half skipped
    "HW36": (2, 37, 2, 1),          # a local crop, one partial half
    "HW128": (2, 129, 2, 1),        # exactly one tile
    "HW129": (2, 130, 2, 1),        # one row in tile 2
    "HW256": (2, 257, 2, 1),        # two full tiles (the single-pass kernel's largest)
    "HW257": (2, 258, 2, 1),        # one row in tile 3: the ring's first reuse of stage 0
    "HW384": (2, 385, 2, 1),        # three full tiles
    "HW385": (2, 386, 2, 1),        # one row in tile 4
    "HW693_2img": (2, 694, 2, 1),   # 336x528: the last tile of image 0 reads image 1's rows
    "HW1024_p0": (2, 1024, 2, 0),   # the pixel decoder at 512x512 (no prefix kernel)
    "HW1024_p1": (2, 1025, 2, 1),   # the trunk at 512x512
    "HW2304": (1, 2305, 2, 1),      # 768x768
    "HW4096": (1, 4097, 2, 1),      # 1024x1024, B = 1: the last tile is TMA zero fill
}


def _stat(check, case, value):
    print(f"ROWSTAT {check} {case} {value:.3e}")


def run_long(qkv, o, dout, lse, B, T, H, prefix, rope):
    buf, before, dqkv = rows._padded(B * T, 3 * H * 64, BF)
    delta = torch.full((B, H, T), float("nan"), device="cuda")
    lib.attention_bwd_long(qkv, o, dout, lse, delta, dqkv, B, T, H, prefix=prefix, rope=rope)
    torch.cuda.synchronize()
    assert rows._sentinels_intact(buf, before)
    assert torch.isfinite(dqkv.float()).all() and torch.isfinite(delta).all()
    return dqkv, delta


def check_delta(delta, o, dout, B, T, H):
    """δ = Σ dO·O per (image, head, token): fp32 sum of 64 exact bf16 products"""
    (do,), (oo,) = ar.heads(dout, B, T, H), ar.heads(o, B, T, H)
    ref = (do * oo).sum(-1)
    mag = (do * oo).abs().sum(-1)
    assert ((delta.double() - ref).abs() <= 2e-6 * mag + 1e-30).all()


def check_rows(case, dqkv, qkv, o, dout, lse, B, T, H, prefix, rope, whole_exact=True):
    sin, cos = rope if rope is not None else (None, None)
    em = ar.emulated_bwd(qkv, o, dout, lse, B, T, H, prefix, False, sin, cos, packed=False)
    e = ar.row_err(dqkv, em, (B, T, 3, H))
    errs = {}
    for i, name in enumerate("qkv"):
        errs[f"d{name} patch"] = e[:, prefix:, i].max().item()
        if prefix:
            errs[f"d{name} cls"] = e[:, :prefix, i].max().item()
    for k, v in errs.items():
        _stat("long_bwd_row_" + k.replace(" ", "_"), case, v)
    assert max(errs.values()) <= ar.BWD_ROW_TOL, errs
    if whole_exact:
        ex = ar.exact_bwd(qkv, dout, B, T, H, prefix, False, sin, cos)
        w = {n: ar.whole_rel(dqkv.view(B * T, 3, -1)[:, i], ex.view(B * T, 3, -1)[:, i]) for i, n in enumerate("qkv")}
        for n, v in w.items():
            _stat(f"long_bwd_whole_exact_d{n}", case, v)
        assert max(w.values()) < rows.BWD_EXACT_TOL, w


@pytest.mark.parametrize("rope", [True, False], ids=["rope", "norope"])
@pytest.mark.parametrize("case", list(LONG_CASES))
def test_attention_bwd_long_rows(case, rope):
    B, T, H, prefix = LONG_CASES[case]
    qkv, dout, tables = rows._setup(B, T, H, prefix, False, rope, seed=B * 1000 + T + 7)
    o, lse = rows.run_fwd(qkv, B, T, H, prefix, False)
    dqkv, delta = run_long(qkv, o, dout, lse, B, T, H, prefix, tables)
    check_delta(delta, o, dout, B, T, H)
    check_rows(f"{case}_{'rope' if rope else 'norope'}", dqkv, qkv, o, dout, lse, B, T, H, prefix, tables)


def test_attention_bwd_long_many_ctas():
    """T = 1025, H = 6, B = 48: 8 x 6 x 48 = 2304 CTAs per kernel, many waves on 132 SMs; three images are checked"""
    B, T, H, prefix = 48, 1025, 6, 1
    qkv, dout, tables = rows._setup(B, T, H, prefix, False, True, seed=99)
    o, lse = rows.run_fwd(qkv, B, T, H, prefix, False)
    dqkv, _ = run_long(qkv, o, dout, lse, B, T, H, prefix, tables)
    for img in (0, 23, 47):
        sl = slice(img * T, (img + 1) * T)
        check_rows(f"many_ctas_img{img}", dqkv[sl], qkv[sl], o[sl], dout[sl], lse[img:img + 1], 1, T, H, prefix, tables,
                   whole_exact=False)


# (B, T, H, prefix): both entry points apply (HW <= 256); the single-pass kernel runs unpacked for all of them
AGREE_CASES = {"T2_B1": (1, 2, 2, 1), "T37_B1": (1, 37, 2, 1), "T129": (2, 129, 2, 1), "T130": (2, 130, 2, 1),
               "T257": (2, 257, 6, 1), "T256_p0": (2, 256, 2, 0)}


@pytest.mark.parametrize("case", list(AGREE_CASES))
def test_attention_bwd_long_agrees_with_single_pass(case):
    B, T, H, prefix = AGREE_CASES[case]
    qkv, dout, tables = rows._setup(B, T, H, prefix, False, True, seed=T + 3)
    o, lse = rows.run_fwd(qkv, B, T, H, prefix, False)
    dl, _ = run_long(qkv, o, dout, lse, B, T, H, prefix, tables)
    ds = rows.run_bwd(qkv, o, dout, lse, B, T, H, prefix, False, tables)
    e = ar.row_err(dl, ds, (B, T, 3, H)).max().item()
    _stat("long_vs_single_pass_row", case, e)
    assert e <= ar.BWD_ROW_TOL, e


STRESS_SHAPES = {"T1025": (1, 1025, 2, 1), "T694": (2, 694, 2, 1)}


@pytest.mark.parametrize("shape", list(STRESS_SHAPES))
@pytest.mark.parametrize("kind", ["sharp", "cls_dominant", "zero_dout"])
def test_attention_bwd_long_stress(kind, shape):
    """sharp: logits up to about ±30; cls_dominant: the cls key leads by ~10 logits for every other token; zero_dout:
    the cls token and every fifth token have dO = 0, so their dS rows and dQ rows are exactly zero"""
    B, T, H, prefix = STRESS_SHAPES[shape]
    qkv, dout, tables = rows._stress_inputs(kind, B, T, H, prefix, seed=T + 17)
    o, lse = rows.run_fwd(qkv, B, T, H, prefix, False)
    dqkv, _ = run_long(qkv, o, dout, lse, B, T, H, prefix, tables)
    check_rows(f"{kind}_{shape}", dqkv, qkv, o, dout, lse, B, T, H, prefix, tables, whole_exact=False)
    if kind == "zero_dout":
        dq = dqkv.view(B, T, 3, -1)[:, ::5, 0]
        assert (dq == 0).all(), dq.abs().max()


@pytest.mark.parametrize("B,T,H,prefix", [(2, 1025, 6, 1), (2, 694, 2, 1), (2, 1024, 2, 0)])
def test_attention_bwd_long_bitwise_deterministic(B, T, H, prefix):
    qkv, dout, tables = rows._setup(B, T, H, prefix, False, True, seed=5)
    o, lse = rows.run_fwd(qkv, B, T, H, prefix, False)
    g1, d1 = run_long(qkv, o, dout, lse, B, T, H, prefix, tables)
    g2, d2 = run_long(qkv, o, dout, lse, B, T, H, prefix, tables)
    assert torch.equal(g1, g2) and torch.equal(d1, d2)


def test_attention_bwd_long_argument_errors():
    def call(B, T, H, prefix, rope=None, rows_=None, delta=True, lse_=True):
        n = rows_ or B * T
        qkv = torch.zeros(n, 3 * H * 64, device="cuda", dtype=BF)
        o = torch.zeros(n, H * 64, device="cuda", dtype=BF)
        lse = torch.zeros(B, H, T, device="cuda") if lse_ else None
        ws = torch.zeros(B, H, T, device="cuda") if delta else None
        lib.attention_bwd_long(qkv, o, o, lse, ws, torch.empty_like(qkv), B, T, H, prefix=prefix, rope=rope)

    sin, cos = rows._tables(1024, 0)
    for kw in (dict(B=1, T=1026, H=2, prefix=2),                     # prefix 2
               dict(B=1, T=1, H=2, prefix=1),                        # no patch token
               dict(B=1, T=1025, H=2, prefix=1, rope=(sin, None)),   # one RoPE table without the other
               dict(B=1, T=1025, H=2, prefix=1, rope=(None, cos)),
               dict(B=1, T=1025, H=2, prefix=1, delta=False),        # no δ workspace
               dict(B=1, T=1025, H=2, prefix=1, lse_=False),         # no lse
               dict(B=65536, T=1, H=1, prefix=0),                    # grid z > 65535
               dict(B=2, T=1025, H=2, prefix=1, rows_=2 * 1026)):    # qkv rows disagree with B, T
        with pytest.raises(lib.VtpError):
            call(**kw)
    torch.cuda.synchronize()
