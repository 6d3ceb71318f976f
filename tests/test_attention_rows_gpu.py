"""Attention forward and backward row by row against the fp64 references of tests/attn_ref.py, on every dispatch path.

Contract: every (token, head, q|k|v) row of 64 values is within FWD_ROW_TOL / BWD_ROW_TOL of the emulated bf16
reference (the kernels' own rounding points, so a correct kernel differs only by fp32 summation order and ex2.approx),
every lse entry within 1e-4 of fp64, and the fp32 kernel within F32_ROW_TOL of fp64 per row.  Outputs are written
into NaN-filled buffers with sentinel rows on both sides, lse is NaN-filled, and the cls (prefix) rows are reported on
their own.  Each shape in CASES names the branch of the dispatch it exists for.

RoPE tables are random angles rather than the model's axial table: that table repeats sin[d] = sin[d + 32], which
would hide a d / d + 32 mix-up in RoPEᵀ.
"""
import pytest
import torch

from tests import attn_ref as ar
from vtp_b200 import lib

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
# whole-tensor bound of dQ, dK, dV against exact_bwd (fp64 O and lse, no roundings): 1.5x the largest value measured
# on an H100 80GB HBM3 (3.7e-3, dQ of packed_T2_B5), against the 2e-2 the suite allowed when its reference took the
# pre-RoPE values in fp32
BWD_EXACT_TOL = 5.5e-3
PAD = 3  # sentinel rows on each side of an output buffer

# (B, T, H, prefix, causal, rope, no_pack, backward) -> branch.  vtp_attention_fwd (attention.cu): packed when
# !causal && T <= 64 && B > 1 (&& VTP_ATTN_NO_PACK unset), else attn_fwd_kernel<1> for HW <= 128, <2> for
# HW <= 256, the streaming kernel + attn_prefix_rows_kernel above.  vtp_attention_bwd (attention_bwd.cu): the same
# packing rule, attn_bwd_kernel<1> / <2> by HW, the cls query row on warp 8 and the cls key column on CUDA cores when
# unpacked with prefix 1.
CASES = {
    "packed_T37_B50": (50, 37, 6, 1, False, True, False, True),    # local crops, 3 per tile, ragged last pack (2)
    "packed_T37_B2": (2, 37, 2, 1, False, True, False, True),      # one pack with one unused sequence slot
    "packed_T17_B9": (9, 17, 1, 1, False, True, False, True),      # 7 per tile, 9 garbage rows in each tile
    "packed_T64_B4": (4, 64, 2, 0, False, True, False, True),      # exact fill (2 x 64), no prefix
    "packed_T2_B5": (5, 2, 1, 1, False, True, False, True),        # HW = 1, 64 sequences per tile
    "one_tile_T37_B1": (1, 37, 2, 1, False, True, False, True),    # B = 1: unpacked (stochastic-depth subset)
    "one_tile_T2_B1": (1, 2, 16, 1, False, True, False, True),     # unpacked HW = 1
    "no_pack_T37_B3": (3, 37, 2, 1, False, True, True, True),      # VTP_ATTN_NO_PACK
    "one_tile_T101": (2, 101, 6, 1, False, True, False, True),     # <1>, partial tile
    "one_tile_T129": (2, 129, 2, 1, False, True, False, True),     # <1>, HW = 128 (full tile)
    "two_tiles_T130": (2, 130, 2, 1, False, True, False, True),    # <2>, HW = 129 (one row in tile 2)
    "two_tiles_T257_B16": (16, 257, 6, 1, False, True, False, True),  # <2>, the training encoder
    "two_tiles_T256_p0": (2, 256, 16, 0, False, True, False, True),   # <2>, decoder (no prefix)
    "two_tiles_T257_norope": (2, 257, 2, 1, False, False, False, True),
    "causal_T77": (3, 77, 2, 0, True, False, False, True),         # <1> causal, text tower
    "causal_T200": (2, 200, 1, 0, True, True, False, True),        # <2> causal
    "prefix2_T100": (2, 100, 2, 2, False, False, False, False),    # short kernel, prefix rows on warp 8
    "prefix3_T100": (2, 100, 2, 3, False, False, False, False),
    "prefix4_T100": (2, 100, 2, 4, False, False, False, False),
    "prefix2_T300": (1, 300, 2, 2, False, False, False, False),    # HW > 256: streaming kernel + prefix-row kernel
    "prefix3_T300": (1, 300, 2, 3, False, False, False, False),
    "prefix4_T300": (1, 300, 2, 4, False, False, False, False),
    "causal_prefix1_T50_B1": (1, 50, 2, 1, True, False, False, False),  # causal with a prefix (forward only)
}


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _qkv(B, T, H, seed, scale=1.2):
    return (torch.randn(B * T, 3 * H * 64, device="cuda", generator=_gen(seed)) * scale).to(BF)


def _tables(HW, seed):
    ang = torch.rand(HW, 64, device="cuda", generator=_gen(seed)) * 6.28
    return torch.sin(ang).to(BF), torch.cos(ang).to(BF)


def _padded(rows, cols, dtype):
    buf = torch.full((rows + 2 * PAD, cols), float("nan"), device="cuda", dtype=dtype)
    buf[:PAD], buf[-PAD:] = 7.0, -7.0
    return buf, buf.clone(), buf[PAD:PAD + rows]


def _sentinels_intact(buf, before):
    return torch.equal(buf[:PAD], before[:PAD]) and torch.equal(buf[-PAD:], before[-PAD:])


def run_fwd(qkv, B, T, H, prefix, causal):
    buf, before, out = _padded(B * T, H * 64, BF)
    lse = torch.full((B, H, T), float("nan"), device="cuda")
    lib.attention_fwd(qkv, out, B, T, H, prefix=prefix, causal=causal, lse=lse)
    torch.cuda.synchronize()
    assert _sentinels_intact(buf, before)
    assert torch.isfinite(out.float()).all() and torch.isfinite(lse).all()
    return out, lse


def run_bwd(qkv, o, dout, lse, B, T, H, prefix, causal, rope):
    buf, before, dqkv = _padded(B * T, 3 * H * 64, BF)
    lib.attention_bwd(qkv, o, dout, lse, dqkv, B, T, H, prefix=prefix, causal=causal, rope=rope)
    torch.cuda.synchronize()
    assert _sentinels_intact(buf, before)
    assert torch.isfinite(dqkv.float()).all()
    return dqkv


def _stat(check, case, value):
    """one line per measured maximum (pytest -s shows them); the bounds in attn_ref.py were set from these"""
    print(f"ROWSTAT {check} {case} {value:.3e}")


def check_fwd(case, qkv, B, T, H, prefix, causal, whole_exact=True):
    out, lse = run_fwd(qkv, B, T, H, prefix, causal)
    em, _ = ar.emulated_fwd(qkv, B, T, H, prefix, causal)
    ex, lse_ex = ar.exact_fwd(qkv, B, T, H, prefix, causal)
    e = ar.row_err(out, em, (B, T, 1, H))
    e_pre = e[:, :prefix].max().item() if prefix else 0.0
    e_pat = e[:, prefix:].max().item()
    e_lse = ((lse.double() - lse_ex).abs() / lse_ex.abs().clamp(min=1.0)).max().item()
    _stat("fwd_row_prefix", case, e_pre)
    _stat("fwd_row_patch", case, e_pat)
    _stat("fwd_lse", case, e_lse)
    assert max(e_pre, e_pat) <= ar.FWD_ROW_TOL, {"prefix rows": e_pre, "patch rows": e_pat}
    assert e_lse <= 1e-4, e_lse
    if whole_exact:
        w = ar.whole_rel(out, ex)
        _stat("fwd_whole_exact", case, w)
        assert w < 6e-3, w
    return out, lse


def check_bwd(case, qkv, dout, o, lse, B, T, H, prefix, causal, rope, no_pack, whole_exact=True):
    sin, cos = rope if rope is not None else (None, None)
    dqkv = run_bwd(qkv, o, dout, lse, B, T, H, prefix, causal, rope)
    packed = ar.bwd_packed(B, T, causal, no_pack)
    em = ar.emulated_bwd(qkv, o, dout, lse, B, T, H, prefix, causal, sin, cos, packed)
    e = ar.row_err(dqkv, em, (B, T, 3, H))  # [B, T, q|k|v, H]
    errs = {}
    for i, name in enumerate("qkv"):
        errs[f"d{name} patch"] = e[:, prefix:, i].max().item()
        if prefix:
            errs[f"d{name} cls"] = e[:, :prefix, i].max().item()
    for k, v in errs.items():
        _stat("bwd_row_" + k.replace(" ", "_"), case, v)
    assert max(errs.values()) <= ar.BWD_ROW_TOL, errs
    if whole_exact:
        ex = ar.exact_bwd(qkv, dout, B, T, H, prefix, causal, sin, cos)
        w = {n: ar.whole_rel(dqkv.view(B * T, 3, -1)[:, i], ex.view(B * T, 3, -1)[:, i]) for i, n in enumerate("qkv")}
        for n, v in w.items():
            _stat(f"bwd_whole_exact_d{n}", case, v)
        assert max(w.values()) < BWD_EXACT_TOL, w
    return dqkv


def _setup(B, T, H, prefix, causal, rope, seed):
    qkv = _qkv(B, T, H, seed)
    dout = torch.randn(B * T, H * 64, device="cuda", generator=_gen(seed + 1)).to(BF)
    tables = _tables(T - prefix, seed + 2) if rope else None
    return qkv, dout, tables


@pytest.mark.parametrize("case", list(CASES))
def test_attention_rows(case, monkeypatch):
    """Largest values measured on an H100 80GB HBM3 (700 W), per check:
    forward per row vs emulated   patch rows 3.6e-3 (two_tiles_T257_B16), prefix rows 2.9e-3 (prefix4_T300)
    lse per entry vs fp64         1.9e-7
    forward whole tensor vs exact 2.1e-3
    backward per row vs emulated  dQ 3.6e-3, dK 3.6e-3 (two_tiles_T257_B16), dV 4.3e-3 (packed_T37_B50);
                                  cls rows dQ 2.4e-3, dK 2.4e-3, dV 2.3e-3
    backward whole tensor vs exact dQ 3.7e-3, dK 3.5e-3, dV 2.4e-3 (T = 2 shapes)"""
    B, T, H, prefix, causal, rope, no_pack, backward = CASES[case]
    if no_pack:
        monkeypatch.setenv("VTP_ATTN_NO_PACK", "1")
    qkv, dout, tables = _setup(B, T, H, prefix, causal, rope, seed=B * 1000 + T)
    o, lse = check_fwd(case, qkv, B, T, H, prefix, causal)
    if backward:
        check_bwd(case, qkv, dout, o, lse, B, T, H, prefix, causal, tables, no_pack)


# ------------------------------------------------------------------------------------------------------- stress

STRESS_SHAPES = {"packed_T37": (4, 37, 2, 1), "T129": (2, 129, 2, 1), "T257": (2, 257, 2, 1)}


def _stress_inputs(kind, B, T, H, prefix, seed):
    qkv, dout, tables = _setup(B, T, H, prefix, False, True, seed)
    x = qkv.float().view(B, T, 3, H, 64)
    if kind == "sharp":
        # q, k ~ N(0, 3^2): logits q·k / 8 ~ N(0, 9^2), the largest near ±30, so P is nearly one-hot, dP − δ cancels
        # and bf16(P ≈ 1) rounding matters
        x[:, :, :2] *= 3.0 / 1.2
    elif kind == "cls_dominant":
        # the cls key leads by ~10 logits for the odd tokens: nearly all their mass goes through the CUDA-core column
        a = 80 ** 0.5  # a * a / 8 = 10
        x[:, 1::2, 0, :, 0] += a
        x[:, 0, 1, :, 0] = a
    elif kind == "zero_dout":
        d = dout.view(B, T, H * 64)
        d[:, ::5] = 0  # the cls token and every fifth token
    return x.reshape(B * T, -1).to(BF), dout, tables


@pytest.mark.parametrize("shape", list(STRESS_SHAPES))
@pytest.mark.parametrize("kind", ["sharp", "cls_dominant", "zero_dout"])
def test_attention_rows_stress(kind, shape):
    """Largest values measured on an H100 80GB HBM3 (700 W): forward per row 2.5e-3, prefix rows 2.2e-3, lse 2.8e-7;
    backward per row dQ 5.7e-3 (cls_dominant_packed_T37), dK 3.7e-3 and dV 4.6e-3 (sharp_T257), cls rows 2.2e-3"""
    B, T, H, prefix = STRESS_SHAPES[shape]
    qkv, dout, tables = _stress_inputs(kind, B, T, H, prefix, seed=T + 17)
    case = f"{kind}_{shape}"
    o, lse = check_fwd(case, qkv, B, T, H, prefix, False, whole_exact=False)
    dqkv = check_bwd(case, qkv, dout, o, lse, B, T, H, prefix, False, tables, False, whole_exact=False)
    if kind == "zero_dout":
        # dS is exactly zero on a query row whose dO is zero, so its dQ is exactly zero
        dq = dqkv.view(B, T, 3, -1)[:, ::5, 0]
        assert (dq == 0).all(), dq.abs().max()


# ------------------------------------------------------------------------------------------------- determinism

@pytest.mark.parametrize("case", ["packed_T37_B50", "one_tile_T37_B1", "two_tiles_T257_B16", "causal_T200"])
def test_attention_bitwise_deterministic(case):
    """two launches give bit-identical results (the cls column reductions use shared-memory atomics)"""
    B, T, H, prefix, causal, rope, _, _ = CASES[case]
    qkv, dout, tables = _setup(B, T, H, prefix, causal, rope, seed=5)
    o1, l1 = run_fwd(qkv, B, T, H, prefix, causal)
    o2, l2 = run_fwd(qkv, B, T, H, prefix, causal)
    assert torch.equal(o1, o2) and torch.equal(l1, l2)
    g1 = run_bwd(qkv, o1, dout, l1, B, T, H, prefix, causal, tables)
    g2 = run_bwd(qkv, o1, dout, l1, B, T, H, prefix, causal, tables)
    assert torch.equal(g1, g2)


def test_attention_bwd_argument_errors():
    def call(B, T, H, prefix, causal=False, rope=None, rows=None):
        qkv = torch.zeros((rows or B * T), 3 * H * 64, device="cuda", dtype=BF)
        o = torch.zeros((rows or B * T), H * 64, device="cuda", dtype=BF)
        lse = torch.zeros(B, H, T, device="cuda")
        dqkv = torch.empty_like(qkv)
        lib.attention_bwd(qkv, o, o, lse, dqkv, B, T, H, prefix=prefix, causal=causal, rope=rope)

    sin, cos = _tables(36, 0)
    for kw in (dict(B=2, T=37, H=2, prefix=2),                      # prefix 2
               dict(B=2, T=37, H=2, prefix=1, causal=True),         # causal with a prefix
               dict(B=1, T=258, H=2, prefix=1),                     # HW = 257 > 256
               dict(B=1, T=257, H=2, prefix=0),                     # HW = 257 > 256
               dict(B=2, T=37, H=2, prefix=1, rope=(sin, None)),    # one RoPE table without the other
               dict(B=2, T=37, H=2, prefix=1, rope=(None, cos)),
               dict(B=2, T=37, H=2, prefix=1, rows=2 * 38)):        # qkv rows disagree with B, T
        with pytest.raises(lib.VtpError):
            call(**kw)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ fp32 kernel

F32_CASES = {"T2": (3, 2, 2, False, 1.0), "T37": (2, 37, 6, False, 1.0), "T256": (2, 256, 2, False, 1.0),
             "T257": (2, 257, 3, False, 1.0), "T411_smem_last": (1, 411, 2, False, 1.0),
             "T412_tiled_first": (1, 412, 2, False, 1.0), "T77_causal": (3, 77, 2, True, 1.0),
             "T257_sharp": (2, 257, 2, False, 3.0), "T412_sharp": (1, 412, 2, False, 3.0)}


@pytest.mark.parametrize("case", list(F32_CASES))
def test_attention_f32_rows(case):
    """attention_fwd_f32: smem-resident kernel up to T = 411, the tiled kernel from 412; sharp = logits up to ±30.
    Largest per-row error measured on an H100 80GB HBM3 (700 W): 6.0e-6 (T257_sharp)."""
    B, T, H, causal, sc = F32_CASES[case]
    qkv = torch.randn(B * T, 3 * H * 64, device="cuda", generator=_gen(T)) * sc
    buf, before, out = _padded(B * T, H * 64, torch.float32)
    lib.attention_fwd_f32(qkv, out, B, T, H, causal=causal)
    torch.cuda.synchronize()
    assert _sentinels_intact(buf, before) and torch.isfinite(out).all()
    ref, _ = ar.exact_fwd(qkv, B, T, H, 0, causal)
    e = ar.row_err(out, ref, (B, T, 1, H)).max().item()
    _stat("f32_row", case, e)
    assert e <= ar.F32_ROW_TOL, e


# ------------------------------------------------------------------------------------------------------ RoPE

def _rope_bf16(qkv, sin, cos, B, T, H, prefix):
    """layers/attention.py:70-89 in torch bf16: x * cos + rotate_half(x) * sin, every op rounded to bf16"""
    x = qkv.view(B, T, 3, H, 64).clone()
    for i in (0, 1):
        y = x[:, prefix:, i]
        y1, y2 = y.chunk(2, dim=-1)
        x[:, prefix:, i] = y * cos[None, :, None] + torch.cat([-y2, y1], -1) * sin[None, :, None]
    return x.view(B * T, -1)


@pytest.mark.parametrize("B,T,H,prefix", [(2, 257, 6, 1), (3, 256, 2, 0)])
def test_rope_fwd_bitwise(B, T, H, prefix):
    qkv = _qkv(B, T, H, seed=T)
    sin, cos = _tables(T - prefix, T + 1)
    want = _rope_bf16(qkv, sin, cos, B, T, H, prefix)
    got = qkv.clone()
    lib.rope_fwd(got, sin, cos, B * T, T, prefix, H * 64)
    torch.cuda.synchronize()
    g, q0 = got.view(B, T, 3, -1), qkv.view(B, T, 3, -1)
    assert torch.equal(g[:, :, 2], q0[:, :, 2]) and torch.equal(g[:, :prefix], q0[:, :prefix])
    assert torch.equal(got, want)


def test_gemm_rope_epilogue_equals_gemm_then_rope():
    """the QKV GEMM's fused RoPE epilogue is bit for bit the plain GEMM followed by rope_fwd"""
    B, T, prefix, D, K = 2, 257, 1, 384, 384
    A = (torch.randn(B * T, K, device="cuda", generator=_gen(14))).to(BF)
    W = (torch.randn(3 * D, K, device="cuda", generator=_gen(15)) * 0.05).to(BF)
    bias = torch.randn(3 * D, device="cuda", generator=_gen(16)) * 0.1
    sin, cos = _tables(T - prefix, 17)
    fused = torch.empty(B * T, 3 * D, device="cuda", dtype=BF)
    lib.gemm(A, W, fused, M=B * T, N=3 * D, K=K, bias=bias, act=lib.ACT_ROPE, rope=(sin, cos, T, prefix, 2 * D))
    plain = torch.empty_like(fused)
    lib.gemm(A, W, plain, M=B * T, N=3 * D, K=K, bias=bias)
    lib.rope_fwd(plain, sin, cos, B * T, T, prefix, D)
    torch.cuda.synchronize()
    assert torch.equal(fused, plain), (fused.float() - plain.float()).abs().max()
