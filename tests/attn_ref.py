"""Plain-torch references for the attention kernels, on the CPU or the GPU (no kernels, nothing from oracle/).

exact_fwd / exact_bwd        fp64 attention and its gradient, computed from the very bf16 values the kernels receive.
emulated_fwd / emulated_bwd  the same maths with the kernels' bf16 rounding points (attention.cu, attention_long.cu,
                             attention_bwd.cu), so that only fp32 accumulation order and ex2.approx separate a correct
                             kernel from them.
row_err                      the per-row metric: one row is one (token, head, q|k|v) slice of 64 values, so one wrong
                             row, key or RoPE position cannot hide in a whole-tensor norm.

Layouts follow the kernels: qkv [B*T, 3*H*64] (q | k | v, heads inside each third), out / dout [B*T, H*64],
lse [B, H, T], RoPE tables [HW, 64] for the T - prefix patch tokens.  Internally every operand is fp64 [B, H, T, 64].
"""
import torch

SCALE = 0.125  # 1 / sqrt(head_dim = 64)

# Per-row bounds of the GPU tests (tests/test_attention_rows_gpu.py, tests/test_kernels_gpu.py): about 1.5x the
# largest error measured on an H100 80GB HBM3 (700 W limit), never above the ceilings 2^-7 (bf16 paths, one bf16 ulp
# at the top of a binade) and 1e-5 (fp32 path).  Measured maxima: forward 3.6e-3; backward 5.7e-3, in dQ of a packed
# tile whose cls key takes ~98 % of the mass (such a row follows one bf16 dS entry, so a single rounding flip there
# would move it by up to an ulp; not traced further), which puts 1.5x above the ceiling and the backward bound at the
# ceiling; fp32 6.0e-6.
FWD_ROW_TOL = 5.4e-3
BWD_ROW_TOL = 2 ** -7
F32_ROW_TOL = 9e-6


def heads(x, B, T, H, parts=1):
    """[B*T, parts*H*64] -> `parts` fp64 tensors [B, H, T, 64]"""
    y = x.reshape(B, T, parts, H, 64).double()
    return [y[:, :, i].transpose(1, 2) for i in range(parts)]


def merge(*parts):
    """fp64 [B, H, T, 64] tensors -> [B*T, len(parts)*H*64]"""
    B, H, T, _ = parts[0].shape
    return torch.stack([p.transpose(1, 2) for p in parts], 2).reshape(B * T, len(parts) * H * 64)


def visible(T, causal, device=None):
    """[T, T] bool, query j sees key t.  The prefix (cls) tokens are ordinary keys and queries; causal: t <= j in
    token positions, which is the kernels' rule for the prefix columns and the patch keys alike."""
    m = torch.ones(T, T, dtype=torch.bool, device=device)
    return m.tril() if causal else m


def to_bf16(x):
    """round to the nearest bf16 the way the kernels convert an fp32 value; keeps x's dtype"""
    return x.float().to(torch.bfloat16).to(x.dtype)


def bwd_packed(B, T, causal, no_pack=False):
    """vtp_attention_fwd / _bwd dispatch: whole sequences share one 128-row tile, cls tokens included as ordinary rows
    and keys (so their P / dS entries go through the bf16 GEMMs too)"""
    return not causal and T <= 64 and B > 1 and not no_pack


# ---------------------------------------------------------------------------------------------------------- forward

def fwd_core(q, k, v, vis, rounding=True):
    """softmax(SCALE q kᵀ) v over the visible keys -> (o [B,H,T,64], lse [B,H,T]).  rounding: the numerators
    P̃ = bf16(exp(SCALE (s - m))) with m the row max over prefix and patch keys feed P·V, while l sums the unrounded
    numerators (attention.cu:146-161, 274-287; the streaming kernel rounds relative to its running max instead, which
    changes P̃ by well under one ulp of the row)."""
    s = (q @ k.transpose(-1, -2)).masked_fill(~vis, float("-inf"))
    m = s.amax(-1, keepdim=True)
    e = torch.exp(SCALE * (s - m))
    l = e.sum(-1)
    o = ((to_bf16(e) if rounding else e) @ v) / l[..., None]
    return o, SCALE * m[..., 0] + torch.log(l)


def exact_fwd(qkv, B, T, H, prefix=0, causal=False):
    """fp64 attention output [B*T, H*64] and lse [B, H, T] per sequence.  `prefix` does not enter the maths: the cls
    tokens are ordinary keys and queries."""
    q, k, v = heads(qkv, B, T, H, 3)
    s = (q @ k.transpose(-1, -2) * SCALE).masked_fill(~visible(T, causal, q.device), float("-inf"))
    lse = torch.logsumexp(s, -1)
    return merge(torch.exp(s - lse[..., None]) @ v), lse


def emulated_fwd(qkv, B, T, H, prefix=0, causal=False, rounding=True):
    """exact_fwd with the forward kernels' bf16 numerators (fwd_core)"""
    q, k, v = heads(qkv, B, T, H, 3)
    o, lse = fwd_core(q, k, v, visible(T, causal, q.device), rounding)
    return merge(o), lse


# --------------------------------------------------------------------------------------------------------- backward

def bwd_core(q, k, v, o, dout, lse, vis, rounded=None, delta=None):
    """Gradients (dq, dk, dv) [B,H,T,64] of softmax(SCALE q kᵀ) v with respect to the post-RoPE q, k and v, as a
    function of the forward's o and lse (the kernel's backward reads those rather than recomputing them):
        δ = Σ dO·O      P = exp(SCALE s − lse)      dS = SCALE P (dP − δ)
        dV = Pᵀ dO      dK = dSᵀ Q                  dQ = dS K
    rounded: [T, T] bool or None, the (query, key) entries whose P and dS enter a GEMM as bf16."""
    if delta is None:
        delta = (dout * o).sum(-1)
    s = (q @ k.transpose(-1, -2)).masked_fill(~vis, float("-inf"))
    p = torch.exp(SCALE * s - lse[..., None])
    ds = SCALE * p * (dout @ v.transpose(-1, -2) - delta[..., None])
    if rounded is not None:
        p = torch.where(rounded, to_bf16(p), p)
        ds = torch.where(rounded, to_bf16(ds), ds)
    return ds @ k, ds.transpose(-1, -2) @ q, p.transpose(-1, -2) @ dout


def rope_t(g, sin, cos, prefix, pos=None):
    """RoPEᵀ on gradients [B,H,T,64]: token prefix + i uses table row pos[i] (default i); prefix tokens are not rotated.
    The forward rotation is y[d] = x[d] cos[d] − x[d+32] sin[d], y[d+32] = x[d+32] cos[d+32] + x[d] sin[d+32]."""
    if sin is None:
        return g
    sn, cs = sin.to(g), cos.to(g)
    if pos is not None:
        sn, cs = sn[pos], cs[pos]
    a, b = g[..., prefix:, :32], g[..., prefix:, 32:]
    rot = torch.cat([a * cs[:, :32] + b * sn[:, 32:], b * cs[:, 32:] - a * sn[:, :32]], -1)
    return torch.cat([g[..., :prefix, :], rot], -2)


def exact_bwd(qkv_post, dout, B, T, H, prefix=0, causal=False, sin=None, cos=None):
    """fp64 gradient [B*T, 3*H*64] with respect to the PRE-RoPE qkv, from the post-RoPE qkv the kernel receives: the
    exact attention gradient with the exact fp64 O and lse, then RoPEᵀ with the (bf16) table values."""
    q, k, v = heads(qkv_post, B, T, H, 3)
    (do,) = heads(dout, B, T, H)
    vis = visible(T, causal, q.device)
    o, lse = fwd_core(q, k, v, vis, rounding=False)
    dq, dk, dv = bwd_core(q, k, v, o, do, lse, vis)
    return merge(rope_t(dq, sin, cos, prefix), rope_t(dk, sin, cos, prefix), dv)


def bwd_rounded(T, prefix, packed, device=None):
    """[T, T] entries whose P / dS are bf16 in attention_bwd.cu: all of them in packed mode; otherwise the patch-patch
    block, because the prefix key column (p0 / ds0 per query row) and the prefix query row (warp 8) stay in fp32"""
    r = torch.ones(T, T, dtype=torch.bool, device=device)
    if not packed:
        r[:prefix] = False
        r[:, :prefix] = False
    return r


def emulated_bwd(qkv_post, o, dout, lse, B, T, H, prefix=0, causal=False, sin=None, cos=None, packed=False,
                 rounding=True):
    """exact_bwd as attention_bwd.cu computes it: from the forward kernel's own o (bf16) and lse (fp32), with P and dS
    rounded to bf16 where they enter a patch-key GEMM (bwd_rounded)"""
    q, k, v = heads(qkv_post, B, T, H, 3)
    (do,) = heads(dout, B, T, H)
    (oo,) = heads(o, B, T, H)
    rounded = bwd_rounded(T, prefix, packed, q.device) if rounding else None
    dq, dk, dv = bwd_core(q, k, v, oo, do, lse.double(), visible(T, causal, q.device), rounded)
    return merge(rope_t(dq, sin, cos, prefix), rope_t(dk, sin, cos, prefix), dv)


# ----------------------------------------------------------------------------------------------------------- metric

def row_err(x, ref, rows_of):
    """Per-row relative error, shape [B, T, parts, H], of x against ref (both [B*T, parts*H*64]); rows_of = (B, T,
    parts, H).  e = ‖x − ref‖ / (‖ref‖ + f) with f = 1e-3 x the RMS row norm of ref over that part and head: rows with
    a near-zero reference (a key that causal masking almost never shows) are measured against the tensor's scale."""
    B, T, parts, H = rows_of
    d = (x.double() - ref.double()).reshape(B, T, parts, H, 64).norm(dim=-1)
    r = ref.double().reshape(B, T, parts, H, 64).norm(dim=-1)
    f = 1e-3 * r.pow(2).mean(dim=(0, 1), keepdim=True).sqrt()
    return torch.where(d == 0, torch.zeros_like(d), d / (r + f))


def whole_rel(x, ref):
    """‖x − ref‖ / ‖ref‖ over a whole tensor (what the suite checked before the per-row metric)"""
    return ((x.double() - ref.double()).norm() / (ref.double().norm() + 1e-300)).item()
