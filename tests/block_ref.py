"""Plain-torch fp64 references for the transformer block as the training step composes it (engine.attention_sublayer,
engine.ffn_sublayer, engine.tower_blocks and their backward in train.py), on the CPU or the GPU (no kernels, nothing
from oracle/).

Every stage is computed in fp64 from the values that stage receives, so that a GPU test can feed it the tensors the
kernels actually produced (tape entries, recorded intermediates) and hold each stage to the error of one kernel:
    forward    x -> h (norm) -> qkv (GEMM, RoPE) -> o, lse (attention) -> stream out (GEMM + residual)
               x -> h (norm) -> pre -> hid (GEMM + SwiGLU / GELU) -> stream out (GEMM + residual)
    backward   gb -> do -> dqkv -> dh, dW_qkv, db_qkv, dW_proj            (attention body)
               gb -> dhid -> dpre -> dh, dW_fc1, db_fc1, dW_fc2           (FFN body)
               g, recorded dh -> every gb, every bias / norm gradient, dL/dx   (tower edges, `tower_edges`)
Subset (stochastic-depth) sub-layers run on the gathered images idx and add alpha * (bf16 output) back; their backward
gathers alpha * g[idx] and scatter-adds the norm gradient back into g[idx].

Rounding points are those of the kernels: bf16 GEMM outputs, the RoPE products and sum (`rope_fwd`), the attention
kernels' bf16 P / dS (attn_ref), swiglu_fwd's two roundings (step_ref).  With `rounding=False` (and fp64 inputs) the
composed references `sublayer_fwd` / `body_bwd` / `tower_edges` are the exact chain rule of the block, which
tests/test_block_ref_cpu.py checks against fp64 autograd.

Checkers (tests/test_block_sublayers_gpu.py applies them per row, so a failure names its rows and 128-row tiles):
slack_k  |got − ref| ≤ slack + k·2⁻²⁴·scale per element, where `slack` is one bf16 ulp of every value the kernel rounds
         on the way (its own output, the sub-layer output inside a residual sum, RoPE's products) and `scale` the
         magnitude of the terms summed in fp32; reduces to step_ref.elem_k for a single rounding.
col_rows step_ref.col_k per row of a reduction (weight gradients: one row per output feature).
Per-row attention errors use attn_ref.row_err.

Bounds, against the largest value measured over four runs of every case of the GPU file on an H100 80GB HBM3 (700 W
power limit); the weight gradients and column sums vary from run to run (fp32 atomics), nothing else does:
    bound          value    measured maxima
    LIN_K          13       dh 6.69 (VTP-Large FFN), stream out 4.64, subset output 2.73, qkv before RoPE 2.13,
                            do 2.10, pre 1.95, dhid 1.81, qkv 0.80
    ROPE_K         1.8      qkv with RoPE in the epilogue 0.88; stand-alone RoPE bit-exact
    WGRAD_K        72       fc1_w 35.6 (VTP-Large, ragged N / K tiles), qkv_w 20.2, fc2_w 16.7, proj_w 11.4; at
                            VTP-Small width at most 10.5.  Hopper's fp32 wgmma accumulation over thousands of rows;
                            one dropped 64-row tile of the 131 584-row trunk wgrad is k ~ 8000
    EDGE_K         0.4      dL/dx 0.19 (subset path), gb 0.038
    DQKV_ROW_TOL   2⁻⁶      dq 8.3e-3, dk 7.8e-3, dv 6.8e-3 (attn_ref.row_err).  One dq row of the 512 x 257 trunk is
                            above attn_ref.BWD_ROW_TOL (2⁻⁷), which was set from random-input rows
    LSE_TOL        8e-7     lse 3.7e-7 (relative, at least absolute)
    NORM_FWD_K     6        rstd 2.88, h 0.14, mean 0.03                  = step_ref.NORM_FWD_K
    ACT_K          0.5      hid 0.28 (GELU epilogue), dpre 0.21           = step_ref.ACT_K
    COL_K          5        qkv_b 3.30, fc1_b 2.71, n2_w 1.72, proj_b 1.59 = step_ref.COL_K
    FWD_ROW_TOL    5.4e-3   o 4.0e-3                                      = attn_ref.FWD_ROW_TOL
The whole file takes about 30 s on one H100 80GB HBM3 (700 W).
"""
import math

import torch

from tests import attn_ref as ar
from tests import step_ref as sr

U24 = sr.U24
LIN_K = 13.0        # GEMM outputs: qkv, pre, the stream, do, dhid, dh
ROPE_K = 1.8        # qkv with RoPE applied in the GEMM epilogue
WGRAD_K = 72.0      # split-K weight gradients
EDGE_K = 0.4        # the dY operands gb and dL/dx, from the fp64 stream gradient
DQKV_ROW_TOL = 2.0 ** -6
LSE_TOL = 8e-7
NORM_FWD_K, ACT_K, COL_K = sr.NORM_FWD_K, sr.ACT_K, sr.COL_K
FWD_ROW_TOL = ar.FWD_ROW_TOL

# ---------------------------------------------------------------------------------------------------------- checkers

def _rowmax(k):
    return k.reshape(k.shape[0], -1).amax(1) if k.dim() > 1 else k


def slack_k(got, ref, slack, scale):
    """per row: max over its elements of the k with |got − ref| ≤ slack + k·2⁻²⁴·scale (inf where got is not finite, or
    an error remains where scale is 0)"""
    got, ref = got.double(), ref.double()
    d = (got - ref).abs()
    ex = (d - torch.as_tensor(slack, dtype=torch.float64, device=d.device)).clamp(min=0)
    s = torch.as_tensor(scale, dtype=torch.float64, device=d.device).expand_as(d)
    k = torch.where(ex == 0, torch.zeros_like(ex), ex / (U24 * s))
    k = torch.where(torch.isfinite(got), k, torch.full_like(k, math.inf))
    return _rowmax(k)


def col_rows(got, ref, abs_sum):
    """per row of a reduction's output: max of |got − ref| / (2⁻²⁴ Σ|terms|)"""
    got, ref = got.double(), ref.double()
    d = (got - ref).abs()
    s = torch.as_tensor(abs_sum, dtype=torch.float64, device=d.device).expand_as(d)
    k = torch.where(d == 0, torch.zeros_like(d), d / (U24 * s))
    k = torch.where(torch.isfinite(got), k, torch.full_like(k, math.inf))
    return _rowmax(k)


def image_rows(idx, T):
    """token rows of the images idx in a [n*T, D] stream"""
    return (idx.long()[:, None] * T + torch.arange(T, device=idx.device)).reshape(-1)


# -------------------------------------------------------------------------------------------------------- linears

def linear(a, w, b=None, resid=None, stream_bf16=False):
    """a forward GEMM: round(a·wᵀ + b) (+ resid, rounded again for a bf16 stream) -> (ref, slack, scale), ref in fp64
    without roundings"""
    y = a.double() @ w.double().t()
    scale = a.double().abs() @ w.double().abs().t()
    if b is not None:
        y = y + b.double()
        scale = scale + b.double().abs()
    slack = sr.ulp_bf16(y)
    if resid is not None:
        y = y + resid.double()
        scale = scale + resid.double().abs()
        if stream_bf16:
            slack = slack + sr.ulp_bf16(y)
    return y, slack, scale


def subset_out(x, y, slack, scale, idx, alpha, T):
    """x + alpha·scatter(idx, round(y)): a subset sub-layer's bf16 output y (with its linear() slack / scale) added into
    a copy of the fp32 stream x -> (ref, slack, scale)"""
    rows = image_rows(idx, T)
    out, sl, sc = x.double().clone(), torch.zeros_like(x, dtype=torch.float64), x.double().abs()
    out[rows] += alpha * y
    sl[rows] += alpha * slack
    sc[rows] += alpha * scale
    return out, sl, sc


def dgrad(dy, w):
    """dY·W into bf16 -> (ref, slack, scale)"""
    y = dy.double() @ w.double()
    return y, sr.ulp_bf16(y), dy.double().abs() @ w.double().abs()


def wgrad(dy, x):
    """dYᵀ·X (accumulated by the kernel onto its pre-filled fp32 buffer) -> (sum, Σ|terms|)"""
    return dy.double().t() @ x.double(), dy.double().abs().t() @ x.double().abs()


def colsum(t):
    return t.double().sum(0), t.double().abs().sum(0)


# ----------------------------------------------------------------------------------------------------------- RoPE

def _halves(qkv, T, prefix):
    """[n*T, 3D] -> view [n, T - prefix, 2 (q|k), H, 2 (halves), 32] of the rotated entries"""
    M, N = qkv.shape
    return qkv.reshape(M // T, T, 3, N // 192, 2, 32)[:, prefix:, :2]


def rope_fwd(qkv, sin, cos, T, prefix, rounding=True, absolute=False):
    """the q and k thirds of qkv [n*T, 3D] rotated per 64-wide head, token prefix + i by table row i (sin / cos
    [T − prefix, 64]; prefix tokens unrotated): y_lo = a·cos_lo − b·sin_lo, y_hi = b·cos_hi + a·sin_hi for the halves
    a, b.  rounding (bf16 qkv): rope_fwd_kernel and the GEMM's RoPE epilogue, bit for bit: each product of two bf16
    values rounded to bf16, their sum formed in fp32 and rounded to bf16.  Otherwise fp64; absolute: both terms added
    (the magnitude |a||cos| + |b||sin| for absolute inputs)."""
    dt = torch.float32 if rounding else torch.float64
    out = qkv.to(dt).clone()
    v = _halves(qkv.to(dt), T, prefix)
    a, b = v[..., 0, :], v[..., 1, :]
    s = sin.to(dt).reshape(T - prefix, 1, 1, 2, 32)
    c = cos.to(dt).reshape(T - prefix, 1, 1, 2, 32)
    r = sr.bf16 if rounding else (lambda t: t)
    o = _halves(out, T, prefix)
    o[..., 0, :] = r(a * c[..., 0, :]) + (1 if absolute else -1) * r(b * s[..., 0, :])
    o[..., 1, :] = r(b * c[..., 1, :]) + r(a * s[..., 1, :])
    return out.to(torch.bfloat16) if rounding else out


def rope_bounds(qkv, scale, sin, cos, T, prefix):
    """(slack, scale) of rope_fwd(round(qkv)) against fp64 rope_fwd(qkv, rounding=False), qkv the fp64 GEMM value with
    its linear() scale: the rounding of qkv (≤ one ulp of each product), of the two products and of the sum, and the
    GEMM's fp32 error carried through the rotation"""
    mag = rope_fwd(qkv.abs(), sin.abs(), cos.abs(), T, prefix, rounding=False, absolute=True)
    y = rope_fwd(qkv, sin, cos, T, prefix, rounding=False)
    slack = 3 * sr.ulp_bf16(mag) + sr.ulp_bf16(y)
    slack = torch.where(_rotated(qkv, T, prefix), slack, sr.ulp_bf16(qkv))
    return slack, rope_fwd(scale, sin.abs(), cos.abs(), T, prefix, rounding=False, absolute=True)


def _rotated(qkv, T, prefix):
    m = torch.zeros(qkv.shape, dtype=torch.bool, device=qkv.device)
    _halves(m, T, prefix)[...] = True
    return m


def rope_t(dqkv, sin, cos, n, T, H, prefix):
    """RoPEᵀ of the q and k thirds of a post-RoPE gradient [n*T, 3D] (attn_ref.rope_t), fp64"""
    q, k, v = ar.heads(dqkv, n, T, H, 3)
    return ar.merge(ar.rope_t(q, sin, cos, prefix), ar.rope_t(k, sin, cos, prefix), v)


# ------------------------------------------------------------------------------------------------------ attention

def _chunk(H, T):
    return max(1, (1 << 25) // (H * T * T))   # images per fp64 [c, H, T, T] block of 256 MB


def attention_fwd(qkv, n, T, H, causal, rounding=True):
    """attn_ref.emulated_fwd in chunks of images -> (o [n*T, D] fp64, lse [n, H, T])"""
    c = _chunk(H, T)
    os, ls = [], []
    for i in range(0, n, c):
        m = min(c, n - i)
        o, lse = ar.emulated_fwd(qkv[i * T:(i + m) * T], m, T, H, 0, causal, rounding)
        os.append(o)
        ls.append(lse)
    return torch.cat(os), torch.cat(ls)


def attention_bwd(qkv, o, dout, lse, n, T, H, prefix, causal, rope, rounding=True):
    """attn_ref.emulated_bwd in chunks of images: dL/d(pre-RoPE qkv) [n*T, 3D] fp64 from the post-RoPE qkv, the
    forward's o and lse and dout; the packed / unpacked rounding pattern is that of the whole call"""
    sin, cos = rope if rope is not None else (None, None)
    packed = ar.bwd_packed(n, T, causal)
    c = _chunk(H, T)
    out = []
    for i in range(0, n, c):
        m = min(c, n - i)
        r = slice(i * T, (i + m) * T)
        out.append(ar.emulated_bwd(qkv[r], o[r], dout[r], lse[i:i + m], m, T, H, prefix, causal, sin, cos, packed,
                                   rounding))
    return torch.cat(out)


def lse_err(lse, ref):
    """max |lse − ref| / max(|ref|, 1)"""
    return ((lse.double() - ref.double()).abs() / ref.double().abs().clamp(min=1.0)).max().item()


# ------------------------------------------------------------------------------------------------------- FFN gates

def gelu_fwd(pre):
    """exact-erf GELU of the bf16 pre-activation -> (hid fp64, scale)"""
    x = pre.double()
    return 0.5 * x * (1 + torch.erf(x / math.sqrt(2))), x.abs() + 1e-30


def swiglu_exact(pre, Hs):
    """silu(x1)·x2 of the 8-interleaved pre-activation, fp64 without roundings"""
    x1, x2 = [t.double() for t in sr.split8(pre, Hs)]
    return x1 * torch.sigmoid(x1) * x2


# ------------------------------------------------------------------------------- composed references (chain rule)

def sublayer_fwd(kind, p, cfg, x, n, T, rounding=True):
    """One sub-layer forward composed from the stage references, each fed the previous stage's reference (no
    resid).  cfg: dict(H, eps, prefix, ffn, hidden, causal, rope=(sin, cos) | None).  -> tape-like dict with 'y', the
    sub-layer's output before the residual"""
    nw, nb = (p["n1_w"], p["n1_b"]) if kind == "attn" else (p["n2_w"], p["n2_b"])
    h, rstd, mean, _ = sr.norm_fwd(x, nw, nb, cfg["eps"])
    r = sr.bf16 if rounding else (lambda t: t)
    e = dict(x=x, rstd=rstd, mean=None if nb is None else mean, h=r(h))
    if kind == "attn":
        qkv = r(linear(e["h"], p["qkv_w"], p["qkv_b"])[0])
        if cfg["rope"] is not None:
            qkv = rope_fwd(qkv, *cfg["rope"], T, cfg["prefix"], rounding).double()
        o, lse = attention_fwd(qkv, n, T, cfg["H"], cfg["causal"], rounding)
        e.update(qkv=qkv, o=r(o), lse=lse)
        e["y"] = linear(e["o"], p["proj_w"], p["proj_b"])[0]
    else:
        pre = r(linear(e["h"], p["fc1_w"], p["fc1_b"])[0])
        if cfg["ffn"] == "swiglu":
            hid = sr.swiglu_fwd(pre, cfg["hidden"])[0] if rounding else swiglu_exact(pre, cfg["hidden"])
        else:
            hid = r(gelu_fwd(pre)[0])
        e.update(pre=pre, hid=hid)
        e["y"] = linear(hid, p["fc2_w"], p["fc2_b"])[0]
    return e


def body_bwd(kind, p, cfg, e, gb, n, T, rounding=True):
    """The backward body of one sub-layer composed from the stage references: gb (dL/d of its last GEMM's output)
    -> dict(dh, inner stage values, and the weight / bias gradients as (sum, Σ|terms|))"""
    r = sr.bf16 if rounding else (lambda t: t)
    if kind == "attn":
        do = r(dgrad(gb, p["proj_w"])[0])
        dqkv = r(attention_bwd(e["qkv"], e["o"], do, e["lse"], n, T, cfg["H"], cfg["prefix"], cfg["causal"],
                               cfg["rope"], rounding))
        return dict(do=do, dqkv=dqkv, dh=r(dgrad(dqkv, p["qkv_w"])[0]), proj_w=wgrad(gb, e["o"]),
                    qkv_w=wgrad(dqkv, e["h"]), qkv_b=colsum(dqkv))
    dhid = r(dgrad(gb, p["fc2_w"])[0])
    if cfg["ffn"] == "swiglu":
        dpre, _, db, dba = sr.swiglu_bwd(e["pre"], dhid, cfg["hidden"])
    else:
        dpre, _, db, dba = sr.gelu_bwd(e["pre"], dhid)
    dpre = r(dpre)
    return dict(dhid=dhid, dpre=dpre, dh=r(dgrad(dpre, p["fc1_w"])[0]), fc2_w=wgrad(gb, e["hid"]),
                fc1_w=wgrad(dpre, e["h"]), fc1_b=(db, dba))


# --------------------------------------------------------------------------------------------------- tower edges

def edge_order(depth):
    """(block, sub-layer) in the order the backward runs them"""
    return [(li, kind) for li in reversed(range(depth)) for kind in ("ffn", "attn")]


def last_bias(kind):
    return "fc2_b" if kind == "ffn" else "proj_b"


def tower_edges(entries, norm_ws, body, g_out, T, depth):
    """The fp32 stream gradient through the backward's edges, in fp64, from the recorded body outputs.
    entries / norm_ws: the tape entry (x, rstd, mean, subset) and norm weight of every sub-layer in edge_order;
    body(i, gs) -> the dh of sub-layer i (the recorded one, or body_bwd of its operand gs); g_out = dL/d(stream out).  Plain sub-layer: its dY operand is g itself (gb = bf16(g)); subset: alpha·g
    on its images.  Either way the operand's column sum is the gradient of the sub-layer's last bias; its norm gradient
    (norm_bwd of dh into zeros) is then added to g, on the subset's images for a subset.
    -> dict(gs: [dY operand (fp64)], gs_scale, bias: {(li, key): (sum, Σ|terms|)}, norm: {(li, key): (sum, Σ|·|)}, g,
            g_scale)"""
    g = g_out.double().clone()
    gsc = g.abs()
    out = dict(gs=[], gs_scale=[], bias={}, norm={})
    for i, ((li, kind), e, w) in enumerate(zip(edge_order(depth), entries, norm_ws)):
        sub = e["subset"]
        rows = None if sub is None else image_rows(sub[0], T)
        alpha = 1.0 if sub is None else sub[1]
        gs = g if rows is None else alpha * g[rows]
        ss = gsc if rows is None else alpha * gsc[rows]
        out["gs"].append(gs.clone())
        out["gs_scale"].append(ss.clone())
        out["bias"][(li, last_bias(kind))] = colsum(gs)
        dh = body(i, gs)
        nb = sr.norm_bwd(e["x"], e["rstd"], e["mean"], w, dh, torch.zeros_like(e["x"], dtype=torch.float64))
        n = "n1" if kind == "attn" else "n2"
        out["norm"][(li, n + "_w")] = (nb["dw"], nb["dw_abs"])
        out["norm"][(li, n + "_b")] = (nb["db"], nb["db_abs"])
        if rows is None:
            g = g + nb["g"]
            gsc = gsc + nb["g_scale"]
        else:
            g = g.index_add(0, rows, nb["g"])
            gsc = gsc.index_add(0, rows, nb["g_scale"])
    out["g"], out["g_scale"] = g, gsc
    return out


# ------------------------------------------------------------------------------------------------------ stage checks

def _rows_of_heads(e):
    """[n, T, parts, H] per-head errors -> per token row"""
    return e.amax((2, 3)).reshape(-1)


def check_forward(kind, p, cfg, e, x_in, x_out, T, qkv_pre=None, res=None):
    """Every forward stage of one sub-layer from its tape entry e, each from the recorded value that fed it
    -> [(name, value per row, bound)].  x_in / x_out: the stream before and after the sub-layer (x_in is e["x"] unless
    the sub-layer ran on a subset); qkv_pre: the qkv GEMM's output before a stand-alone RoPE pass (None: RoPE in the
    epilogue, or none); res: a subset sub-layer's bf16 output, before the scatter."""
    out = []
    nw, nb = (p["n1_w"], p["n1_b"]) if kind == "attn" else (p["n2_w"], p["n2_b"])
    D = e["x"].shape[1]
    n = e["x"].shape[0] // T
    y, rstd, mean, sc = sr.norm_fwd(e["x"], nw, nb, cfg["eps"], rstd_kernel=e["rstd"])
    out.append(("h", slack_k(e["h"], y, sr.ulp_bf16(y), sc), NORM_FWD_K))
    out.append(("rstd", slack_k(e["rstd"], rstd, 0, rstd), NORM_FWD_K))
    if nb is not None:
        out.append(("mean", slack_k(e["mean"], mean, 0, e["x"].double().abs().mean(1) * D ** 0.5), NORM_FWD_K))
    if kind == "attn":
        q, sl, sc = linear(e["h"], p["qkv_w"], p["qkv_b"])
        rope = cfg["rope"]
        if rope is None:
            out.append(("qkv", slack_k(e["qkv"], q, sl, sc), LIN_K))
        elif qkv_pre is not None:
            out.append(("qkv before RoPE", slack_k(qkv_pre, q, sl, sc), LIN_K))
            same = (e["qkv"] == rope_fwd(qkv_pre, *rope, T, cfg["prefix"])).all(1)
            out.append(("qkv RoPE (bit-exact)", torch.where(same, 0.0, math.inf).double(), 0.0))
        else:
            sl, sc = rope_bounds(q, sc, *rope, T, cfg["prefix"])
            out.append(("qkv with RoPE in the epilogue",
                        slack_k(e["qkv"], rope_fwd(q, *rope, T, cfg["prefix"], rounding=False), sl, sc), ROPE_K))
        o, lse = attention_fwd(e["qkv"], n, T, cfg["H"], cfg["causal"])
        out.append(("o", _rows_of_heads(ar.row_err(e["o"], o, (n, T, 1, cfg["H"]))), FWD_ROW_TOL))
        le = (e["lse"].double() - lse).abs() / lse.abs().clamp(min=1.0)
        out.append(("lse", le.amax(1).reshape(-1), LSE_TOL))
        a, w, b = e["o"], p["proj_w"], p["proj_b"]
    else:
        pr, sl, sc = linear(e["h"], p["fc1_w"], p["fc1_b"])
        out.append(("pre", slack_k(e["pre"], pr, sl, sc), LIN_K))
        if cfg["ffn"] == "swiglu":
            hid, alt, hsc = sr.swiglu_fwd(e["pre"], cfg["hidden"])
            hid = torch.where((e["hid"].double() - alt).abs() < (e["hid"].double() - hid).abs(), alt, hid)
            out.append(("hid", slack_k(e["hid"], hid, 0, hsc), ACT_K))
        else:
            hid, hsc = gelu_fwd(e["pre"])
            out.append(("hid", slack_k(e["hid"], hid, sr.ulp_bf16(hid), hsc), ACT_K))
        a, w, b = e["hid"], p["fc2_w"], p["fc2_b"]
    if e["subset"] is None:
        ref = linear(a, w, b, resid=x_in, stream_bf16=cfg["stream_bf16"])
        out.append(("stream out", slack_k(x_out, *ref), LIN_K))
    else:
        idx, alpha = e["subset"]
        ys = linear(a, w, b)
        out.append(("subset output", slack_k(res, *ys), LIN_K))
        out.append(("stream out", slack_k(x_out, *subset_out(x_in, *ys, idx, alpha, T)), LIN_K))
    return out


def check_body(kind, p, cfg, e, rec, T):
    """The backward body of one sub-layer, each stage from the recorded value that fed it.  rec: gb, dh and do, dqkv
    (attention) or dhid, dpre (FFN).  -> ([(name, value per row, bound)], {weight key: (sum, Σ|terms|)})"""
    n = e["x"].shape[0] // T
    gb = rec["gb"]
    if kind == "attn":
        dqkv = attention_bwd(e["qkv"], e["o"], rec["do"], e["lse"], n, T, cfg["H"], cfg["prefix"], cfg["causal"],
                             cfg["rope"])
        err = ar.row_err(rec["dqkv"], dqkv, (n, T, 3, cfg["H"]))
        checks = [("do", slack_k(rec["do"], *dgrad(gb, p["proj_w"])), LIN_K)]
        checks += [(part, _rows_of_heads(err[:, :, i:i + 1]), DQKV_ROW_TOL) for i, part in enumerate(("dq", "dk", "dv"))]
        checks.append(("dh", slack_k(rec["dh"], *dgrad(rec["dqkv"], p["qkv_w"])), LIN_K))
        return checks, dict(proj_w=wgrad(gb, e["o"]), qkv_w=wgrad(rec["dqkv"], e["h"]), qkv_b=colsum(rec["dqkv"]))
    if cfg["ffn"] == "swiglu":
        dpre, dsc, db, dba = sr.swiglu_bwd(e["pre"], rec["dhid"], cfg["hidden"])
    else:
        dpre, dsc, db, dba = sr.gelu_bwd(e["pre"], rec["dhid"])
    checks = [("dhid", slack_k(rec["dhid"], *dgrad(gb, p["fc2_w"])), LIN_K),
              ("dpre", slack_k(rec["dpre"], dpre, sr.ulp_bf16(dpre), dsc), ACT_K),
              ("dh", slack_k(rec["dh"], *dgrad(rec["dpre"], p["fc1_w"])), LIN_K)]
    return checks, dict(fc2_w=wgrad(gb, e["hid"]), fc1_w=wgrad(rec["dpre"], e["h"]), fc1_b=(db, dba))


def check_backward(P, cfg, entries, recs, g_out, g, grads, prefill, T):
    """The whole tower backward from what it recorded.  P: per-block weights; entries / recs: tape entry and record of
    every sub-layer in edge_order; g_out / g: the stream gradient before and after; grads / prefill: {(block, key):
    tensor} of the gradient buffers after the backward and before it.  -> [(name, value per row, bound)]"""
    depth = len(P)
    order = edge_order(depth)
    norm_ws = [P[li]["n1_w" if kind == "attn" else "n2_w"] for li, kind in order]
    edges = tower_edges(entries, norm_ws, lambda i, gs: recs[i]["dh"], g_out, T, depth)
    out = []
    total = {k: (v.double().clone(), v.double().abs()) for k, v in prefill.items()}

    def acc(key, sa):
        s, a = total[key]
        total[key] = (s + sa[0], a + sa[1])

    for i, ((li, kind), e, rec) in enumerate(zip(order, entries, recs)):
        name = f"block {li} {kind}"
        gs = edges["gs"][i]
        out.append((f"{name} gb", slack_k(rec["gb"], gs, sr.ulp_bf16(gs), edges["gs_scale"][i]), EDGE_K))
        checks, contrib = check_body(kind, P[li], cfg, e, rec, T)
        out += [(f"{name} {c}", v, b) for c, v, b in checks]
        for key, sa in contrib.items():
            acc((li, key), sa)
    for key, sa in list(edges["bias"].items()) + list(edges["norm"].items()):
        if key in total:
            acc(key, sa)
    for (li, key), (s, a) in total.items():
        bound = WGRAD_K if key.endswith("_w") and not key.startswith("n") else COL_K
        out.append((f"block {li} grad {key}", col_rows(grads[(li, key)], s, a), bound))
    out.append(("dL/dx", slack_k(g, edges["g"], 0, edges["g_scale"]), EDGE_K))
    return out
