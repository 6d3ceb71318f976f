"""The block references of tests/block_ref.py and their checkers, proved without a GPU, at tiny shapes (D 128, 2 heads,
depth 2): an RMSNorm + SwiGLU tower with a cls prefix and RoPE (T 17), and a LayerNorm + GELU causal tower (T 37).

- With every rounding point off, the composed references (sublayer_fwd, body_bwd, tower_edges) equal fp64 autograd of
  a plain torch restatement of the blocks, on the plain path and on the subset path (index_add with alpha), to 1e-12.
- A stand-in for the kernels, written like train.tower_blocks_backward and built from the rounded references, passes
  check_forward / check_backward; each seeded composition bug below makes them fail by at least 10x a bound, and the
  test prints the margin.
"""
import pytest
import torch
import torch.nn.functional as F

from tests import block_ref as br
from tests import step_ref as sr

D64 = torch.float64
D, H, DEPTH = 128, 2, 2
TOWERS = {
    "rms_swiglu_rope": dict(norm="rms", ffn="swiglu", hidden=96, prefix=1, grid=(4, 4), causal=False, eps=1e-5),
    "ln_gelu_causal": dict(norm="ln", ffn="gelu", hidden=256, prefix=0, T=37, causal=True, eps=1e-5),
}
MARGIN = 10.0


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _tower(name, n=4):
    """(per-block weights, cfg, T, n): bf16-representable fp64 weights, so that the rounded stand-in below computes
    what a kernel would"""
    t = TOWERS[name]
    g = _g(len(name))
    T = t["grid"][0] * t["grid"][1] + t["prefix"] if "grid" in t else t["T"]
    Hd = t["hidden"]
    n1 = 2 * Hd if t["ffn"] == "swiglu" else Hd
    r = lambda *s, sc=1.0: sr.bf16(torch.randn(*s, generator=g, dtype=D64) * sc)
    ln = t["norm"] == "ln"
    P = []
    for _ in range(DEPTH):
        P.append(dict(n1_w=1 + r(D, sc=0.2), n1_b=r(D, sc=0.1) if ln else None, qkv_w=r(3 * D, D, sc=1.2 / D ** 0.5),
                      qkv_b=r(3 * D, sc=0.1), proj_w=r(D, D, sc=D ** -0.5), proj_b=r(D, sc=0.1),
                      n2_w=1 + r(D, sc=0.2), n2_b=r(D, sc=0.1) if ln else None, fc1_w=r(n1, D, sc=D ** -0.5),
                      fc1_b=r(n1, sc=0.1), fc2_w=r(D, Hd, sc=Hd ** -0.5), fc2_b=r(D, sc=0.1)))
    rope = None
    if "grid" in t:
        ang = torch.rand(T - t["prefix"], 64, generator=g, dtype=D64) * 6.28
        rope = (sr.bf16(torch.sin(ang)), sr.bf16(torch.cos(ang)))
    cfg = dict(H=H, eps=t["eps"], prefix=t["prefix"], ffn=t["ffn"], hidden=Hd, causal=t["causal"], rope=rope,
               stream_bf16=False)
    return P, cfg, T, n


def _subsets(n, on):
    """a subset (unsorted, with the first and the last image) for every sub-layer, or None everywhere"""
    if not on:
        return {(li, k): None for li in range(DEPTH) for k in ("attn", "ffn")}
    picks = [[n - 1, 0], [2, 0, 3], [1], [3, 1]]
    return {(li, k): (torch.tensor(picks[2 * li + j]), n / len(picks[2 * li + j]))
            for li in range(DEPTH) for j, k in enumerate(("attn", "ffn"))}


# ---------------------------------------------------------------------------------------------- torch restatement

def _torch_sublayer(kind, p, cfg, x, m, T):
    w, b = (p["n1_w"], p["n1_b"]) if kind == "attn" else (p["n2_w"], p["n2_b"])
    eps = sr.f32(cfg["eps"])
    h = F.layer_norm(x, (D,), w, b, eps) if b is not None else x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps) * w
    if kind == "ffn":
        pre = F.linear(h, p["fc1_w"], p["fc1_b"])
        if cfg["ffn"] == "swiglu":
            x1, x2 = sr.split8(pre, cfg["hidden"])
            hid = F.silu(x1) * x2
        else:
            hid = F.gelu(pre)
        return F.linear(hid, p["fc2_w"], p["fc2_b"])
    q, k, v = F.linear(h, p["qkv_w"], p["qkv_b"]).view(m, T, 3, H, 64).permute(2, 0, 3, 1, 4)
    if cfg["rope"] is not None:
        sin, cos = cfg["rope"]
        pf = cfg["prefix"]

        def rot(t):  # layers/attention.py: x * cos + rotate_half(x) * sin on the patch tokens
            a = t[:, :, pf:]
            half = torch.cat([-a[..., 32:], a[..., :32]], -1)
            return torch.cat([t[:, :, :pf], a * cos + half * sin], 2)
        q, k = rot(q), rot(k)
    s = (q @ k.transpose(-1, -2)) * 0.125
    if cfg["causal"]:
        s = s.masked_fill(~torch.ones(T, T, dtype=torch.bool).tril(), float("-inf"))
    o = (s.softmax(-1) @ v).transpose(1, 2).reshape(m * T, D)
    return F.linear(o, p["proj_w"], p["proj_b"])


def _torch_tower(P, cfg, x, n, T, subsets):
    for li, p in enumerate(P):
        for kind in ("attn", "ffn"):
            sub = subsets[(li, kind)]
            if sub is None:
                x = x + _torch_sublayer(kind, p, cfg, x, n, T)
            else:
                idx, alpha = sub
                xs = x.view(n, T, D)[idx].reshape(-1, D)
                y = _torch_sublayer(kind, p, cfg, xs, idx.numel(), T)
                x = x.view(n, T, D).index_add(0, idx, y.view(-1, T, D), alpha=alpha).reshape(n * T, D)
    return x


# ----------------------------------------------------------------------------------- composed reference / stand-in

def _forward(P, cfg, x, n, T, subsets, rounding, bug=None):
    """the tower forward from block_ref.sublayer_fwd: -> ({(block, kind): tape entry}, {(block, kind): (x_in, x_out,
    subset output)}, stream out).  rounding: a kernel stand-in (bf16 sub-layer outputs)."""
    r = sr.bf16 if rounding else (lambda t: t)
    entries, streams = {}, {}
    for li in range(len(P)):
        for kind in ("attn", "ffn"):
            sub = subsets[(li, kind)]
            if sub is None:
                e = br.sublayer_fwd(kind, P[li], cfg, x, n, T, rounding)
                x_out = x + r(e["y"])
                res = None
            else:
                idx, alpha = sub
                rows = br.image_rows(idx, T)
                e = br.sublayer_fwd(kind, P[li], cfg, x[rows], idx.numel(), T, rounding)
                res = r(e["y"])
                a = {"alpha_missing": 1.0, "alpha_doubled": alpha * alpha}.get(bug, alpha)
                x_out = x.index_add(0, rows, a * res)
            e["subset"] = sub
            entries[(li, kind)] = e
            streams[(li, kind)] = (x, x_out, res)
            x = x_out
    return entries, streams, x


def _stand_in_backward(P, cfg, entries, g_out, T, prefill, bug=None):
    """train.tower_blocks_backward restated on the rounded references, with one seeded bug -> (records in edge order,
    gradient buffers, dL/dx)"""
    g = g_out.clone()
    grads = {k: v.clone() for k, v in prefill.items()}
    recs, gb_next = [], None
    for li, kind in br.edge_order(len(P)):
        e, p = entries[(li, kind)], P[li]
        sub = e["subset"]
        if sub is None:
            gs = g
        else:
            idx, alpha = sub
            rows = br.image_rows(idx, T)
            a = {"alpha_missing": 1.0, "alpha_doubled": alpha * alpha}.get(bug, alpha)
            gs = a * g[rows]
        gb = gb_next if sub is None and gb_next is not None else sr.bf16(gs)
        bias = (li, br.last_bias(kind))
        if bug == "bias_to_wrong_block" and kind == "ffn" and li + 1 < len(P):
            bias = (li + 1, "fc2_b")   # the column sum from block li + 1's attention backward kept in that block
        grads[bias] = grads[bias] + gs.sum(0)
        m = e["x"].shape[0] // T
        c = dict(cfg, rope=None) if bug == "rope_transpose_missing" and kind == "attn" else cfg
        out = br.body_bwd(kind, p, c, e, gb, m, T)
        if kind == "attn":
            if bug == "proj_wgrad_reads_h":
                out["proj_w"] = br.wgrad(gb, e["h"])
            if bug == "qkv_bias_without_cls":
                keep = (torch.arange(m * T) % T) >= cfg["prefix"]
                out["qkv_b"] = br.colsum(out["dqkv"][keep])
            if bug == "wgrad_tile_dropped":
                out["qkv_w"] = br.wgrad(out["dqkv"][64:], e["h"][64:])
            rec = dict(gb=gb, dh=out["dh"], do=out["do"], dqkv=out["dqkv"])
            keys = ("proj_w", "qkv_w", "qkv_b")
        else:
            rec = dict(gb=gb, dh=out["dh"], dhid=out["dhid"], dpre=out["dpre"])
            keys = ("fc2_w", "fc1_w", "fc1_b")
        for k in keys:
            grads[(li, k)] = grads[(li, k)] + out[k][0]
        recs.append(rec)
        pre = "n1" if kind == "attn" else "n2"
        nb = sr.norm_bwd(e["x"], e["rstd"], e["mean"], p[pre + "_w"], out["dh"], torch.zeros_like(e["x"]))
        grads[(li, pre + "_w")] = grads[(li, pre + "_w")] + nb["dw"]
        if (li, pre + "_b") in grads:
            grads[(li, pre + "_b")] = grads[(li, pre + "_b")] + nb["db"]
        if sub is None:
            g_new = nb["g"] if bug == "norm_bwd_overwrites_g" else g + nb["g"]
            gb_next = sr.bf16(g if bug == "gb_before_norm_grad" else g_new)
            g = g_new
        else:
            back = idx.roll(1) if bug == "subset_permuted_idx" else idx
            g = g.index_add(0, br.image_rows(back, T), nb["g"])
            gb_next = None
    return recs, grads, g


def _prefill(P, g):
    return {(li, k): torch.randn(v.shape, generator=g, dtype=D64) * 0.5 for li, p in enumerate(P)
            for k, v in p.items() if v is not None}


# ------------------------------------------------------------------------------------------------------ chain rule

# stochastic depth runs on the vision trunk only (engine.tower_blocks)
PATHS = [("rms_swiglu_rope", False), ("rms_swiglu_rope", True), ("ln_gelu_causal", False)]
PATH_IDS = ["rms_swiglu_rope-plain", "rms_swiglu_rope-subset", "ln_gelu_causal-plain"]


@pytest.mark.parametrize("tower,subset", PATHS, ids=PATH_IDS)
def test_composed_references_match_autograd(tower, subset):
    P, cfg, T, n = _tower(tower)
    subsets = _subsets(n, subset)
    g = _g(5)
    x0 = torch.randn(n * T, D, generator=g, dtype=D64)
    g_out = torch.randn(n * T, D, generator=g, dtype=D64)

    leaves = [{k: (v.clone().requires_grad_(True) if v is not None else None) for k, v in p.items()} for p in P]
    x = x0.clone().requires_grad_(True)
    y = _torch_tower(leaves, cfg, x, n, T, subsets)
    (y * g_out).sum().backward()

    entries, _, y_ref = _forward(P, cfg, x0, n, T, subsets, rounding=False)
    assert (y_ref - y.detach()).abs().max() <= 1e-12 * y.detach().abs().max()
    order = br.edge_order(DEPTH)
    wg = {}

    def body(i, gs):
        li, kind = order[i]
        e = entries[(li, kind)]
        out = br.body_bwd(kind, P[li], cfg, e, gs, e["x"].shape[0] // T, T, rounding=False)
        for k in ("proj_w", "qkv_w", "qkv_b", "fc2_w", "fc1_w", "fc1_b"):
            if k in out:
                wg[(li, k)] = out[k][0]
        return out["dh"]

    norm_ws = [P[li]["n1_w" if kind == "attn" else "n2_w"] for li, kind in order]
    edges = br.tower_edges([entries[o] for o in order], norm_ws, body, g_out, T, DEPTH)
    got = dict(wg)
    got.update({k: v[0] for k, v in edges["bias"].items()})
    got.update({k: v[0] for k, v in edges["norm"].items()})
    worst = 0.0
    for li, p in enumerate(leaves):
        for k, v in p.items():
            if v is not None:
                ref = v.grad
                worst = max(worst, ((got[(li, k)] - ref).abs().max() / ref.abs().max()).item())
    worst = max(worst, ((edges["g"] - x.grad).abs().max() / x.grad.abs().max()).item())
    print(f"{tower} {'subset' if subset else 'plain'}: composed references vs autograd, worst relative {worst:.2e}")
    assert worst < 1e-12


# ----------------------------------------------------------------------------------------------- seeded bugs

def _run_checks(tower, subset, bug=None):
    P, cfg, T, n = _tower(tower)
    subsets = _subsets(n, subset)
    g = _g(6)
    x0 = torch.randn(n * T, D, generator=g, dtype=D64).float().double()
    g_out = torch.randn(n * T, D, generator=g, dtype=D64).float().double()
    prefill = _prefill(P, g)
    entries, streams, _ = _forward(P, cfg, x0, n, T, subsets, rounding=True, bug=bug)
    checks = []
    for (li, kind), e in entries.items():
        x_in, x_out, res = streams[(li, kind)]
        checks += [(f"block {li} {kind} {c}", v, b)
                   for c, v, b in br.check_forward(kind, P[li], cfg, e, x_in, x_out, T, None, res)]
    order = br.edge_order(DEPTH)
    recs, grads, gx = _stand_in_backward(P, cfg, entries, g_out, T, prefill, bug)
    checks += br.check_backward(P, cfg, [entries[o] for o in order], recs, g_out, gx, grads, prefill, T)
    return {name: (v.max().item() if torch.is_tensor(v) and v.numel() else float(v)) / b if b else
            (0.0 if float(torch.as_tensor(v).max()) == 0 else float("inf")) for name, v, b in checks}


@pytest.mark.parametrize("tower,subset", PATHS, ids=PATH_IDS)
def test_stand_in_passes(tower, subset):
    ratios = _run_checks(tower, subset)
    worst = max(ratios.items(), key=lambda kv: kv[1])
    print(f"{tower}: {len(ratios)} checks, worst {worst[0]} at {worst[1]:.3g} of its bound")
    assert worst[1] <= 1.0, worst


BUGS = {  # bug: (tower, subset path, a check name it must fail)
    "proj_wgrad_reads_h": ("rms_swiglu_rope", False, "grad proj_w"),
    "rope_transpose_missing": ("rms_swiglu_rope", False, "attn dq"),
    "qkv_bias_without_cls": ("rms_swiglu_rope", False, "grad qkv_b"),
    "alpha_missing": ("rms_swiglu_rope", True, "gb"),
    "alpha_doubled": ("rms_swiglu_rope", True, "gb"),
    "bias_to_wrong_block": ("ln_gelu_causal", False, "grad fc2_b"),
    "norm_bwd_overwrites_g": ("ln_gelu_causal", False, "dL/dx"),
    "gb_before_norm_grad": ("rms_swiglu_rope", False, "gb"),
    "subset_permuted_idx": ("rms_swiglu_rope", True, "dL/dx"),
    "wgrad_tile_dropped": ("ln_gelu_causal", False, "grad qkv_w"),
}


@pytest.mark.parametrize("bug", list(BUGS))
def test_seeded_composition_bug_rejected(bug):
    tower, subset, where = BUGS[bug]
    ratios = _run_checks(tower, subset, bug)
    hit = {k: v for k, v in ratios.items() if where in k}
    worst = max(hit.items(), key=lambda kv: kv[1])
    print(f"{bug}: {worst[0]} at {worst[1]:.3g}x its bound")
    assert worst[1] >= MARGIN, (bug, worst)
