"""The transformer blocks of the training step, sub-layer by sub-layer, against the fp64 references of tests/block_ref.py
at the step's shapes, on the plain and the stochastic-depth (batch-subset) paths.

Each case runs engine.tower_blocks with a tape on two seeded blocks of a VTPTrainer tower, then
train.tower_blocks_backward into gradient buffers pre-filled with seeded non-zero values.  Spies (fixtures below that
only observe and pass every call through) record what the kernels received and produced: the stream around each
subset sub-layer, qkv before a stand-alone RoPE pass, dout / dqkv of the attention backward, dhid / dpre of the gate
backward, and gb / dh of every backward body.  Every stage is then checked from the recorded value that fed it, so each
bound is that of one kernel; where a recorded input came from is checked too (a tape entry's own tensors, or the
reference of the stage that produced it).  Every gradient must end as prefill + gradient.  A second run must repeat
dL/dx, the tape and every recorded bf16 intermediate bit for bit; only the split-K weight gradients and the atomic
column sums may differ.

Bounds are block_ref.py's; its header lists the maxima measured behind them.
"""
import pytest
import torch

from tests import block_ref as br
from tests.util import load_golden
from vtp_b200 import engine, lib, train
from vtp_b200.config import VTPConfig
from vtp_b200.train import TrainConfig, VTPTrainer

pytestmark = pytest.mark.gpu
BF = torch.bfloat16

GEOS = {  # VTP-Small and VTP-Large widths at depth 2 (tests/test_train_gpu.py small2 / large2)
    "small": dict(vision_embed_dim=384, vision_depth=2, vision_num_heads=6, text_embed_dim=384, text_num_heads=6,
                  text_depth=2, decoder_embed_dim=384, decoder_num_heads=6, decoder_depth=2, text_vocab_size=2048),
    "large": "large2",
}

# name: (geometry, tower, images per call, patch grid (or text length))
CASES = {
    "trunk_global": ("small", "trunk", 512, (16, 16)),      # T 257, single-pass attention backward, HW 256
    "trunk_local": ("small", "trunk", 2048, (6, 6)),        # T 37, packed attention tiles
    "decoder": ("small", "decoder", 256, (16, 16)),         # T 256, LayerNorm, bf16 stream, no prefix
    "text": ("small", "text", 256, 77),                     # LayerNorm, GELU, causal, no RoPE
    "trunk_large": ("large", "trunk", 66, (16, 16)),        # D 1024 / 16 heads / hidden 2736: ragged N / K tiles
    "trunk_512": ("small", "trunk", 8, (32, 32)),           # T 1025: streaming long attention backward
}
VARIANTS = [("trunk_global", None), ("trunk_local", None), ("decoder", None), ("text", None), ("trunk_large", None),
            ("trunk_512", None), ("trunk_global", "drop_half"), ("trunk_global", "drop_one"),
            ("trunk_local", "drop_half"), ("trunk_local", "drop_one"), ("trunk_global", "rope_epilogue"),
            ("trunk_global", "swiglu_fwd")]

@pytest.fixture(scope="module")
def trainers():
    """one VTPTrainer per geometry, built on first use and freed with the module"""
    cache = {}
    yield cache
    cache.clear()


def _trainer(cache, geo):
    """a VTPTrainer whose block parameters (weights, biases, norm weights and biases) are all seeded non-trivially"""
    if geo not in cache:
        if isinstance(GEOS[geo], str):
            meta, _ = load_golden(GEOS[geo])
            cfg = VTPConfig(**meta["config"])
        else:
            cfg = VTPConfig(**GEOS[geo])
        tr = VTPTrainer(cfg, TrainConfig(head_out_dim=512, head_hidden=256, head_bottleneck=64, n_local_crops=2))
        st = tr.store
        g = torch.Generator().manual_seed(11)
        for name, shape, _, _ in st.specs:
            if ".blocks." not in name:
                continue
            leaf = name.rsplit(".", 1)[-1]
            if leaf in ("n1_w", "n2_w"):
                v = 1 + 0.2 * torch.randn(shape, generator=g)
            elif leaf in ("n1_b", "n2_b", "b"):
                v = 0.1 * torch.randn(shape, generator=g)
            else:
                v = torch.randn(shape, generator=g) * (1.2 / shape[1] ** 0.5)
            st.f32(name).copy_(v)
        st.sync_compute_copies()
        cache[geo] = tr
    return cache[geo]


def _params(bw):
    return dict(n1_w=bw.n1_w, n1_b=bw.n1_b, qkv_w=bw.qkv.w, qkv_b=bw.qkv.b, proj_w=bw.proj.w, proj_b=bw.proj.b,
                n2_w=bw.n2_w, n2_b=bw.n2_b, fc1_w=bw.fc1.w, fc1_b=bw.fc1.b, fc2_w=bw.fc2.w, fc2_b=bw.fc2.b)


def _grad_views(G):
    return {(li, k): v for li, gw in enumerate(G.blocks) for k, v in _params(gw).items() if v is not None}


def _presets(n, variant):
    """the subset of every sub-layer call: ratio 0.5 with unsorted indices holding the first and the last image, or a
    ratio that keeps one image (a different one per call)"""
    if variant == "drop_one":
        return 1 - 0.5 / n, [torch.tensor([i]) for i in (n - 1, 0, n // 2, 1)]
    out = []
    for c in range(4):
        g = torch.Generator().manual_seed(100 + c)
        rest = torch.randperm(n - 2, generator=g)[:n // 2 - 2] + 1
        idx = torch.cat([rest[:n // 5], torch.tensor([n - 1]), rest[n // 5:], torch.tensor([0])])
        out.append(idx[torch.randperm(idx.numel(), generator=g)] if c % 2 else idx)
    return 0.5, out


# ------------------------------------------------------------------------------------------------------------ spies

class Spies:
    def __init__(self):
        self.rec = {}

    def clear(self):
        self.rec = {}

    def add(self, key, r):
        self.rec.setdefault(key, []).append(r)


@pytest.fixture
def spies(monkeypatch):
    s = Spies()

    def wrap(mod, name, before=None, after=None):
        f = getattr(mod, name)

        def spy(*a, **k):
            r = before(*a, **k) if before is not None else {}
            out = f(*a, **k)
            if after is not None:
                r.update(after(*a, **k))
            s.add(name, r)
            return out
        monkeypatch.setattr(mod, name, spy)

    def attn(qkv, o, dout, lse, *rest, **k):
        dqkv = rest[-1]
        return dict(ptrs=(qkv.data_ptr(), o.data_ptr(), lse.data_ptr()), do=dout.clone(), dqkv=dqkv.clone())

    wrap(lib, "attention_bwd", after=lambda qkv, o, dout, lse, dqkv, *a, **k: attn(qkv, o, dout, lse, dqkv))
    wrap(lib, "attention_bwd_long", after=lambda qkv, o, dout, lse, delta, dqkv, *a, **k: attn(qkv, o, dout, lse, dqkv))
    gate = lambda pre, dhid, dpre, *a, **k: dict(pre=pre.data_ptr(), dhid=dhid.clone(), dpre=dpre.clone())
    wrap(lib, "swiglu_bwd", after=gate)
    wrap(lib, "gelu_bwd", after=gate)
    body = dict(before=lambda W, bw, gw, e, gb, dh, *a, **k: dict(gb=gb.clone()),
                after=lambda W, bw, gw, e, gb, dh, *a, **k: dict(dh=dh.clone()))
    wrap(train, "attention_sublayer_backward", **body)
    wrap(train, "ffn_sublayer_backward", **body)
    wrap(lib, "rope_fwd", before=lambda qkv, *a, **k: dict(qkv_pre=qkv.clone()))
    wrap(lib, "gather_images", before=lambda x, out, idx, *a, **k: dict(x=x.clone()))
    wrap(lib, "scatter_add_images", after=lambda src, dst, *a, **k: dict(src=src.clone(), dst=dst.clone()))
    return s


# ------------------------------------------------------------------------------------------------------------- runs

def _run(W, G, x0, g_out, prefill, n, T, rope, causal, drop, spies):
    """forward with a tape + backward; -> dict(y, g, tape (copy), fwd / bwd spy records, grads)"""
    for k, v in _grad_views(G).items():
        v.copy_(prefill[k])
    spies.clear()
    tape = []
    plan = None if drop is None else engine.DropPlan(drop[0], preset=drop[1])
    y = engine.tower_blocks(W, x0.clone(), n, T, rope, "bf16", causal=causal, tape=tape, drop=plan)
    saved = [dict(b) for b in tape]
    fwd = spies.rec
    spies.clear()
    g = g_out.clone()
    train.tower_blocks_backward(W, G, tape, g, n, T, rope, causal)
    torch.cuda.synchronize()
    grads = {k: v.clone() for k, v in _grad_views(G).items()}
    return dict(y=y, g=g, tape=saved, fwd=fwd, bwd=spies.rec, grads=grads)


def _report(case, checks):
    bad = []
    for name, v, bound in checks:
        v = torch.as_tensor(v).double().reshape(-1)
        m = v.max().item() if v.numel() else 0.0
        print(f"BLOCKSTAT {case} | {name} | {m:.4g} | bound {bound:g}")
        if not m <= bound:
            rows = (~(v <= bound)).nonzero().flatten()
            bad.append(f"{name}: {m:.4g} > {bound:g} in {rows.numel()} rows, first {rows[:6].tolist()} "
                       f"(128-row tiles {sorted(set((rows[:256] // 128).tolist()))[:6]})")
    assert not bad, f"{case}:\n" + "\n".join(bad)


@pytest.mark.parametrize("case,variant", VARIANTS, ids=[c + ("" if v is None else "-" + v) for c, v in VARIANTS])
def test_block_sublayers(case, variant, trainers, spies, monkeypatch):
    geo, tower, n, grid = CASES[case]
    tr = _trainer(trainers, geo)
    W, G = tr.towers[(tower, "param")], tr.towers[(tower, "grad")]
    dev = tr.device
    if variant == "rope_epilogue":
        monkeypatch.setattr(engine, "SPLIT_EPILOGUES", False)
    if variant == "swiglu_fwd":
        monkeypatch.setattr(engine, "FUSED_SWIGLU", False)
    causal = tower == "text"
    if tower == "text":
        T, rope = grid, None
    else:
        T = grid[0] * grid[1] + W.prefix
        rope = W.rope(grid[0], grid[1], dev)
    D = W.D
    drop = None if variant not in ("drop_half", "drop_one") else _presets(n, variant)
    cfg = dict(H=W.heads, eps=W.eps, prefix=W.prefix, ffn=W.ffn, hidden=W.blocks[0].hidden, causal=causal,
               rope=None if rope is None else (rope[0], rope[1]), stream_bf16=W.stream_bf16)
    gen = torch.Generator(device="cuda").manual_seed(len(case) * 7 + n)
    x0 = torch.randn(n * T, D, device="cuda", generator=gen).to(BF if W.stream_bf16 else torch.float32)
    g_out = torch.randn(n * T, D, device="cuda", generator=gen)
    views = _grad_views(G)
    prefill = {k: 0.5 * torch.randn(v.shape, device="cuda", generator=gen) for k, v in views.items()}
    P = [_params(bw) for bw in W.blocks]
    depth = len(P)

    r = _run(W, G, x0, g_out, prefill, n, T, rope, causal, drop, spies)
    checks = []

    # ---- forward, in forward order
    fwd_order = [(li, kind) for li in range(depth) for kind in ("attn", "ffn")]
    entries = {(li, kind): r["tape"][li][kind] for li, kind in fwd_order}
    rope_pre = iter(r["fwd"].get("rope_fwd", []))
    gathers, scatters = r["fwd"].get("gather_images", []), r["fwd"].get("scatter_add_images", [])
    assert len(gathers) == len(scatters) == (0 if drop is None else 2 * depth)
    for j, (li, kind) in enumerate(fwd_order):
        e = entries[(li, kind)]
        if drop is None:
            x_in = e["x"]
            x_out = entries[fwd_order[j + 1]]["x"] if j + 1 < len(fwd_order) else r["y"]
            res = None
            assert e["subset"] is None
        else:
            x_in, x_out, res = gathers[j]["x"], scatters[j]["dst"], scatters[j]["src"]
            idx, alpha = e["subset"]
            assert torch.equal(idx.cpu(), drop[1][j]) and alpha == n / idx.numel()
            assert torch.equal(e["x"], x_in[br.image_rows(idx, T)]), f"block {li} {kind}: gathered stream"
            nxt = gathers[j + 1]["x"] if j + 1 < len(fwd_order) else r["y"]
            assert torch.equal(x_out, nxt), f"block {li} {kind}: stream out is not the next sub-layer's stream in"
        qkv_pre = next(rope_pre)["qkv_pre"] if kind == "attn" and "rope_fwd" in r["fwd"] else None
        checks += [(f"block {li} {kind} {c}", v, b)
                   for c, v, b in br.check_forward(kind, P[li], cfg, e, x_in, x_out, T, qkv_pre, res)]
    assert len(r["fwd"].get("rope_fwd", [])) == (depth if rope is not None and variant != "rope_epilogue" else 0)

    # ---- backward, in edge order
    order = br.edge_order(depth)
    bodies = r["bwd"]["attention_sublayer_backward"], r["bwd"]["ffn_sublayer_backward"]
    attn_k = r["bwd"].get("attention_bwd", []) + r["bwd"].get("attention_bwd_long", [])
    long_path = T - W.prefix > 256 and not causal
    assert len(r["bwd"].get("attention_bwd_long" if long_path else "attention_bwd", [])) == depth
    gates = r["bwd"].get("swiglu_bwd" if W.ffn == "swiglu" else "gelu_bwd", [])
    assert len(gates) == depth
    recs, ents = [], []
    for i, (li, kind) in enumerate(order):
        e = entries[(li, kind)]
        j = i // 2
        rec = dict(bodies[0 if kind == "attn" else 1][j])
        if kind == "attn":
            a = attn_k[j]
            assert a["ptrs"] == (e["qkv"].data_ptr(), e["o"].data_ptr(), e["lse"].data_ptr()), \
                f"block {li}: attention backward not fed the tape's qkv / o / lse"
            rec.update(do=a["do"], dqkv=a["dqkv"])
        else:
            assert gates[j]["pre"] == e["pre"].data_ptr(), f"block {li}: gate backward not fed the tape's pre"
            rec.update(dhid=gates[j]["dhid"], dpre=gates[j]["dpre"])
        recs.append(rec)
        ents.append(e)
    checks += br.check_backward(P, cfg, ents, recs, g_out, r["g"], r["grads"], prefill, T)
    _report(f"{case}" + ("" if variant is None else f"-{variant}"), checks)

    # ---- determinism: everything but the split-K wgrads and the atomic column sums repeats bit for bit
    r2 = _run(W, G, x0, g_out, prefill, n, T, rope, causal, drop, spies)
    diff = []
    if not torch.equal(r["g"], r2["g"]):
        diff.append("dL/dx")
    if not torch.equal(r["y"], r2["y"]):
        diff.append("stream out")
    for li in range(depth):
        for kind in ("attn", "ffn"):
            for k, v in r["tape"][li][kind].items():
                if torch.is_tensor(v) and not torch.equal(v, r2["tape"][li][kind][k]):
                    diff.append(f"tape block {li} {kind} {k}")
    for key, lst in r["bwd"].items():
        for i, (a, b) in enumerate(zip(lst, r2["bwd"][key])):
            for k, v in a.items():
                if torch.is_tensor(v) and not torch.equal(v, b[k]):
                    diff.append(f"{key} call {i} {k}")
    assert not diff, f"not bit-identical across two runs: {diff}"
