"""HBM budget model of the training step (vtp_b200/memory.py) — host logic, no GPU."""
import pytest

from vtp_b200 import memory as m
from vtp_b200.config import preset


def test_small_matches_the_measured_peak():
    """Measured on an H100: VTP-Small, 256 images/GPU, K = 65536 -> 42.7 GiB peak (torch.cuda.max_memory_allocated)."""
    est = m.train_step_bytes(preset("small"), 256)
    assert abs(est["peak"] / m.GIB - 42.7) < 0.15 * 42.7
    assert est["ssl"] > est["rec"] > est["clip"]
    assert abs(est["params"] / 1e6 - 106.2) < 1.0          # SURVEY §8d: 83.8 M model + ~22.3 M DINO head


def test_large_needs_chunks_and_chunks_fit():
    cfg = preset("large")
    est = m.train_step_bytes(cfg, 256)
    assert est["peak"] > 80e9                                # config 4 does not fit an H100 in one piece
    with pytest.raises(ValueError):                           # 256 per GPU: the contrastive pass alone exceeds 64 GiB
        m.suggest_chunks(cfg, 256)
    B = m.fit_batch(cfg, 256)                                 # what bench.py runs for VTP-Large on an 80 GB H100
    assert B == 128
    ssl_chunk, rec_chunk = m.suggest_chunks(cfg, B)
    assert 0 < ssl_chunk < B
    fit = m.train_step_bytes(cfg, B, ssl_chunk=ssl_chunk, rec_chunk=rec_chunk)
    assert fit["peak"] <= 64 * m.GIB
    assert m.fit_batch(preset("small"), 256) == 256 and m.fit_batch(preset("base"), 256) == 256
    assert m.suggest_chunks(preset("small"), 256) == (0, 0)               # VTP-Small runs in one piece on 80 GB
    bs, br = m.suggest_chunks(preset("base"), 256)
    assert m.train_step_bytes(preset("base"), 256, ssl_chunk=bs, rec_chunk=br)["peak"] <= 64 * m.GIB


def test_tape_bytes_formula():
    # trunk block, fp32 stream, SwiGLU: 20 D + 6 Hs (+ lse / rstd floats)
    D, Hs, H = 384, 1024, 6
    assert m.block_tape_bytes(D, Hs, "swiglu", False, H) == 20 * D + 6 * Hs + 4 * H + 8
    assert m.block_tape_bytes(D, Hs, "swiglu", True, H) == 16 * D + 6 * Hs + 4 * H + 8
    assert m.block_tape_bytes(D, 4 * D, "gelu", False, H) == 20 * D + 4 * 4 * D + 4 * H + 8


def test_suggest_chunks_rejects_what_cannot_fit():
    import pytest

    with pytest.raises(ValueError):
        m.suggest_chunks(preset("large"), 256, budget_bytes=40 * m.GIB)     # the contrastive pass alone is larger
    # a tighter but feasible budget only makes the groups smaller
    a = m.suggest_chunks(preset("large"), 256, budget_bytes=150 * m.GIB)
    b = m.suggest_chunks(preset("large"), 256, budget_bytes=110 * m.GIB)
    assert 0 < b[0] <= a[0]


def test_latent_statistics_formula():
    """LatentShardWriter.stats(): mean / unbiased std from fp64 sums (host arithmetic only)."""
    import torch

    from vtp_b200.generation import LatentShardWriter

    z = torch.randn(5, 4, 3, 3, dtype=torch.float64, generator=torch.Generator().manual_seed(0)) * 2 + 1
    w = LatentShardWriter.__new__(LatentShardWriter)
    w._sum, w._sumsq, w._n = z.sum(dim=(0, 2, 3)), (z * z).sum(dim=(0, 2, 3)), z.numel() // z.shape[1]
    st = w.stats()
    assert st["mean"].shape == (1, 4, 1, 1) and st["std"].dtype == torch.float32
    assert torch.allclose(st["mean"].double(), z.mean(dim=(0, 2, 3), keepdim=True), atol=1e-6)
    assert torch.allclose(st["std"].double(), z.std(dim=(0, 2, 3), keepdim=True), atol=1e-6)


def test_gradient_buckets_partition_the_table_store():
    """train.grad_buckets: the per-tower all-reduce ranges cover [0, n) exactly once, and every tensor lies inside the
    bucket of its tower (text + clip projection + logit scale | DINO head | pixel decoder | trunk)."""
    from vtp_b200.params import table
    from vtp_b200.train import ParamStore, grad_buckets

    st = ParamStore("cpu")
    for e in table(preset("tiny"), (512, 256, 64)):
        st.add(e.name, e.shape, e.decay, e.teacher)
    st.finalize()
    b = grad_buckets(st.offset, st.n)
    ranges = sorted(r for rs in b.values() for r in rs)
    assert ranges[0][0] == 0 and ranges[-1][1] == st.n
    assert all(a[1] == c[0] for a, c in zip(ranges, ranges[1:]))          # no gap, no overlap
    inside = lambda name, which: any(lo <= st.offset[name] < hi for lo, hi in b[which])
    assert inside("text.blocks.1.fc1.w", "text") and inside("logit_scale", "text") and inside("visual_proj.w", "text")
    assert inside("head.last_g", "head") and inside("decoder.blocks.0.qkv.b", "decoder") and inside("trunk.cls", "trunk")
    assert sum(len(v) for v in b.values()) <= 16                          # a handful of NCCL calls per step
