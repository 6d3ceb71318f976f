"""The cluster-pair attention backward (attn_bwd_pair_kernel, csrc/attention_bwd.cu): vtp_attention_bwd routes every
non-causal, unpacked call with 128 < HW <= 256 to it.  Row by row against the emulated fp64 reference, at the edges of
its tiling (HW = 129: one query row in tile 2 and one key on rank 1; 192: three query tiles; 255: ragged last tile and
key; 256: full), with and without the cls token and RoPE; one launch at the training step's grid; bit-identical
repeats; agreement with the streaming backward; and the dispatch itself, through the profiler's kernel names."""
import pytest
import torch

from tests import attn_ref as ar
from tests.test_attention_rows_gpu import _setup, check_bwd, run_bwd, run_fwd
from vtp_b200 import lib

pytestmark = pytest.mark.gpu
BF = torch.bfloat16

SHAPES = [(hw, prefix, rope) for hw in (129, 192, 255, 256) for prefix in (0, 1) for rope in (True, False)]


@pytest.mark.parametrize("hw,prefix,rope", SHAPES)
def test_pair_rows(hw, prefix, rope):
    B, H, T = 3, 2, hw + prefix
    qkv, dout, tables = _setup(B, T, H, prefix, False, rope, seed=hw * 10 + prefix)
    o, lse = run_fwd(qkv, B, T, H, prefix, False)
    check_bwd(f"pair_HW{hw}_p{prefix}_{'rope' if rope else 'norope'}", qkv, dout, o, lse, B, T, H, prefix, False,
              tables, False)


def test_pair_training_grid_rows():
    """B = 176, H = 6: 2 112 CTAs in 1 056 clusters, far more than the card holds at once; every row checked"""
    B, T, H, prefix = 176, 257, 6, 1
    qkv, dout, tables = _setup(B, T, H, prefix, False, True, seed=11)
    o, lse = run_fwd(qkv, B, T, H, prefix, False)
    check_bwd("pair_B176_H6", qkv, dout, o, lse, B, T, H, prefix, False, tables, False, whole_exact=False)


@pytest.mark.parametrize("T,prefix", [(257, 1), (256, 0), (130, 1)])
def test_pair_bitwise_deterministic(T, prefix):
    B, H = 8, 6
    qkv, dout, tables = _setup(B, T, H, prefix, False, True, seed=T)
    o, lse = run_fwd(qkv, B, T, H, prefix, False)
    g1 = run_bwd(qkv, o, dout, lse, B, T, H, prefix, False, tables)
    g2 = run_bwd(qkv, o, dout, lse, B, T, H, prefix, False, tables)
    assert torch.equal(g1, g2)


@pytest.mark.parametrize("T,prefix", [(257, 1), (256, 0), (193, 1), (130, 0)])
def test_pair_agrees_with_streaming(T, prefix):
    """same op, same rounding points, different fp32 summation order: rows agree far inside BWD_ROW_TOL"""
    B, H = 4, 6
    qkv, dout, tables = _setup(B, T, H, prefix, False, True, seed=T + 3)
    o, lse = run_fwd(qkv, B, T, H, prefix, False)
    g = run_bwd(qkv, o, dout, lse, B, T, H, prefix, False, tables)
    gl = torch.empty_like(g)
    delta = torch.empty(B, H, T, device="cuda")
    lib.attention_bwd_long(qkv, o, dout, lse, delta, gl, B, T, H, prefix=prefix, rope=tables)
    torch.cuda.synchronize()
    e = ar.row_err(g, gl.double(), (B, T, 3, H)).max().item()
    print(f"ROWSTAT pair_vs_long T{T}_p{prefix} {e:.3e}")
    assert e <= ar.BWD_ROW_TOL / 4, e


@pytest.mark.parametrize("T,prefix,causal,kernel", [(257, 1, False, "attn_bwd_pair_kernel"),
                                                     (256, 0, False, "attn_bwd_pair_kernel"),
                                                     (200, 0, True, "attn_bwd_kernel<2>"),
                                                     (129, 1, False, "attn_bwd_kernel<1>")])
def test_pair_dispatch(T, prefix, causal, kernel):
    B, H = 2, 2
    qkv, dout, tables = _setup(B, T, H, prefix, causal, True, seed=1)
    o, lse = run_fwd(qkv, B, T, H, prefix, causal)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        run_bwd(qkv, o, dout, lse, B, T, H, prefix, causal, tables)
    names = [ev.name for ev in prof.events() if "attn_bwd" in ev.name]
    assert names and all(kernel in n for n in names), names
