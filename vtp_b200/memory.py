"""HBM budget of the 3-objective training step (what `VTPTrainer` keeps resident), used to size the per-pass image
groups (`TrainConfig.ssl_chunk / rec_chunk`) for the 80 GB of an H100.

The step saves, per token and per block, exactly what `engine.tower_blocks(..., tape=...)` appends, one entry per
sub-layer:
    attn: x (its norm's input: the residual stream, fp32 in the trunk / text tower, bf16 in the autocast decoder),
          h (bf16 [D]), qkv (bf16 [3D]), o (bf16 [D]), lse + rstd (a few floats)
    ffn:  x (as above), h (bf16 [D]), pre (bf16 [2·Hs] SwiGLU / [Hd] GELU), hid (bf16 [Hs] / [Hd]), rstd
(under stochastic depth x is the gathered fp32 rows of the kept images, so the bytes scale with the kept fraction)
=> 20·D + 6·Hs bytes (fp32 stream, SwiGLU),  16·D + 6·Hs (bf16 stream),  20·D + 4·Hd (GELU MLP): `block_tape_bytes`.
The three objectives run one after the other, so the peak is the largest single objective plus the persistent state.
Calibration point (torch.cuda.max_memory_allocated on an H100, graph-captured step): VTP-Small, 256 images/GPU,
K = 65 536 -> 42.7 GiB peak.
"""
from __future__ import annotations

import math
from typing import Dict, Tuple

from .config import VTPConfig
from .params import Geometry, geometry, table

GIB = float(2 ** 30)


def block_tape_bytes(D: int, hidden: int, ffn: str, stream_bf16: bool, heads: int) -> int:
    """Bytes saved for backward per token per block (engine.tower_blocks with a tape)."""
    s = 2 if stream_bf16 else 4
    pre = 2 * (2 * hidden if ffn == "swiglu" else hidden)
    return 2 * s * D + 3 * 2 * D + 2 * 3 * D + pre + 2 * hidden + 4 * heads + 8


def tower_tape_bytes(tokens: int, g: Geometry) -> int:
    return tokens * g.depth * block_tape_bytes(g.D, g.hidden, g.ffn, g.stream_bf16, g.heads)


def param_count(cfg: VTPConfig, head_out_dim: int = 65536, head_hidden: int = 2048, head_bottleneck: int = 256) -> Dict[str, int]:
    """Parameters of the training step: all of them, and those the EMA teacher keeps a copy of."""
    sizes = [(math.prod(e.shape), e.teacher) for e in table(cfg, (head_out_dim, head_hidden, head_bottleneck))]
    return {"total": sum(n for n, _ in sizes), "teacher": sum(n for n, t in sizes if t)}


def train_step_bytes(cfg: VTPConfig, B: int, *, image: int = 256, local: int = 96, n_local: int = 8,
                     head_out_dim: int = 65536, head_hidden: int = 2048, head_bottleneck: int = 256,
                     mask_ratio: float = 0.3, mask_prob: float = 0.5, ssl_chunk: int = 0, rec_chunk: int = 0,
                     lpips: bool = True, lpips_chunk: int = 32) -> Dict[str, float]:
    """Estimated resident bytes: persistent state + the peak of each objective (they run sequentially)."""
    gv, gd, gt = (geometry(cfg, tower) for tower in ("trunk", "decoder", "text"))
    D, Dd, hs, hsd = gv.D, gd.D, gv.hidden, gd.hidden
    ps = cfg.vision_patch_size
    HW, HWl = (image // ps) ** 2, (local // ps) ** 2
    T, Tl = HW + 1, HWl + 1
    K = head_out_dim
    n = param_count(cfg, head_out_dim, head_hidden, head_bottleneck)
    persistent = n["total"] * (4 + 2 + 4 + 4 + 4) + n["teacher"] * (4 + 2) + 3 * K * head_bottleneck * 2
    inputs = B * (3 * image * image * 4 * (1 + 2 + 1) + n_local * 3 * local * local * 4)

    def trunk(tokens):
        return tower_tape_bytes(tokens, gv) + tokens * (4 * D + 2 * 3 * ps * ps)

    # transient working set of one backward sub-layer (dh, dhid, dpre, dqkv, do, g, gb ...) on the largest token group
    def transient(tokens, dim, hidden):
        return tokens * (4 * dim * 2 + 2 * dim * 2 + 2 * hidden * 3 * 2 + 2 * 3 * dim)

    clip = trunk(B * T) + tower_tape_bytes(B * cfg.text_context_length, gt) + transient(B * T, D, hs)
    bs = ssl_chunk if 0 < ssl_chunk < B else B
    n_m = int(round(2 * bs * mask_prob * mask_ratio * HW))
    rows_s, rows_t = n_local * bs + 2 * bs + n_m, 2 * bs + n_m
    head = (rows_s + rows_t) * K * 2 + rows_s * (2 * D + 4 * 2 * head_hidden + 3 * 2 * head_bottleneck) + K * head_bottleneck * 4
    ssl = trunk(2 * bs * T) + trunk(n_local * bs * Tl) + head + transient(2 * bs * T, D, hs)
    br = rec_chunk if 0 < rec_chunk < B else B
    vgg_per_img = 2 * (64 * 2 * image ** 2 + 128 * 2 * (image // 2) ** 2 + 256 * 3 * (image // 4) ** 2 +
                       512 * 3 * (image // 8) ** 2 + 512 * 3 * (image // 16) ** 2)
    rec = trunk(br * T) + tower_tape_bytes(br * HW, gd) + br * 3 * image * image * (2 + 4 + 2) + transient(br * HW, Dd, hsd) + \
        (2 * 2 * min(lpips_chunk, br) * vgg_per_img if lpips else 0)
    peak = persistent + inputs + max(clip, ssl, rec)
    return {"persistent": persistent, "inputs": inputs, "clip": clip, "ssl": ssl, "rec": rec, "peak": peak,
            "params": n["total"]}


def suggest_chunks(cfg: VTPConfig, B: int, budget_bytes: float = 64 * GIB, **kw) -> Tuple[int, int]:
    """Largest power-of-two-divided image groups (B, B/2, B/4, ...) whose estimated peak fits the budget.
    Returns (ssl_chunk, rec_chunk) with 0 = whole batch."""
    def fit(which: str) -> int:
        c = B
        while c >= 1:
            est = train_step_bytes(cfg, B, **{**kw, ("ssl_chunk" if which == "ssl" else "rec_chunk"): c})
            if est["persistent"] + est["inputs"] + est[which] <= budget_bytes:
                return 0 if c == B else c
            if c == 1:
                break
            c = max(1, c // 2)
        raise ValueError(f"the {which} objective does not fit {budget_bytes / GIB:.0f} GiB even one image at a time")

    est = train_step_bytes(cfg, B, **kw)
    if est["persistent"] + est["inputs"] + est["clip"] > budget_bytes:
        raise ValueError("the contrastive objective cannot be split across passes and does not fit the budget; "
                         "lower the per-GPU batch")
    return fit("ssl"), fit("rec")


def fit_batch(cfg: VTPConfig, B: int = 256, budget_bytes: float = 64 * GIB, **kw) -> int:
    """Largest per-GPU batch B, B/2, B/4, ... for which `suggest_chunks` finds image groups that fit the budget (the
    contrastive objective is not split, so it bounds the batch: VTP-Large runs 128 images per 80 GB GPU)."""
    b = B
    while b >= 1:
        try:
            suggest_chunks(cfg, b, budget_bytes, **kw)
            return b
        except ValueError:
            b //= 2
    raise ValueError(f"{cfg} does not fit {budget_bytes / GIB:.0f} GiB even one image per GPU")
