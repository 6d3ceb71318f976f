"""Host orchestration of the sm_90a kernels: weight packing and tower forwards.

Mirrors, stage by stage, the reference's L1/L2 code (vtp/models/layers/*, encoders/*, decoders/*) — every numeric op
is a C-ABI kernel call from `lib`; torch is used for device memory (torch.empty) and integer index glue only.

Two precision modes, selected by the caller (VTPModel maps them from the autocast state like the reference):
  "bf16" — equals the reference under torch.autocast(bfloat16): bf16 GEMM/attention operands, fp32 accumulation,
           fp32 norms, fp32 residual stream in the encoder/text tower, bf16 stream in the decoder.
  "fp32" — equals the reference in fp32: every GEMM runs as a bf16x3 split (hi·hi + hi·lo + lo·hi, K-concatenated so
           the same wgmma kernel is used; error ~2^-16), activations fp32, attention on fp32 CUDA cores.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import torch

from . import lib
from .rope import rope_sincos

BF = torch.bfloat16
F32 = torch.float32
# bf16 hot path: run the RoPE rotation and the SwiGLU gate as stand-alone full-occupancy kernels after a plain GEMM instead
# of inside the GEMM epilogue (see csrc/elementwise.cu).  The fused epilogues stay available
# (fp32 mode uses them; set False to use them in bf16 mode too — identical numerics, tests cover both).
SPLIT_EPILOGUES = True
# SwiGLU gate: the lean TMA-store epilogue variant (csrc/gemm.cu fast_swiglu_tile) writes the hidden tensor
# (and, for training, the pre-activation) straight from the fc1 GEMM — no stand-alone gate pass re-reading [M, 2Hs].
# VTP_FUSED_SWIGLU=0 restores the stand-alone swiglu_fwd kernel.
import os as _os
FUSED_SWIGLU = _os.environ.get("VTP_FUSED_SWIGLU", "1") != "0"


def _e(shape, dtype, dev):
    return torch.empty(shape, dtype=dtype, device=dev)


# ------------------------------------------------------------------------------------------------------ packing
@dataclass
class Lin:
    """One packed linear: w bf16 [N, Kp] (Kp = K in bf16 mode, 3K split hi|lo|hi in fp32 mode), b fp32 [N] | None."""
    w: torch.Tensor
    b: Optional[torch.Tensor]
    N: int
    K: int

    @property
    def Kp(self) -> int:
        return self.w.shape[1]


def pack_lin(w: torch.Tensor, b: Optional[torch.Tensor], mode: str) -> Lin:
    """w fp32 [N, K] (already on the device).  bf16 mode rounds the bias to bf16 as autocast does."""
    N, K = w.shape
    w = w.detach().to(F32).contiguous()
    if mode == "bf16":
        wp = w.to(BF).contiguous()
        bp = None if b is None else b.detach().to(BF).to(F32).contiguous()
    else:
        Kpad = (K + 7) // 8 * 8
        if Kpad != K:
            w = torch.nn.functional.pad(w, (0, Kpad - K))
        wp = _e((N, 3 * Kpad), BF, w.device)
        lib.split3(w, wp, N, Kpad, b_side=True)
        bp = None if b is None else b.detach().to(F32).contiguous()
    return Lin(wp, bp, N, K)


def interleave8(w1: torch.Tensor, w2: torch.Tensor) -> torch.Tensor:
    """rows [16g,16g+8) = w1[8g:8g+8], rows [16g+8,16g+16) = w2[8g:8g+8]  (SwiGLU gate epilogue layout)."""
    Hs = w1.shape[0]
    rest = w1.shape[1:]
    return torch.stack([w1.reshape(Hs // 8, 8, *rest), w2.reshape(Hs // 8, 8, *rest)], dim=1).reshape(2 * Hs, *rest)


@dataclass
class BlockW:
    n1_w: torch.Tensor
    n1_b: Optional[torch.Tensor]
    qkv: Lin
    proj: Lin
    n2_w: torch.Tensor
    n2_b: Optional[torch.Tensor]
    fc1: Lin          # SwiGLU: 8-interleaved w1|w2 (N = 2*Hs);  text MLP: c_fc (N = 4*D)
    fc2: Lin          # w3 / c_proj
    hidden: int


@dataclass
class TowerW:
    """A ViT-style stack (vision trunk, pixel decoder or text transformer) in packed form."""
    D: int
    heads: int
    norm: str                 # "rms" | "ln"
    eps: float
    stream_bf16: bool         # residual stream dtype under autocast (decoder: bf16)
    prefix: int               # cls tokens
    ffn: str                  # "swiglu" | "gelu"
    blocks: List[BlockW] = field(default_factory=list)
    norm_w: Optional[torch.Tensor] = None
    norm_b: Optional[torch.Tensor] = None
    periods: Optional[torch.Tensor] = None
    extra: Dict[str, object] = field(default_factory=dict)
    _rope: Dict[Tuple[int, int], Tuple[torch.Tensor, torch.Tensor]] = field(default_factory=dict)

    def rope(self, H: int, W: int, dev):
        key = (H, W)
        if key not in self._rope:
            sin, cos = rope_sincos(H, W, self.periods.to(BF))
            self._rope[key] = (sin.to(dev).contiguous(), cos.to(dev).contiguous())
        return self._rope[key]


# ------------------------------------------------------------------------------------------------------ primitives
def operand(x: torch.Tensor, M: int, K: int, mode: str) -> torch.Tensor:
    """GEMM A operand of an activation: bf16 mode -> x itself (bf16); fp32 mode -> bf16x3 split [M, 3K]."""
    if mode == "bf16":
        assert x.dtype == BF
        return x
    assert x.dtype == F32
    Kpad = (K + 7) // 8 * 8
    assert Kpad == K, "fp32 mode needs K % 8 == 0"
    out = _e((M, 3 * K), BF, x.device)
    lib.split3(x, out, M, K, b_side=False)
    return out


def linear(a_op: torch.Tensor, lin: Lin, out: torch.Tensor, M: int, mode: str, **epi) -> None:
    """out = epi(a_op · lin.wᵀ + lin.b).  a_op from `operand()` / norm(y_mode=split)."""
    lib.gemm(a_op, lin.w, out, M=M, N=lin.N, K=lin.Kp, lda=lin.Kp, ldb=lin.Kp, bias=lin.b,
             round_bf16=(mode == "bf16"), **epi)


def norm(x, M, D, w, b, eps, mode, *, want: str, tape=None):
    """want: 'op' -> GEMM operand (bf16 | split3), 'f32' -> fp32 values.  Returns tensor."""
    dev = x.device
    rstd = mean = None
    if tape is not None:
        rstd = _e((M,), F32, dev)
        mean = _e((M,), F32, dev) if b is not None else None
    if want == "f32":
        y = _e((M, D), F32, dev)
        lib.norm_fwd(x, y, w, b, eps, M, D, y_mode=lib.OUT_F32, rstd=rstd, mean=mean)
    elif mode == "bf16":
        y = _e((M, D), BF, dev)
        lib.norm_fwd(x, y, w, b, eps, M, D, y_mode=lib.OUT_BF16, rstd=rstd, mean=mean)
    else:
        y = _e((M, 3 * D), BF, dev)
        lib.norm_fwd(x, y, w, b, eps, M, D, y_mode=lib.OUT_SPLIT3, rstd=rstd, mean=mean)
    if tape is not None:
        tape["rstd"], tape["mean"] = rstd, mean
    return y


class DropPlan:
    """Batch-subset stochastic depth for one tower pass (layers/block.py:20-118 `get_branges_scales`, :201-298): every
    sub-layer (attention, FFN) of every block runs on a fresh random subset of the images and its output is added back
    scaled by residual_scale_factor.

      single process:  keep = max(int(b (1 - ratio)), 1),  scale = b / keep                     (block.py:33-38)
      data parallel:   global_keep = max(int(b W (1 - ratio)), W) dealt out evenly over the W ranks (the first
                       global_keep % W ranks get one more, capped at b), scale = b W / Σ allocation  (block.py:40-67)
    The reference has rank 0 compute that allocation and broadcast it (block.py:94); it is a pure function of
    (b, ratio, W), so every rank derives it locally here — no collective.  The subset itself is
    `torch.randperm(b, device)[:keep]` like the reference (device-side, graph-capturable).  `preset` (a sequence of index
    tensors) replaces the random draws — used by the parity tests."""

    def __init__(self, ratio: float, world: int = 1, rank: int = 0, preset: Optional[Sequence[torch.Tensor]] = None):
        self.ratio, self.world, self.rank = float(ratio), int(world), int(rank)
        self.preset = list(preset) if preset is not None else None
        self.calls = 0

    def keep_and_scale(self, b: int) -> Tuple[int, float]:
        if self.world <= 1:
            keep = max(int(b * (1 - self.ratio)), 1)
            return keep, b / keep
        gb = b * self.world
        global_keep = max(int(gb * (1 - self.ratio)), self.world)
        base, extra = divmod(global_keep, self.world)
        alloc = [min(base + (1 if i < extra else 0), b) for i in range(self.world)]
        return alloc[self.rank], gb / max(sum(alloc), 1)

    def next(self, b: int, dev) -> Tuple[torch.Tensor, float]:
        keep, scale = self.keep_and_scale(b)
        if self.preset is not None:
            idx = self.preset[self.calls].to(dev, torch.long).contiguous()
            assert idx.numel() == keep, f"preset subset {self.calls} has {idx.numel()} images, the plan keeps {keep}"
        else:
            idx = torch.randperm(b, device=dev)[:keep].contiguous()
        self.calls += 1
        return idx, scale


def attention_sublayer(W: TowerW, bw: BlockW, x: torch.Tensor, n: int, T: int, mode: str, out: torch.Tensor,
                       resid: Optional[torch.Tensor], tape: Optional[dict], *, rope, causal: bool) -> None:
    """out = proj(attn(rope(qkv(norm1 x)))) (+ resid) on the n images of x [n*T, D] (layers/block.py:293,
    attention.py:91-126).  A tape dict is filled with what the backward reads: x, rstd / mean, h, qkv, o, lse."""
    dev, D, H = x.device, W.D, W.heads
    M = n * T
    act = BF if mode == "bf16" else F32
    h = norm(x, M, D, bw.n1_w, bw.n1_b, W.eps, mode, want="op", tape=tape)
    qkv = _e((M, 3 * D), act, dev)
    if rope is not None and mode == "bf16" and SPLIT_EPILOGUES:
        linear(h, bw.qkv, qkv, M, mode)                 # rounding to bf16 == q.to(bf16) of the reference
        lib.rope_fwd(qkv, rope[0], rope[1], M, T, W.prefix, D)
    elif rope is not None:
        linear(h, bw.qkv, qkv, M, mode, act=lib.ACT_ROPE, rope=(rope[0], rope[1], T, W.prefix, 2 * D))
    else:
        linear(h, bw.qkv, qkv, M, mode)
    o = _e((M, D), act, dev)
    lse = _e((n, H, T), F32, dev) if tape is not None else None
    if mode == "bf16":
        lib.attention_fwd(qkv, o, n, T, H, prefix=W.prefix, causal=causal, lse=lse)
    else:
        lib.attention_fwd_f32(qkv, o, n, T, H, causal=causal)
    linear(operand(o, M, D, mode), bw.proj, out, M, mode, resid=resid)
    if tape is not None:
        tape.update(x=x, h=h, qkv=qkv, o=o, lse=lse)


def ffn_sublayer(W: TowerW, bw: BlockW, x: torch.Tensor, n: int, T: int, mode: str, out: torch.Tensor,
                 resid: Optional[torch.Tensor], tape: Optional[dict]) -> None:
    """out = w3(silu(w1 h) * w2 h)  /  c_proj(gelu(c_fc h)),  h = norm2 x  (+ resid) on the n images of x [n*T, D]
    (layers/block.py:294).  A tape dict is filled with what the backward reads: x, rstd / mean, h, pre, hid."""
    dev, D, Hd = x.device, W.D, bw.hidden
    M = n * T
    act = BF if mode == "bf16" else F32
    h = norm(x, M, D, bw.n2_w, bw.n2_b, W.eps, mode, want="op", tape=tape)
    hid = _e((M, Hd), act, dev)
    if W.ffn == "swiglu" and mode == "bf16" and SPLIT_EPILOGUES and not FUSED_SWIGLU:
        pre = _e((M, 2 * Hd), BF, dev)
        linear(h, bw.fc1, pre, M, mode)
        lib.swiglu_fwd(pre, hid, M, Hd)
    elif W.ffn == "swiglu":
        pre = _e((M, 2 * Hd), BF, dev) if tape is not None else None
        linear(h, bw.fc1, hid, M, mode, act=lib.ACT_SWIGLU8, ldo=Hd, out2=pre)
    else:
        pre = _e((M, Hd), BF, dev) if tape is not None else None
        linear(h, bw.fc1, hid, M, mode, act=lib.ACT_GELU, out2=pre)
    linear(operand(hid, M, Hd, mode), bw.fc2, out, M, mode, resid=resid)
    if tape is not None:
        tape.update(x=x, h=h, pre=pre, hid=hid)


def tower_blocks(W: TowerW, x: torch.Tensor, B: int, T: int, rope, mode: str, *, causal: bool = False,
                 tape: Optional[list] = None, taps: Optional[Dict[int, torch.Tensor]] = None,
                 drop: Optional[DropPlan] = None, hook: Optional[Callable[[int, torch.Tensor], None]] = None) -> torch.Tensor:
    """The block loop (encoders/vision_transformer.py:228-233, decoders/pixel_decoder.py:147-148,
    encoders/text_transformer.py:100-104): x [B*T, D] residual stream (fp32, or bf16 for the autocast decoder).
    Inference updates x in place; with a tape every sub-layer writes a fresh stream buffer and every block appends
    {"attn": entry, "ffn": entry}, each entry holding what that sub-layer's backward reads plus its `subset`
    ((idx, alpha) under stochastic depth, else None).  `taps` {block index: None} is filled with copies of the stream
    after those blocks; `hook(li, x)` is called after every block with the stream itself (read it before returning:
    inference overwrites it in place)."""
    dev, D = x.device, W.D
    on_subsets = drop is not None and drop.ratio > 0.0
    if on_subsets and (mode != "bf16" or W.stream_bf16 or W.ffn != "swiglu" or causal):
        raise NotImplementedError("batch-subset stochastic depth is implemented for the vision trunk in bf16 mode "
                                  "(the only tower the reference applies drop_ratio to: vtp.py:275-293,452-463,487-500)")

    def run(sublayer, bw: BlockW, x: torch.Tensor, e: Optional[dict], **kw) -> torch.Tensor:
        """One sub-layer: on the whole stream with the residual added in its last GEMM's epilogue, or (stochastic
        depth, layers/block.py:201-233) on a fresh random subset of the images, gathered, whose bf16 output is added
        back into a copy of the stream with alpha = residual_scale_factor."""
        subset = None
        if not on_subsets:
            out = x if e is None else torch.empty_like(x)
            sublayer(W, bw, x, B, T, mode, out, x, e, **kw)
        else:
            idx, alpha = drop.next(B, dev)
            n = idx.numel()
            xs = _e((n * T, D), F32, dev)
            lib.gather_images(x, xs, idx, T, D)
            res = _e((n * T, D), BF, dev)
            sublayer(W, bw, xs, n, T, mode, res, None, e, **kw)
            out = x.clone()
            lib.scatter_add_images(res, out, idx, T, D, alpha)
            subset = (idx, alpha)
        if e is not None:
            e["subset"] = subset
        return out

    for li, bw in enumerate(W.blocks):
        ta, tf = ({}, {}) if tape is not None else (None, None)
        x = run(attention_sublayer, bw, x, ta, rope=rope, causal=causal)
        x = run(ffn_sublayer, bw, x, tf)
        if tape is not None:
            tape.append({"attn": ta, "ffn": tf})
        if taps is not None and li in taps:
            taps[li] = x.clone()
        if hook is not None:
            hook(li, x)
    return x


# ------------------------------------------------------------------------------------------------------ vision trunk
def trunk_tokens(W: TowerW, img: torch.Tensor, mode: str, mask_idx: Optional[torch.Tensor] = None):
    """layers/embeddings.py:61-70 + encoders/vision_transformer.py:189-219: image -> token stream [B*(1+HW), D] fp32."""
    dev = img.device
    B, C, Hi, Wi = img.shape
    ps = W.extra["patch_size"]
    gh, gw = Hi // ps, Wi // ps
    HW, T, D = gh * gw, gh * gw + 1, W.D
    img = img.to(F32).contiguous()
    patch: Lin = W.extra["patch"]
    if mode == "bf16":
        a = _e((B * HW, patch.K), BF, dev)
        lib.patchify(img, a, ps)
    else:
        a32 = _e((B * HW, patch.K), F32, dev)
        lib.patchify(img, a32, ps)
        a = operand(a32, B * HW, patch.K, mode)
    x = _e((B * T, D), F32, dev)
    linear(a, patch, x, B * HW, mode, rr_group=HW, rr_skip=1)
    lib.fill_prefix_tokens(x, W.extra["cls"], B, T, 1, D)
    if mask_idx is not None and mask_idx.numel() > 0:
        lib.apply_mask_tokens(x, W.extra["mask_token"], mask_idx, HW, T, 1, D)
    return x, (B, T, gh, gw), a


def trunk_forward(W: TowerW, img: torch.Tensor, mode: str, *, mask_idx=None, tape: Optional[dict] = None,
                  taps=None, drop: Optional[DropPlan] = None, hook=None):
    """encoders/vision_transformer.py:221-258 for one resolution group.  Returns (x_prenorm [B*T,D] fp32, meta).
    A tape dict is filled with what train.trunk_backward reads: patch_a, mask_idx, the block tape, x (the stream the
    final norm reads: pass the same tape to that norm for its statistics) and meta."""
    x, (B, T, gh, gw), a = trunk_tokens(W, img, mode, mask_idx)
    rope = W.rope(gh, gw, img.device)
    blk_tape = [] if tape is not None else None
    x = tower_blocks(W, x, B, T, rope, mode, tape=blk_tape, taps=taps, drop=drop, hook=hook)
    if tape is not None:
        tape.update(patch_a=a, mask_idx=mask_idx, blocks=blk_tape, x=x, meta=(B, T, gh, gw))
    return x, (B, T, gh, gw)


def trunk_outputs(W: TowerW, x: torch.Tensor, meta, mode: str, *, use_bottleneck: bool):
    """final norm + cls/patch split + optional bottleneck (encoders/vision_transformer.py:246-258,
    vision_transformer_bottleneck.py:66-79).  Returns dict of [B, ...] tensors in the reference's dtypes."""
    B, T, gh, gw = meta
    M, D = B * T, W.D
    dev = x.device
    if use_bottleneck and "bneck" in W.extra:
        bn: Lin = W.extra["bneck"]
        xn = norm(x, M, D, W.norm_w, W.norm_b, W.eps, mode, want="op")
        out = _e((M, bn.N), BF if mode == "bf16" else F32, dev)
        linear(xn, bn, out, M, mode)
        out = out.view(B, T, bn.N)
    else:
        out = norm(x, M, D, W.norm_w, W.norm_b, W.eps, mode, want="f32").view(B, T, D)
    return {"x_norm_clstoken": out[:, 0], "x_norm_patchtokens": out[:, 1:], "x_prenorm": x.view(B, T, D)}


def latents_nchw(patch_tokens: torch.Tensor, gh: int, gw: int) -> torch.Tensor:
    """vtp_hf/modeling_vtp.py:379-395: (B, N, C) -> (B, C, h, w); patch_tokens is a strided view [B, HW, C] of the
    [B, T, C] bottleneck output (cls row skipped via the batch stride)."""
    B, HW, C = patch_tokens.shape
    out = _e((B, C, gh, gw), patch_tokens.dtype, patch_tokens.device)
    lib.transpose_batched(patch_tokens, out, B, HW, C, in_bstride=patch_tokens.stride(0))
    return out


# ------------------------------------------------------------------------------------------------------ pixel decoder
def decoder_forward(W: TowerW, lat: torch.Tensor, mode: str) -> torch.Tensor:
    """decoders/pixel_decoder.py:134-162: latents [B, C, h, w] -> image [B, 3, 16h, 16w]."""
    B, C, gh, gw = lat.shape
    lat = lat.contiguous()
    if lat.dtype not in (BF, F32):
        lat = lat.to(F32)
    tok = _e((B * gh * gw, C), BF if mode == "bf16" else F32, lat.device)  # flatten(2).transpose(1,2)
    lib.transpose_batched(lat, tok, B, C, gh * gw)
    return decoder_tokens(W, tok, (B, gh, gw), mode)


def decoder_tokens(W: TowerW, tok: torch.Tensor, grid: Tuple[int, int, int], mode: str, *,
                   tape: Optional[dict] = None) -> torch.Tensor:
    """The decoder on token-major latents tok [B*h*w, C] of grid (B, h, w): proj_in, blocks, norm, proj_out with the
    PixelShuffle store -> image [B, 3, r h, r w].  A tape dict is filled with what train.decoder_backward reads: tok,
    the block tape, x (the stream before the norm), rstd / mean, xn (the norm output) and meta."""
    B, gh, gw = grid
    M, D, dev = B * gh * gw, W.D, tok.device
    pin: Lin = W.extra["proj_in"]
    x = _e((M, D), BF if W.stream_bf16 else F32, dev)
    linear(operand(tok, M, tok.shape[1], mode), pin, x, M, mode)
    blk_tape = [] if tape is not None else None
    x = tower_blocks(W, x, B, gh * gw, W.rope(gh, gw, dev), mode, tape=blk_tape)
    xn = norm(x, M, D, W.norm_w, W.norm_b, W.eps, mode, want="op", tape=tape)
    pout: Lin = W.extra["proj_out"]
    r = int(round((pout.N // 3) ** 0.5))
    img = _e((B, 3, gh * r, gw * r), BF if mode == "bf16" else F32, dev)
    linear(xn, pout, img, M, mode, pixel_shuffle=(r, gh, gw, 3), ldo=gw * r)
    if tape is not None:
        tape.update(tok=tok, blocks=blk_tape, x=x, xn=xn, meta=(B, gh * gw, gh, gw))
    return img


# ------------------------------------------------------------------------------------------------------ text tower
def text_forward(W: TowerW, ids: torch.Tensor, mode: str, *, tape: Optional[dict] = None) -> torch.Tensor:
    """vtp_hf/modeling_vtp.py:278-310 up to (not including) the final normalize: ids int64 [B, L] -> [B, E].  A tape
    dict is filled with what train.text_backward reads: ids, the block tape, x (the stream before the final norm),
    rstd / mean, eot, pooled and meta."""
    dev = ids.device
    B, L = ids.shape
    D = W.D
    M = B * L
    ids = ids.contiguous()
    x = _e((M, D), F32, dev)
    lib.embed_tokens(ids, W.extra["tok_emb"], W.extra["pos"], x)
    blk_tape = [] if tape is not None else None
    x = tower_blocks(W, x, B, L, None, mode, causal=True, tape=blk_tape)
    xn = norm(x, M, D, W.norm_w, W.norm_b, W.eps, mode, want="f32", tape=tape)
    # text_global_pool 'argmax' (encoders/text_transformer.py:222-224): integer index glue, bit-exact
    eot = ids.argmax(dim=-1) + torch.arange(B, device=dev) * L
    act = BF if mode == "bf16" else F32
    pooled = _e((B, D), act, dev)
    lib.gather_rows(xn, pooled, eot, D)
    proj: Lin = W.extra["proj"]
    f = _e((B, proj.N), act, dev)
    linear(operand(pooled, B, D, mode), proj, f, B, mode)
    if tape is not None:
        tape.update(ids=ids, blocks=blk_tape, x=x, eot=eot, pooled=pooled, meta=(B, L))
    return f


def l2_normalize(f: torch.Tensor, eps: float = 1e-12, norm_out=None) -> torch.Tensor:
    out = torch.empty_like(f)
    lib.l2norm_fwd(f, out, f.shape[0], f.shape[1], eps, norm_out=norm_out)
    return out
