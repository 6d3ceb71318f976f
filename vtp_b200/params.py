"""The parameter layout of every tower, stated once.

`table(cfg, head)` lists the parameters in flat-store order.  Each entry says which reference state-dict key(s) become
which kernel-layout tensor, under which store name and shape, whether AdamW decays it and whether the EMA teacher keeps
a copy.  `VTPTrainer` builds its `ParamStore` from it and imports / exports state dicts through it; `VTPModel` packs its
inference weights from it; `memory.param_count` sums it.  `geometry` gives each tower's shape and numerics, and
`assemble` turns named tensors (flat-buffer views, or packed reference tensors) into a `TowerW`.
"""
from __future__ import annotations

from typing import Callable, Dict, List, NamedTuple, Optional, Tuple

import torch

from .config import VTPConfig
from .engine import BF, F32, BlockW, Lin, TowerW, interleave8, pack_lin


def swiglu_hidden(dim: int, ratio: float, ffn_layer: str) -> int:
    """layers/block.py:176 + layers/ffn.py:71-72 (+ align variants encoders/vision_transformer.py:22-28)."""
    align = {"swiglu": 8, "swiglu32": 32, "swiglu64": 64, "swiglu128": 128}[ffn_layer]
    d = int(int(dim * ratio) * 2 / 3)
    return d + (-d % align)


class Geometry(NamedTuple):
    D: int
    heads: int
    depth: int
    hidden: int          # SwiGLU Hs / MLP width
    norm: str            # "rms" | "ln"
    eps: float
    prefix: int          # cls tokens
    ffn: str             # "swiglu" | "gelu"
    stream_bf16: bool    # residual stream dtype (the decoder's is bf16 under autocast)


_EPS = {"rmsnorm": 1e-5, "layernorm": 1e-6, "layernormbf16": 1e-5}


def geometry(cfg: VTPConfig, tower: str, mode: str = "bf16") -> Geometry:
    c = cfg
    if tower == "trunk":
        D = c.vision_embed_dim
        return Geometry(D, c.vision_num_heads, c.vision_depth, swiglu_hidden(D, c.vision_mlp_ratio, c.vision_ffn_layer),
                        "rms" if c.vision_norm_layer == "rmsnorm" else "ln", _EPS[c.vision_norm_layer], 1, "swiglu", False)
    if tower == "decoder":
        D = c.decoder_embed_dim
        return Geometry(D, c.decoder_num_heads, c.decoder_depth, swiglu_hidden(D, 4.0, c.decoder_ffn_layer),
                        "rms" if c.decoder_norm_layer == "rmsnorm" else "ln", _EPS[c.decoder_norm_layer], 0, "swiglu",
                        mode == "bf16")
    if tower == "text":
        return Geometry(c.text_embed_dim, c.text_num_heads, c.text_depth, int(c.text_embed_dim * c.text_mlp_ratio), "ln",
                        1e-5, 0, "gelu", False)
    raise KeyError(tower)


class Entry(NamedTuple):
    name: str                    # flat-store name
    shape: Tuple[int, ...]       # kernel layout
    decay: bool                  # AdamW weight decay
    teacher: bool                # kept by the EMA teacher
    ref: Tuple[str, ...]         # reference key(s): VTPModel's state dict, DINOHead's for "head." entries
    ref_shape: Tuple[int, ...]   # shape of each reference tensor
    form: str                    # "reshape" | "t" (transposed) | "swiglu" (w1, w2 interleaved by 8 rows)


def table(cfg: VTPConfig, head: Optional[Tuple[int, int, int]] = None) -> List[Entry]:
    """Every parameter of VTPModel(cfg) (but the RoPE periods buffers), then, given head = (out_dim, hidden,
    bottleneck), the DINO head's.  The trunk, the clip projection and the head have an EMA teacher (vtp.py:239-262)."""
    c = cfg
    out: List[Entry] = []

    def add(name, shape, decay, ref, ref_shape=None, form="reshape"):
        ref = (ref,) if isinstance(ref, str) else ref
        teacher = name.startswith(("trunk.", "visual_proj.", "head."))
        out.append(Entry(name, tuple(shape), decay, teacher, ref, tuple(shape if ref_shape is None else ref_shape), form))

    def blocks(tower, ref):
        """The block stack and final norm: ViT blocks (trunk, pixel decoder) or open_clip residual blocks (text)."""
        g = geometry(c, tower)
        D, H, ln, text = g.D, g.hidden, g.norm == "ln", tower == "text"
        for i in range(g.depth):
            p = f"{tower}.blocks.{i}."
            if text:
                r = f"{ref}resblocks.{i}."
                n1, n2, qkv_w, qkv_b = r + "ln_1.", r + "ln_2.", r + "attn.in_proj_weight", r + "attn.in_proj_bias"
                proj, fc2 = r + "attn.out_proj.", r + "mlp.c_proj."
            else:
                r = f"{ref}blocks.{i}."
                n1, n2, qkv_w, qkv_b = r + "norm1.", r + "norm2.", r + "attn.qkv.weight", r + "attn.qkv.bias"
                proj, fc2 = r + "attn.proj.", r + "mlp.w3."
            add(p + "n1_w", (D,), False, n1 + "weight")
            if ln: add(p + "n1_b", (D,), False, n1 + "bias")
            add(p + "qkv.w", (3 * D, D), True, qkv_w); add(p + "qkv.b", (3 * D,), False, qkv_b)
            add(p + "proj.w", (D, D), True, proj + "weight"); add(p + "proj.b", (D,), False, proj + "bias")
            add(p + "n2_w", (D,), False, n2 + "weight")
            if ln: add(p + "n2_b", (D,), False, n2 + "bias")
            if text:
                add(p + "fc1.w", (H, D), True, r + "mlp.c_fc.weight"); add(p + "fc1.b", (H,), False, r + "mlp.c_fc.bias")
            else:
                add(p + "fc1.w", (2 * H, D), True, (r + "mlp.w1.weight", r + "mlp.w2.weight"), (H, D), "swiglu")
                add(p + "fc1.b", (2 * H,), False, (r + "mlp.w1.bias", r + "mlp.w2.bias"), (H,), "swiglu")
            add(p + "fc2.w", (D, H), True, fc2 + "weight"); add(p + "fc2.b", (D,), False, fc2 + "bias")
        norm = "ln_final." if text else ref + "norm."
        add(tower + ".norm_w", (D,), False, norm + "weight")
        if ln: add(tower + ".norm_b", (D,), False, norm + "bias")

    D, Dd, Dt, ps = c.vision_embed_dim, c.decoder_embed_dim, c.text_embed_dim, c.vision_patch_size
    bn = c.vision_feature_bottleneck or D
    add("trunk.patch.w", (D, 3 * ps * ps), True, "trunk.patch_embed.proj.weight", (D, 3, ps, ps))
    add("trunk.patch.b", (D,), False, "trunk.patch_embed.proj.bias")
    add("trunk.cls", (D,), False, "trunk.cls_token", (1, 1, D))
    add("trunk.mask_token", (D,), False, "trunk.mask_token", (1, D))
    blocks("trunk", "trunk.")
    if bn != D:
        add("trunk.bneck.w", (bn, D), True, "trunk.feature_bottleneck.weight")
    if c.train_clip:
        add("visual_proj.w", (Dt, D if c.vision_bottleneck_ae_only else bn), True, "visual_proj.weight")
    if head is not None:
        K, hh, hb = head
        for j, (n_out, n_in) in ((0, (hh, D)), (2, (hh, hh)), (4, (hb, hh))):
            add(f"head.mlp{j}.w", (n_out, n_in), True, f"mlp.{j}.weight"); add(f"head.mlp{j}.b", (n_out,), False, f"mlp.{j}.bias")
        add("head.last_v", (K, hb), True, "last_layer.weight_v")
        add("head.last_g", (K,), False, "last_layer.weight_g", (K, 1))
    if c.train_reconstruction:
        add("decoder.proj_in.w", (Dd, bn), True, "pixel_decoder.proj_in.weight", (Dd, bn, 1, 1))
        add("decoder.proj_in.b", (Dd,), False, "pixel_decoder.proj_in.bias")
        blocks("decoder", "pixel_decoder.")
        add("decoder.proj_out.w", (3 * 256, Dd), True, "pixel_decoder.proj_out.weight", (3 * 256, Dd, 1, 1))
        add("decoder.proj_out.b", (3 * 256,), False, "pixel_decoder.proj_out.bias")
    if c.train_clip:
        add("text.tok_emb", (c.text_vocab_size, Dt), True, "token_embedding.weight")
        add("text.pos", (c.text_context_length, Dt), False, "positional_embedding")
        blocks("text", "text_transformer.")
        add("text.proj.w", (Dt, Dt), True, "text_projection", form="t")   # x @ P  ==  linear(x, Pᵀ)
        add("logit_scale", (1,), False, "logit_scale", (1,) if c.nonscalar_logit_scale else ())
    return out


# torch.nn.utils.parametrizations.weight_norm's spelling of the DINO head's last-layer keys
_WEIGHT_NORM = {"last_layer.weight_g": "last_layer.parametrizations.weight.original0",
                "last_layer.weight_v": "last_layer.parametrizations.weight.original1"}


def to_kernel(e: Entry, src: Dict[str, torch.Tensor]) -> torch.Tensor:
    """Entry e's kernel-layout tensor from the reference tensors in src."""
    get = lambda k: src[k] if k in src else src[_WEIGHT_NORM[k]]
    if e.form == "swiglu":
        t = interleave8(get(e.ref[0]), get(e.ref[1]))
    else:
        t = get(e.ref[0])
        t = t.t() if e.form == "t" else t
    return t.reshape(e.shape)


def to_reference(e: Entry, t: torch.Tensor) -> Dict[str, torch.Tensor]:
    """Entry e's reference tensors (fresh copies) from its kernel-layout tensor t."""
    if e.form == "swiglu":
        n = e.ref_shape[0]
        v = t.reshape(n // 8, 2, 8, *e.ref_shape[1:])
        return {e.ref[0]: v[:, 0].reshape(e.ref_shape).clone(), e.ref[1]: v[:, 1].reshape(e.ref_shape).clone()}
    return {e.ref[0]: t.t().contiguous() if e.form == "t" else t.reshape(e.ref_shape).clone()}


def import_reference(entries: List[Entry], view: Callable[[str], torch.Tensor], sd: Dict[str, torch.Tensor],
                     head_sd: Optional[Dict[str, torch.Tensor]] = None) -> None:
    """view(name).copy_(kernel-layout tensor) for every entry, from the model state dict sd, or from the DINOHead
    state dict head_sd for "head." entries (skipped without one)."""
    for e in entries:
        src = head_sd if e.name.startswith("head.") else sd
        if src is not None:
            view(e.name).copy_(to_kernel(e, src))


def export_reference(entries: List[Entry], view: Callable[[str], torch.Tensor]) -> Dict[str, torch.Tensor]:
    out = {}
    for e in entries:
        out.update(to_reference(e, view(e.name)))
    return out


def assemble(cfg: VTPConfig, tower: str, mode: str, vec: Callable[[str], torch.Tensor],
             lin: Callable[[str], Lin]) -> TowerW:
    """The TowerW of one tower from vec(store name) -> vector and lin(store name without ".w" / ".b") -> Lin."""
    g = geometry(cfg, tower, mode)
    W = TowerW(D=g.D, heads=g.heads, norm=g.norm, eps=g.eps, stream_bf16=g.stream_bf16, prefix=g.prefix, ffn=g.ffn)
    ln = g.norm == "ln"
    for i in range(g.depth):
        p = f"{tower}.blocks.{i}."
        W.blocks.append(BlockW(n1_w=vec(p + "n1_w"), n1_b=vec(p + "n1_b") if ln else None, qkv=lin(p + "qkv"),
                               proj=lin(p + "proj"), n2_w=vec(p + "n2_w"), n2_b=vec(p + "n2_b") if ln else None,
                               fc1=lin(p + "fc1"), fc2=lin(p + "fc2"), hidden=g.hidden))
    W.norm_w = vec(tower + ".norm_w")
    W.norm_b = vec(tower + ".norm_b") if ln else None
    if tower == "trunk":
        W.extra.update(patch=lin("trunk.patch"), patch_size=cfg.vision_patch_size, cls=vec("trunk.cls"),
                       mask_token=vec("trunk.mask_token"))
    elif tower == "decoder":
        W.extra.update(proj_in=lin("decoder.proj_in"), proj_out=lin("decoder.proj_out"))
    else:
        W.extra.update(tok_emb=vec("text.tok_emb"), pos=vec("text.pos"), proj=lin("text.proj"))
    return W


def pack_tower(sd: Dict[str, torch.Tensor], cfg: VTPConfig, tower: str, mode: str) -> TowerW:
    """Inference weights of one tower from a VTPModel state dict: GEMMs packed for `mode` by pack_lin, vectors in fp32,
    the RoPE periods as stored.  The trunk also carries the bottleneck and the clip projection when the model has them."""
    entries = {e.name: e for e in table(cfg)}
    vec = lambda name: to_kernel(entries[name], sd).detach().to(F32).contiguous()

    def lin(name):
        b = entries.get(name + ".b")
        return pack_lin(to_kernel(entries[name + ".w"], sd), None if b is None else to_kernel(b, sd), mode)

    W = assemble(cfg, tower, mode, vec, lin)
    if tower == "trunk":
        # cls + 0 * mask_token as in encoders/vision_transformer.py:198; autocast rounds the mask token to bf16
        W.extra["cls"] = (W.extra["cls"] + 0 * W.extra["mask_token"]).contiguous()
        if mode == "bf16":
            W.extra["mask_token"] = W.extra["mask_token"].to(BF).to(F32).contiguous()
        for name, key in (("trunk.bneck", "bneck"), ("visual_proj", "visual_proj")):
            if name + ".w" in entries:
                W.extra[key] = lin(name)
    if tower != "text":
        W.periods = sd[("trunk." if tower == "trunk" else "pixel_decoder.") + "rope_embed.periods"].detach().cpu()
    return W
