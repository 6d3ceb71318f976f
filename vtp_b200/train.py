"""The 3-objective training step (CLIP contrastive + DINO/iBOT self-distillation + pixel reconstruction) on the sm_90a
kernels, with hand-written backward (no torch.autograd): the H100-native counterpart of the reference's legacy
meta-arch `VTP` (vtp/models/vtp.py:88-512: forward_clip / forward_ssl_learning / forward_reconstruction,
update_teacher) plus the loss / optimiser layer that the reference does not release (SURVEY.md M3, a21).

  * parameters live in ONE flat fp32 master buffer with matching bf16 compute copy, fp32 gradient and Adam moments
    (`ParamStore`); GEMM weights are stored in kernel layout (w1|w2 8-interleaved for the SwiGLU-gate epilogue);
    `import_state_dict` / `export_state_dict` convert from/to the reference's state-dict keys;
  * one fused kernel per region does AdamW + bf16 refresh + EMA teacher (vtp.py:388-401) + gradient zeroing;
  * `save_checkpoint` / `load_checkpoint` write and restore the whole training state (format: checkpoint.py) in place,
    under a captured step graph too;
  * data parallel: gradients are all-reduced (NCCL) on the flat buffer, contrastive features are all-gathered and
    their gradients reduced back — the only two collectives on the path (SURVEY.md §8e).
Precision is the reference-under-autocast ("bf16") mode throughout.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch

from . import engine as E
from . import lib
from . import params as P
from .config import VTPConfig
from .engine import BF, F32, BlockW, Lin, TowerW, _e
from .graphs import StepGraph
from .rope import rope_periods

_ALIGN = 64  # elements; keeps every tensor 128B-aligned in the bf16 copy (TMA needs 16B)


# ------------------------------------------------------------------------------------------------------ parameters
class ParamStore:
    def __init__(self, device):
        self.device = device
        self.specs: List[Tuple[str, Tuple[int, ...], bool, bool]] = []
        self.offset: Dict[str, int] = {}
        self.shape: Dict[str, Tuple[int, ...]] = {}
        self.regions: List[Tuple[int, int, bool, bool]] = []  # (start, end, decay, teacher)

    def add(self, name, shape, decay=True, teacher=False):
        self.specs.append((name, tuple(int(s) for s in shape), bool(decay), bool(teacher)))

    def finalize(self):
        off = 0
        for teacher in (True, False):
            for decay in (True, False):
                start = off
                for name, shape, d, t in self.specs:
                    if d == decay and t == teacher:
                        self.offset[name], self.shape[name] = off, shape
                        n = 1
                        for s in shape:
                            n *= s
                        off += (n + _ALIGN - 1) // _ALIGN * _ALIGN
                if off > start:
                    self.regions.append((start, off, decay, teacher))
        self.n = off
        self.n_teacher = max([e for s, e, d, t in self.regions if t], default=0)
        dev = self.device
        self.p = torch.zeros(self.n, dtype=F32, device=dev)
        self.pb = torch.zeros(self.n, dtype=BF, device=dev)
        self.g = torch.zeros(self.n, dtype=F32, device=dev)
        self.m = torch.zeros(self.n, dtype=F32, device=dev)
        self.v = torch.zeros(self.n, dtype=F32, device=dev)
        self.tp = torch.zeros(self.n_teacher, dtype=F32, device=dev)
        self.tpb = torch.zeros(self.n_teacher, dtype=BF, device=dev)

    def _view(self, buf, name):
        o, shape = self.offset[name], self.shape[name]
        n = 1
        for s in shape:
            n *= s
        return buf[o:o + n].view(shape)

    def f32(self, name): return self._view(self.p, name)
    def bf16(self, name): return self._view(self.pb, name)
    def grad(self, name): return self._view(self.g, name)
    def exp_avg(self, name): return self._view(self.m, name)
    def exp_avg_sq(self, name): return self._view(self.v, name)
    def tf32(self, name): return self._view(self.tp, name)
    def tbf16(self, name): return self._view(self.tpb, name)

    def sync_compute_copies(self, init_teacher: bool = False):
        lib.cast_f32_to_bf16(self.p, self.pb, self.n)
        if init_teacher and self.n_teacher:
            self.tp.copy_(self.p[:self.n_teacher])
            self.tpb.copy_(self.pb[:self.n_teacher])


def store_tower(cfg: VTPConfig, names, tower: str, wv, fv) -> TowerW:
    """One tower as views of the flat buffers: GEMM weights through wv(name), vectors and biases through fv(name);
    `names` holds the store names.  The trunk also carries the bottleneck, the clip projection and the DINO head."""
    def lin(name):
        w = wv(name + ".w")
        return Lin(w, fv(name + ".b") if name + ".b" in names else None, w.shape[0], w.shape[1])

    W = P.assemble(cfg, tower, "bf16", fv, lin)
    W.periods = rope_periods(64)
    if tower == "trunk":
        W.extra.update(bneck=lin("trunk.bneck"), visual_proj=lin("visual_proj"), mlp0=lin("head.mlp0"),
                       mlp2=lin("head.mlp2"), mlp4=lin("head.mlp4"), last_v=fv("head.last_v"), last_g=fv("head.last_g"))
    return W


# ------------------------------------------------------------------------------------------------------ backward
def wgrad(dy: torch.Tensor, x: torch.Tensor, dw: torch.Tensor, Mtok: int):
    """dW[N_out, K_in] += dYᵀ X  (dY [Mtok, N_out] bf16, X [Mtok, K_in] bf16): TN GEMM, split-K + fp32 atomics."""
    n_out, k_in = dw.shape
    # split_k = -1: the library picks the split that fills its persistent grid most evenly for the tile shape it chose
    lib.gemm(dy, x, dw, M=n_out, N=k_in, K=Mtok, a_mn=True, b_mn=True, lda=dy.stride(0), ldb=x.stride(0), ldo=k_in,
             accumulate=True, split_k=-1, round_bf16=False)


def dgrad(dy: torch.Tensor, w: torch.Tensor, out: torch.Tensor, Mtok: int, **kw):
    """dX[Mtok, K_in] = dY[Mtok, N_out] · W[N_out, K_in]  (W consumed as an MN-major B operand, no transpose copy)."""
    n_out, k_in = w.shape
    lib.gemm(dy, w, out, M=Mtok, N=k_in, K=n_out, b_mn=True, lda=dy.stride(0), ldb=k_in, round_bf16=False, **kw)


def attention_backward(t: dict, do: torch.Tensor, dqkv: torch.Tensor, B: int, T: int, H: int, prefix: int, causal: bool,
                       rope):
    """dqkv = d/d(pre-RoPE qkv) of one attention sub-layer from its tape entry t (qkv, o, lse).  Up to 256 patch tokens
    the single-pass kernel holds the whole sequence in one CTA; longer non-causal sequences (images above 256x256) go
    to the streaming kernels, which need an fp32 workspace for δ = Σ dO·O laid out like lse."""
    if T - prefix > 256 and not causal:
        delta = _e((B, H, T), F32, do.device)
        lib.attention_bwd_long(t["qkv"], t["o"], do, t["lse"], delta, dqkv, B, T, H, prefix=prefix, rope=rope)
    else:
        lib.attention_bwd(t["qkv"], t["o"], do, t["lse"], dqkv, B, T, H, prefix=prefix, causal=causal, rope=rope)


def attention_sublayer_backward(W: TowerW, bw: BlockW, gw: BlockW, e: dict, gb: torch.Tensor, dh: torch.Tensor, n: int,
                                T: int, *, rope, causal: bool) -> None:
    """Reverse of engine.attention_sublayer from its tape entry e: gb (bf16 dL/d(proj output) [n*T, D]) -> dh
    (dL/d(norm1 output)); accumulates the proj and qkv weight gradients and the qkv bias gradient."""
    M, D = n * T, W.D
    do = _e((M, D), BF, gb.device)
    dgrad(gb, bw.proj.w, do, M)
    wgrad(gb, e["o"], gw.proj.w, M)
    dqkv = _e((M, 3 * D), BF, gb.device)
    attention_backward(e, do, dqkv, n, T, W.heads, W.prefix, causal, rope)
    lib.cast_colsum(dqkv, None, gw.qkv.b, M, 3 * D)
    dgrad(dqkv, bw.qkv.w, dh, M)
    wgrad(dqkv, e["h"], gw.qkv.w, M)


def ffn_sublayer_backward(W: TowerW, bw: BlockW, gw: BlockW, e: dict, gb: torch.Tensor, dh: torch.Tensor, n: int,
                          T: int) -> None:
    """Reverse of engine.ffn_sublayer from its tape entry e: gb (bf16 dL/d(fc2 output) [n*T, D]) -> dh
    (dL/d(norm2 output)); accumulates the fc2 and fc1 weight gradients and the fc1 bias gradient."""
    M, Hd = n * T, bw.hidden
    dhid = _e((M, Hd), BF, gb.device)
    dgrad(gb, bw.fc2.w, dhid, M)
    wgrad(gb, e["hid"], gw.fc2.w, M)
    dpre = torch.empty_like(e["pre"])
    gate_bwd = lib.swiglu_bwd if W.ffn == "swiglu" else lib.gelu_bwd
    gate_bwd(e["pre"], dhid, dpre, gw.fc1.b, M, Hd)
    dgrad(dpre, bw.fc1.w, dh, M)
    wgrad(dpre, e["h"], gw.fc1.w, M)


def tower_blocks_backward(W: TowerW, G: TowerW, tape: list, g: torch.Tensor, B: int, T: int, rope, causal=False):
    """Reverse of engine.tower_blocks.  g fp32 [B*T, D]: in = dL/d(stream out), out = dL/d(stream in) (in place).
    Each sub-layer's body maps the bf16 dY operand gb of its last GEMM to dh; the edges around it follow its path.
    Plain: g passes the residual unchanged, and gb with its column sums (that GEMM's bias gradient) is a by-product of
    the norm_bwd of the sub-layer differentiated before it; only the first one needs a stand-alone cast.  Subset
    (layers/block.py:201-233): d(residual) = alpha * g[idx] goes down the sub-layer, and what comes out of its norm
    backward is scatter-added into g[idx]."""
    dev, D = g.device, W.D
    M = B * T
    gb = dh = None
    if tape[-1]["ffn"]["subset"] is None:
        gb, dh = _e((M, D), BF, dev), _e((M, D), BF, dev)
        lib.cast_colsum(g, gb, G.blocks[-1].fc2.b, M, D)

    def run(body, bw, gw, e, norm_w, norm_gw, norm_gb, bias, next_bias, **kw):
        """body with its path's edges.  bias: gradient of the sub-layer's last GEMM bias; next_bias: that of the
        sub-layer differentiated next (None after the first block's attention)."""
        if e["subset"] is None:
            body(W, bw, gw, e, gb, dh, B, T, **kw)
            lib.norm_bwd(e["x"], e["rstd"], e["mean"], norm_w, dh, g, norm_gw, norm_gb, M, D,
                         gb_out=None if next_bias is None else gb, g_colsum=next_bias)
            return
        idx, alpha = e["subset"]
        n = idx.numel()
        gs = _e((n * T, D), F32, dev)
        lib.gather_images(g, gs, idx, T, D, alpha)
        gbs = _e((n * T, D), BF, dev)
        lib.cast_colsum(gs, gbs, bias, n * T, D)
        dhs = _e((n * T, D), BF, dev)
        body(W, bw, gw, e, gbs, dhs, n, T, **kw)
        gs.zero_()
        lib.norm_bwd(e["x"], e["rstd"], e["mean"], norm_w, dhs, gs, norm_gw, norm_gb, n * T, D)
        lib.scatter_add_images(gs, g, idx, T, D, 1.0)

    for li in reversed(range(len(W.blocks))):
        bw, gw, t = W.blocks[li], G.blocks[li], tape[li]
        run(ffn_sublayer_backward, bw, gw, t["ffn"], bw.n2_w, gw.n2_w, gw.n2_b, gw.fc2.b, gw.proj.b)
        run(attention_sublayer_backward, bw, gw, t["attn"], bw.n1_w, gw.n1_w, gw.n1_b, gw.proj.b,
            G.blocks[li - 1].fc2.b if li > 0 else None, rope=rope, causal=causal)
        tape[li] = None  # free the saved activations of this block
    return g


def trunk_backward(W: TowerW, G: TowerW, tape: dict, dxn: torch.Tensor, g: Optional[torch.Tensor] = None):
    """Reverse of engine.trunk_forward and the final norm from their tape: dxn (bf16 dL/d(final-norm output) [B*T, D])
    -> accumulates every trunk parameter gradient.  g: zeroed fp32 [B*T, D] to differentiate the stream into (a fresh
    one if None)."""
    B, T, gh, gw = tape["meta"]
    D, HW, M, dev = W.D, gh * gw, B * T, dxn.device
    if g is None:
        g = torch.zeros((M, D), dtype=F32, device=dev)
    lib.norm_bwd(tape["x"], tape["rstd"], tape["mean"], W.norm_w, dxn, g, G.norm_w, G.norm_b, M, D)
    tower_blocks_backward(W, G, tape["blocks"], g, B, T, W.rope(gh, gw, dev))
    gp = _e((B * HW, D), BF, dev)
    lib.strip_prefix(g, gp, G.extra["cls"], B, T, 1, D)
    mask_idx = tape["mask_idx"]
    if mask_idx is not None and mask_idx.numel() > 0:
        rows = (mask_idx // HW) * T + 1 + mask_idx % HW
        tmp = _e((mask_idx.numel(), D), F32, dev)
        lib.gather_rows(g, tmp, rows, D)
        lib.cast_colsum(tmp, None, G.extra["mask_token"], mask_idx.numel(), D)
        zeros = torch.zeros(D, dtype=F32, device=dev)
        lib.apply_mask_tokens(gp, zeros, mask_idx, HW, HW, 0, D)
    wgrad(gp, tape["patch_a"], G.extra["patch"].w, B * HW)
    lib.cast_colsum(gp, None, G.extra["patch"].b, B * HW, D)


def decoder_backward(W: TowerW, G: TowerW, tape: dict, dY: torch.Tensor, dtok: torch.Tensor, **row_map):
    """Reverse of engine.decoder_tokens from its tape: dY (bf16 dL/d(proj_out output) [B*h*w, 3r²]) -> dtok
    (dL/d(tok), written through the caller's `row_map` GEMM epilogue arguments); accumulates every decoder gradient."""
    B, HW, gh, gw = tape["meta"]
    D, M, dev = W.D, B * HW, dY.device
    pout, pin = W.extra["proj_out"], W.extra["proj_in"]
    dxn = _e((M, D), BF, dev)
    dgrad(dY, pout.w, dxn, M)
    wgrad(dY, tape["xn"], G.extra["proj_out"].w, M)
    lib.cast_colsum(dY, None, G.extra["proj_out"].b, M, pout.N)
    g = torch.zeros((M, D), dtype=F32, device=dev)
    lib.norm_bwd(tape["x"], tape["rstd"], tape["mean"], W.norm_w, dxn, g, G.norm_w, G.norm_b, M, D)
    tower_blocks_backward(W, G, tape["blocks"], g, B, HW, W.rope(gh, gw, dev))
    gb = _e((M, D), BF, dev)
    lib.cast_colsum(g, gb, G.extra["proj_in"].b, M, D)
    dgrad(gb, pin.w, dtok, M, **row_map)
    wgrad(gb, tape["tok"], G.extra["proj_in"].w, M)


def text_backward(W: TowerW, G: TowerW, tape: dict, dft_raw: torch.Tensor):
    """Reverse of engine.text_forward from its tape: dft_raw (bf16 dL/d(projected feature) [B, E]) -> accumulates
    every text-tower parameter gradient."""
    B, L = tape["meta"]
    D, M, dev = W.D, B * L, dft_raw.device
    dpool = _e((B, D), F32, dev)
    dgrad(dft_raw, W.extra["proj"].w, dpool, B)
    wgrad(dft_raw, tape["pooled"], G.extra["proj"].w, B)
    dxn32 = torch.zeros((M, D), dtype=F32, device=dev)
    lib.scatter_add_rows(dpool, dxn32, tape["eot"], D)
    dxn = _e((M, D), BF, dev)
    lib.cast_colsum(dxn32, dxn, None, M, D)
    g = torch.zeros((M, D), dtype=F32, device=dev)
    lib.norm_bwd(tape["x"], tape["rstd"], tape["mean"], W.norm_w, dxn, g, G.norm_w, G.norm_b, M, D)
    tower_blocks_backward(W, G, tape["blocks"], g, B, L, None, causal=True)
    lib.scatter_add_rows(g, G.extra["tok_emb"], tape["ids"].reshape(-1), D)
    lib.cast_colsum(g, None, G.extra["pos"].view(-1), B, L * D, ldx=L * D)


def grad_buckets(offset: Dict[str, int], n: int) -> Dict[str, List[Tuple[int, int]]]:
    """Contiguous ranges of the flat gradient buffer per tower.  A tower's gradient is FINAL as soon as its last
    backward of the step has run: text tower + clip projection + logit scale after the contrastive objective, DINO head
    after the SSL head backward, pixel decoder after its backward inside the reconstruction objective; the trunk (all
    three objectives accumulate into it) only at the end of the step.  Each finished bucket is all-reduced right away
    (NCCL's own stream) under the remaining backward; only the trunk bucket is exposed."""
    def bucket_of(name: str) -> str:
        if name.startswith("text.") or name.startswith("visual_proj") or name == "logit_scale":
            return "text"
        if name.startswith("head."):
            return "head"
        if name.startswith("decoder."):
            return "decoder"
        return "trunk"
    spans = sorted((off, name) for name, off in offset.items())
    out: Dict[str, List[Tuple[int, int]]] = {"text": [], "head": [], "decoder": [], "trunk": []}
    for i, (off, name) in enumerate(spans):
        end = spans[i + 1][0] if i + 1 < len(spans) else n   # incl. the alignment padding behind the tensor
        r = out[bucket_of(name)]
        if r and r[-1][1] == off:
            r[-1] = (r[-1][0], end)
        else:
            r.append((off, end))
    return out


# ------------------------------------------------------------------------------------------------------ trainer
@dataclass
class TrainConfig:
    lr: float = 1e-4
    beta1: float = 0.9
    beta2: float = 0.95
    eps: float = 1e-8
    weight_decay: float = 0.05
    teacher_momentum: float = 0.994
    teacher_temp: float = 0.07
    student_temp: float = 0.1
    center_momentum: float = 0.9
    head_out_dim: int = 65536
    head_hidden: int = 2048
    head_bottleneck: int = 256
    n_local_crops: int = 8
    w_clip: float = 1.0
    w_ssl: float = 1.0
    w_rec: float = 1.0
    lpips_weight: float = 1.0
    # contrastive exchange (collective C2): "nccl" = all-gather + local-row logits + all-reduced cross terms;
    # "p2p" = peer-memory gather fused with the full logits / softmax-CE (csrc/clip.cu), no backward collective
    clip_exchange: str = "nccl"
    # activation-memory control (configs 3/4: VTP-Base/Large at 256 images per GPU exceed 180 GB of saved activations
    # in one piece, see vtp_b200/memory.py): source images per forward+backward pass of the SSL / reconstruction
    # objectives; gradients accumulate in the flat buffer, losses and centre statistics are those of the whole batch.
    # 0 = the whole per-GPU batch at once.
    ssl_chunk: int = 0
    rec_chunk: int = 0
    # batch-subset stochastic depth of the student trunk per objective (vtp.py:275-293 clip_drop_rate, :452-463
    # ssl_drop_rate, :487-500 rec_drop_rate; layers/block.py:20-118,201-298); 0 = the plain residual path
    clip_drop_rate: float = 0.0
    ssl_drop_rate: float = 0.0
    rec_drop_rate: float = 0.0
    # collective C3: "end" = ONE all-reduce of the flat gradient buffer after the last backward; "overlap" = every tower's
    # bucket is all-reduced as soon as it is final, under the remaining backward (env VTP_GRAD_REDUCE overrides).
    # "end" is the default: overlapped collectives run NCCL's CTAs beside the persistent, full-machine GEMM and attention
    # kernels and take SMs away from them for the whole backward.
    grad_reduce: str = "end"


class VTPTrainer:
    def __init__(self, cfg: VTPConfig, tc: Optional[TrainConfig] = None, device="cuda", process_group=None):
        self.cfg, self.tc = cfg, tc or TrainConfig()
        self.device = torch.device(device)
        self.pg = process_group
        import torch.distributed as dist
        self.world = dist.get_world_size(process_group) if (dist.is_available() and dist.is_initialized()) else 1
        self.rank = dist.get_rank(process_group) if self.world > 1 else 0
        lib.check(lib.load().vtp_check_device(), "vtp_check_device")
        c = cfg
        if c.vision_norm_layer != "rmsnorm" or c.decoder_norm_layer not in ("layernorm", "layernormbf16"):
            raise NotImplementedError("trainer supports the reference defaults: rmsnorm trunk, layernorm decoder")
        from .model import check_head_dims
        if not (c.train_clip and c.train_reconstruction):
            raise NotImplementedError("the trainer runs all three objectives: train_clip and train_reconstruction must be on")
        if not c.vision_bottleneck_ae_only:
            raise NotImplementedError("the trainer projects the trunk's cls token, not its bottleneck features, for the "
                                      "contrastive objective (vision_bottleneck_ae_only=True)")
        check_head_dims(c)
        self.D, self.Dt = c.vision_embed_dim, c.text_embed_dim
        self.hs = P.geometry(c, "trunk").hidden
        self.bn = c.vision_feature_bottleneck
        K, hb = self.tc.head_out_dim, self.tc.head_bottleneck
        self.table = P.table(c, (K, self.tc.head_hidden, hb))
        st = ParamStore(self.device)
        for e in self.table:
            st.add(e.name, e.shape, e.decay, e.teacher)
        st.finalize()
        self.store = st
        self._build_towers()
        self.step_count = 0
        self.lpips = None  # perceptual term of the reconstruction loss, see enable_lpips()
        self.peer = None   # peer-memory exchange buffers of the contrastive objective (clip_exchange == "p2p")
        self.loss_acc = torch.zeros(8, dtype=F32, device=self.device)  # clip, dino_local, dino_global, ibot, rec
        self.center_dino = torch.zeros(K, dtype=F32, device=self.device)
        self.center_ibot = torch.zeros(K, dtype=F32, device=self.device)
        self.head_wn = _e((K, hb), BF, self.device)       # weight-normed last layer (student), rebuilt every step
        self.head_wn_t = _e((K, hb), BF, self.device)     # teacher
        self.head_vnorm = _e((K,), F32, self.device)
        # device-resident step state (csrc/backward.cu hyper_tick_kernel): {step, 1-b1^t, 1-b2^t, lr, wd, teacher momentum}
        self.hyper = torch.zeros(8, dtype=F32, device=self.device)
        self.hyper[3:6] = torch.tensor([self.tc.lr, self.tc.weight_decay, self.tc.teacher_momentum], device=self.device)
        self._sched = (None, None, None, 0)     # device tables (lr, wd, momentum) + common length
        self._buckets = self._grad_buckets()    # collective C3: gradient all-reduce per tower, overlapped with backward
        self._pending = []                      # in-flight all-reduce handles of the current step
        self._started = set()                   # buckets whose all-reduce has been started this step
        self._graph = None                      # CUDA graph of the whole step, see capture_step()
        self.reset_parameters()

    def _grad_buckets(self) -> Dict[str, List[Tuple[int, int]]]:
        return grad_buckets(self.store.offset, self.store.n)

    def _grad_reduce_mode(self) -> str:
        import os
        mode = os.environ.get("VTP_GRAD_REDUCE", self.tc.grad_reduce)
        if mode not in ("overlap", "end"):
            raise ValueError(f"grad_reduce must be 'overlap' or 'end', got {mode!r}")
        return mode

    def _reduce_bucket(self, which: str, final: bool = False):
        """Start the all-reduce of one finished gradient bucket (no-op single rank / already started this step)."""
        if self.world == 1 or which in self._started:
            return
        if not final and self._grad_reduce_mode() == "end":
            return                       # deferred: allreduce_grads() starts every bucket after the last backward
        import torch.distributed as dist
        self._started.add(which)
        for a, b in self._buckets[which]:
            self._pending.append(dist.all_reduce(self.store.g[a:b], group=self.pg, async_op=True))

    def enable_lpips(self, module=None, seed: int = 0, chunk: int = 32):
        """Attach the LPIPS term (utils/lpips.py) to the reconstruction loss: rec = L1 + lpips_weight * LPIPS.  Without
        a supplied module, frozen seeded-random VGG16/lin weights are used (the trained ones need network access)."""
        from .lpips import LPIPSLoss
        self.lpips = module if module is not None else LPIPSLoss.random_init(seed, device=self.device, chunk=chunk)
        return self.lpips

    # -------------------------------------------------------------- towers as views of the flat buffers
    def _build_towers(self):
        st = self.store
        views = {"param": (st.bf16, st.f32), "teacher": (st.tbf16, st.tf32), "grad": (st.grad, st.grad)}
        self.towers = {(tower, kind): store_tower(self.cfg, st.offset, tower, *views[kind])
                       for tower, kinds in (("trunk", ("param", "teacher", "grad")), ("decoder", ("param", "grad")),
                                            ("text", ("param", "grad"))) for kind in kinds}

    # -------------------------------------------------------------- init / state-dict exchange
    @torch.no_grad()
    def reset_parameters(self, seed: int = 0):
        g = torch.Generator(device="cpu").manual_seed(seed)
        st = self.store
        for name, shape, decay, _ in st.specs:
            v = st.f32(name)
            leaf = name.rsplit(".", 1)[-1]
            if name == "logit_scale":
                v.fill_(math.log(1 / 0.07))
            elif leaf in ("n1_w", "n2_w", "norm_w", "last_g"):
                v.fill_(1.0)
            elif leaf in ("b", "n1_b", "n2_b", "norm_b", "mask_token"):
                v.zero_()
            elif name == "text.pos":
                v.copy_(torch.randn(shape, generator=g) * 0.01)
            else:
                std = 0.02
                v.copy_((torch.randn(shape, generator=g) * std).clamp_(-2 * std, 2 * std))
        st.sync_compute_copies(init_teacher=True)

    @torch.no_grad()
    def import_state_dict(self, sd: Dict[str, torch.Tensor], head_sd: Optional[Dict[str, torch.Tensor]] = None):
        """Load a reference-format VTPModel state dict (+ optional DINOHead state dict with keys mlp.0.weight, ...,
        last_layer.weight_g / weight_v or the parametrizations.* spelling)."""
        P.import_reference(self.table, self.store.f32, sd, head_sd)
        self.store.sync_compute_copies(init_teacher=True)

    @torch.no_grad()
    def export_state_dict(self, teacher: bool = False) -> Dict[str, torch.Tensor]:
        """Student weights in the reference's VTPModel state-dict format.  teacher=True takes the trunk and the clip
        projection from the EMA teacher instead (what DINOv2-style evaluation scores); the pixel decoder and the text
        tower, which the teacher does not have, still come from the student."""
        st = self.store
        ema = {e.name for e in self.table if e.teacher} if teacher else set()
        out = P.export_reference([e for e in self.table if not e.name.startswith("head.")],
                                 lambda name: st.tf32(name) if name in ema else st.f32(name))
        out["trunk.rope_embed.periods"] = rope_periods(64).to(self.device)
        out["pixel_decoder.rope_embed.periods"] = rope_periods(64).to(self.device)
        return out

    # -------------------------------------------------------------- checkpoints (format: checkpoint.py)
    def _checkpoint_tensors(self) -> Dict[str, torch.Tensor]:
        """Views of every buffer a checkpoint holds, named as checkpoint.state_spec names them.  The bf16 compute
        copies are not among them (re-derived on load), nor the gradient (zeroed by the optimiser at every step)."""
        st = self.store
        out = {}
        for prefix, view in (("param", st.f32), ("exp_avg", st.exp_avg), ("exp_avg_sq", st.exp_avg_sq)):
            out.update({f"{prefix}/{e.name}": view(e.name) for e in self.table})
        out.update({f"teacher/{e.name}": st.tf32(e.name) for e in self.table if e.teacher})
        out["center/dino"], out["center/ibot"] = self.center_dino, self.center_ibot
        out["optimizer/hyper"] = self.hyper[0:3]      # step, 1 - beta1^step, 1 - beta2^step
        return out

    @torch.no_grad()
    def save_checkpoint(self, path: str, pipeline=None) -> None:
        """Write the whole training state at a step boundary into the directory `path` (atomically, see checkpoint.py):
        fp32 master weights, Adam moments, EMA teacher, DINO / iBOT centres, the optimiser step, this rank's CUDA
        generator (stochastic-depth subsets) and, given `pipeline` (data.TrainBatchPipeline), its RNG streams.  Every
        rank calls it.  Settings are not state: learning rate, weight decay, momentum and their schedules come from the
        code that resumes; the configs are recorded in the manifest only."""
        import dataclasses

        from . import checkpoint as C
        torch.cuda.current_stream(self.device).synchronize()
        C.save(path, self._checkpoint_tensors(), step=self.step_count, cuda_rng=torch.cuda.get_rng_state(self.device),
               pipeline=None if pipeline is None else pipeline.state_dict(),
               config={"model": self.cfg.to_dict(), "train": dataclasses.asdict(self.tc)},
               rank=self.rank, world=self.world, process_group=self.pg)

    @torch.no_grad()
    def load_checkpoint(self, path: str, rng: bool = True, pipeline=None) -> int:
        """Restore what save_checkpoint wrote, in place: every buffer is overwritten by copy_, none is rebound, so a
        step graph captured before the load replays from the restored state.  The whole checkpoint is validated first;
        a mismatch (another preset, another head_out_dim, ...) raises ValueError and changes nothing.  rng=False skips
        the per-rank RNG state: the way to resume on another number of GPUs (the rest of the state does not depend on
        the world size).  Given `pipeline`, its RNG streams are restored too.  Returns the restored step."""
        from . import checkpoint as C
        spec = C.state_spec(self.table, self.tc.head_out_dim)
        ck = C.load(path, spec, rank=self.rank, world=self.world, rng=rng, pipeline=pipeline is not None)
        if pipeline is not None:
            pipeline.check_loadable()
        torch.cuda.current_stream(self.device).synchronize()
        for name, view in self._checkpoint_tensors().items():
            view.copy_(ck.tensor(name))
        st = self.store
        st.g.zero_()                                      # as at any step boundary
        lib.cast_f32_to_bf16(st.p, st.pb, st.n)          # the bf16 copies, as the fused optimiser rounds them
        if st.n_teacher:
            lib.cast_f32_to_bf16(st.tp, st.tpb, st.n_teacher)
        self.step_count = ck.step
        if rng:
            torch.cuda.set_rng_state(ck.cuda_rng, self.device)
        if pipeline is not None:
            pipeline.load_state_dict(ck.pipeline)
        torch.cuda.current_stream(self.device).synchronize()
        return ck.step

    # -------------------------------------------------------------- pieces shared by the objectives
    def _drop(self, ratio: float):
        """DropPlan of one student trunk pass (None when the objective's drop rate is 0); `drop_presets` (tests) supplies
        fixed subsets instead of random permutations."""
        if ratio <= 0.0:
            return None
        preset = self.drop_presets.pop(0) if getattr(self, "drop_presets", None) else None
        return E.DropPlan(ratio, self.world, self.rank, preset=preset)

    # -------------------------------------------------------------- objective 1: CLIP (vtp.py:340-363 + ClipLoss)
    def clip_fwd_bwd(self, image: torch.Tensor, text: torch.Tensor, weight: float = 1.0):
        import torch.distributed as dist
        dev = self.device
        W, G = self.towers[("trunk", "param")], self.towers[("trunk", "grad")]
        Wt, Gt = self.towers[("text", "param")], self.towers[("text", "grad")]
        D, Dt = self.D, self.Dt
        # ---- image tower -> cls -> visual_proj -> normalise
        tp_i = {}
        x, (B, T, gh, gw) = E.trunk_forward(W, image, "bf16", tape=tp_i, drop=self._drop(self.tc.clip_drop_rate))
        xn = E.norm(x, B * T, D, W.norm_w, None, W.eps, "bf16", want="f32", tape=tp_i)
        cls_rows = torch.arange(B, device=dev, dtype=torch.long) * T
        cls = _e((B, D), BF, dev)
        lib.gather_rows(xn, cls, cls_rows, D)
        vp: Lin = W.extra["visual_proj"]
        fi_raw = _e((B, Dt), BF, dev)
        lib.gemm(cls, vp.w, fi_raw, M=B, N=Dt, K=D)
        nrm_i = _e((B,), F32, dev)
        # ---- text tower
        tp_t = {}
        ft_raw = E.text_forward(Wt, text, "bf16", tape=tp_t)
        nrm_t = _e((B,), F32, dev)
        if self._clip_exchange() == "p2p":
            dfi, dft = self._clip_loss_p2p(fi_raw, ft_raw, nrm_i, nrm_t, B, weight)
            self._clip_backward(tp_i, tp_t, cls, self.peer.img, self.peer.txt, nrm_i, nrm_t, dfi, dft)
            return
        fi = torch.empty_like(fi_raw)
        lib.l2norm_fwd(fi_raw, fi, B, Dt, 1e-12, norm_out=nrm_i)
        ft = torch.empty_like(ft_raw)
        lib.l2norm_fwd(ft_raw, ft, B, Dt, 1e-12, norm_out=nrm_t)
        # ---- contrastive loss over the global batch (features all-gathered: collective C2)
        if self.world > 1:
            fi_all = _e((self.world * B, Dt), BF, dev)
            ft_all = _e((self.world * B, Dt), BF, dev)
            dist.all_gather_into_tensor(fi_all, fi, group=self.pg)
            dist.all_gather_into_tensor(ft_all, ft, group=self.pg)
        else:
            fi_all, ft_all = fi, ft
        Bg = fi_all.shape[0]
        Bgp = (Bg + 7) // 8 * 8
        sim_i = _e((B, Bgp), F32, dev)
        sim_t = _e((B, Bgp), F32, dev)
        pad = lambda t: t if Bg == Bgp else torch.cat([t, torch.zeros(Bgp - Bg, Dt, dtype=BF, device=dev)])
        fi_allp, ft_allp = pad(fi_all), pad(ft_all)
        lib.gemm(fi, ft_allp, sim_i, M=B, N=Bgp, K=Dt, round_bf16=False)
        lib.gemm(ft, fi_allp, sim_t, M=B, N=Bgp, K=Dt, round_bf16=False)
        Gi = torch.zeros((B, Bgp), dtype=BF, device=dev)
        Gt_ = torch.zeros((B, Bgp), dtype=BF, device=dev)
        ls = self.store.f32("logit_scale")
        dls = self.store.grad("logit_scale")
        coef = weight * 0.5 / B
        lib.softmax_ce(sim_i, B, Bg, self.rank * B, Gi, coef, self.loss_acc[0:1], dls, log_scale=ls)
        lib.softmax_ce(sim_t, B, Bg, self.rank * B, Gt_, coef, self.loss_acc[0:1], dls, log_scale=ls)
        # d f_i(local) = Gi · T_all + [Gtᵀ · T_local]_(all ranks summed, local slice)   (and symmetrically for text)
        dfi = _e((B, Dt), F32, dev)
        dft = _e((B, Dt), F32, dev)
        lib.gemm(Gi, ft_allp, dfi, M=B, N=Dt, K=Bgp, b_mn=True, ldb=Dt, round_bf16=False)
        lib.gemm(Gt_, fi_allp, dft, M=B, N=Dt, K=Bgp, b_mn=True, ldb=Dt, round_bf16=False)
        if self.world > 1:
            cross_i = _e((Bgp, Dt), F32, dev)
            cross_t = _e((Bgp, Dt), F32, dev)
            lib.gemm(Gt_, ft, cross_i, M=Bgp, N=Dt, K=B, a_mn=True, b_mn=True, lda=Bgp, ldb=Dt, round_bf16=False)
            lib.gemm(Gi, fi, cross_t, M=Bgp, N=Dt, K=B, a_mn=True, b_mn=True, lda=Bgp, ldb=Dt, round_bf16=False)
            dist.all_reduce(cross_i, group=self.pg)
            dist.all_reduce(cross_t, group=self.pg)
            lib.axpby(dfi, cross_i[self.rank * B:(self.rank + 1) * B].contiguous(), 1.0, 1.0, B * Dt)
            lib.axpby(dft, cross_t[self.rank * B:(self.rank + 1) * B].contiguous(), 1.0, 1.0, B * Dt)
        else:
            lib.gemm(Gt_, ft, dfi, M=B, N=Dt, K=B, a_mn=True, b_mn=True, lda=Bgp, ldb=Dt, accumulate=True, round_bf16=False)
            lib.gemm(Gi, fi, dft, M=B, N=Dt, K=B, a_mn=True, b_mn=True, lda=Bgp, ldb=Dt, accumulate=True, round_bf16=False)
        self._clip_backward(tp_i, tp_t, cls, fi, ft, nrm_i, nrm_t, dfi, dft)

    def _clip_exchange(self) -> str:
        import os
        mode = os.environ.get("VTP_CLIP_EXCHANGE", self.tc.clip_exchange)
        if mode not in ("nccl", "p2p"):
            raise ValueError(f"clip_exchange must be 'nccl' or 'p2p', got {mode!r}")
        return mode

    def _clip_loss_p2p(self, fi_raw, ft_raw, nrm_i, nrm_t, B: int, weight: float):
        """Collective C2 over NVLink peer memory (csrc/clip.cu): the normalised features are written straight into this
        rank's exchange buffer, one kernel gathers every rank's rows and forms the full Bg x Bg logits, two small kernels
        do both softmax directions; returns d(Σ_ranks L_local)/d(f_local) for images and captions (fp32 [B, E])."""
        from .comm import PeerFeatures
        dev, Dt = self.device, self.Dt
        if self.peer is None or self.peer.B != B:
            if self.peer is not None:
                self.peer.check()            # a timed-out barrier of the old buffer must not be dropped silently
                self.peer.close()
            self.peer = PeerFeatures(B, Dt, dev, self.pg, world=self.world, rank=self.rank)
        pf = self.peer
        lib.l2norm_fwd(fi_raw, pf.img, B, Dt, 1e-12, norm_out=nrm_i)
        lib.l2norm_fwd(ft_raw, pf.txt, B, Dt, 1e-12, norm_out=nrm_t)
        Bg = self.world * B
        Bgp = (Bg + 7) // 8 * 8
        S = _e((Bg, Bgp), F32, dev)
        St = _e((Bg, Bgp), F32, dev)
        fi_all = torch.zeros((Bgp, Dt), dtype=BF, device=dev)
        ft_all = torch.zeros((Bgp, Dt), dtype=BF, device=dev)
        pf.barrier(self.loss_acc[0:1])     # every rank's features are written (time-out -> NaN contrastive loss)
        lib.clip_gather_logits(pf.img_ptrs, pf.txt_ptrs, B, Dt, S, St, fi_all, ft_all)
        pf.barrier(self.loss_acc[0:1])     # every rank has read them: the buffers may be overwritten by the next step
        ls = self.store.f32("logit_scale")
        dls = self.store.grad("logit_scale")
        coef = weight * 0.5 / B
        lse = _e((2, Bg), F32, dev)
        lib.clip_lse(S, St, Bg, self.rank * B, B, ls, coef, lse, self.loss_acc[0:1], dls)
        dMi = _e((B, Bgp), BF, dev)
        dMt = _e((B, Bgp), BF, dev)
        lib.clip_grad(S, St, Bg, self.rank * B, B, ls, coef, lse, dMi, dMt)
        dfi = _e((B, Dt), F32, dev)
        dft = _e((B, Dt), F32, dev)
        lib.gemm(dMi, ft_all, dfi, M=B, N=Dt, K=Bgp, b_mn=True, ldb=Dt, round_bf16=False)
        lib.gemm(dMt, fi_all, dft, M=B, N=Dt, K=Bgp, b_mn=True, ldb=Dt, round_bf16=False)
        return dfi, dft

    def _clip_backward(self, tp_i, tp_t, cls, fi, ft, nrm_i, nrm_t, dfi, dft):
        """dfi / dft (fp32 dL/d(normalised feature)) back through the L2 norms, the image head and both towers."""
        dev = self.device
        W, G = self.towers[("trunk", "param")], self.towers[("trunk", "grad")]
        B, T = tp_i["meta"][:2]
        D, Dt = self.D, self.Dt
        dfi_raw = _e((B, Dt), BF, dev)
        lib.l2norm_bwd(fi, nrm_i, dfi, dfi_raw, B, Dt)
        dxn = torch.zeros((B * T, D), dtype=BF, device=dev)
        dgrad(dfi_raw, W.extra["visual_proj"].w, dxn, B, ldo=T * D)   # row b of d(cls) lands on token row b*T
        wgrad(dfi_raw, cls, G.extra["visual_proj"].w, B)
        trunk_backward(W, G, tp_i, dxn)
        dft_raw = _e((B, Dt), BF, dev)
        lib.l2norm_bwd(ft, nrm_t, dft, dft_raw, B, Dt)
        text_backward(self.towers[("text", "param")], self.towers[("text", "grad")], tp_t, dft_raw)

    # -------------------------------------------------------------- objective 3: reconstruction (vtp.py:487-512)
    def rec_fwd_bwd(self, image: torch.Tensor, weight: float = 1.0, return_image: bool = False,
                    norm_B: Optional[int] = None, final_group: bool = False):
        """norm_B: batch size the loss is normalised by (the whole per-GPU batch when `image` is one chunk of it)."""
        dev = self.device
        W, G = self.towers[("trunk", "param")], self.towers[("trunk", "grad")]
        Wd, Gd = self.towers[("decoder", "param")], self.towers[("decoder", "grad")]
        D, bn = self.D, self.bn
        tp_e, tp_d = {}, {}
        x, (B, T, gh, gw) = E.trunk_forward(W, image, "bf16", tape=tp_e, drop=self._drop(self.tc.rec_drop_rate))
        M, HW = B * T, gh * gw
        nB = norm_B if norm_B is not None else B
        xn = E.norm(x, M, D, W.norm_w, None, W.eps, "bf16", want="op", tape=tp_e)
        bneck: Lin = W.extra["bneck"]
        tok = _e((B * HW, bn), BF, dev)                  # latents as decoder tokens (cls rows dropped in the epilogue)
        lib.gemm(xn, bneck.w, tok, M=M, N=bn, K=D, rr_group=T, rr_skip=-1)
        rec = E.decoder_tokens(Wd, tok, (B, gh, gw), "bf16", tape=tp_d)
        r = rec.shape[-1] // gw
        # ---- loss: L1 (+ LPIPS gradient if a perceptual module is attached)
        dlp = None
        if getattr(self, "lpips", None) is not None and self.tc.lpips_weight > 0:
            dlp = self.lpips.loss_and_grad(rec, image, weight * self.tc.lpips_weight / nB, self.loss_acc[5:6])
        dY = _e((B * HW, 3 * r * r), BF, dev)
        lib.recon_l1_grad(rec, image.contiguous(), dlp, dY, self.loss_acc[4:5], B, 3, gh, gw, r,
                          weight / (rec.numel() // B * nB))
        dz = torch.zeros((M, bn), dtype=BF, device=dev)  # d(latent tokens), re-expanded to [B*T] rows (cls rows = 0)
        decoder_backward(Wd, Gd, tp_d, dY, dz, rr_group=HW, rr_skip=1)
        if final_group:
            self._reduce_bucket("decoder")   # pixel-decoder gradient is final: all-reduce under the encoder backward
        # ---- encoder side
        dxn = _e((M, D), BF, dev)
        dgrad(dz, bneck.w, dxn, M)
        wgrad(dz, xn, G.extra["bneck"].w, M)
        trunk_backward(W, G, tp_e, dxn)
        return rec if return_image else None

    # -------------------------------------------------------------- DINO head (heads/dino_head.py:65-126)
    def _head_prepare(self):
        W, Wt = self.towers[("trunk", "param")], self.towers[("trunk", "teacher")]
        K, hb = self.tc.head_out_dim, self.tc.head_bottleneck
        lib.weight_norm_fwd(W.extra["last_v"], W.extra["last_g"], self.head_wn, self.head_vnorm, K, hb)
        lib.weight_norm_fwd(Wt.extra["last_v"], Wt.extra["last_g"], self.head_wn_t, None, K, hb)

    def _head_fwd(self, W: TowerW, wn: torch.Tensor, x: torch.Tensor, tape: Optional[dict]):
        dev = self.device
        Tn, D = x.shape
        hh, hb, K = self.tc.head_hidden, self.tc.head_bottleneck, self.tc.head_out_dim
        m0, m2, m4 = W.extra["mlp0"], W.extra["mlp2"], W.extra["mlp4"]
        pre1 = _e((Tn, hh), BF, dev) if tape is not None else None
        h1 = _e((Tn, hh), BF, dev)
        lib.gemm(x, m0.w, h1, M=Tn, N=hh, K=D, bias=m0.b, act=lib.ACT_GELU, out2=pre1)
        pre2 = _e((Tn, hh), BF, dev) if tape is not None else None
        h2 = _e((Tn, hh), BF, dev)
        lib.gemm(h1, m2.w, h2, M=Tn, N=hh, K=hh, bias=m2.b, act=lib.ACT_GELU, out2=pre2)
        h3 = _e((Tn, hb), BF, dev)
        lib.gemm(h2, m4.w, h3, M=Tn, N=hb, K=hh, bias=m4.b)
        y = _e((Tn, hb), BF, dev)
        nrm = _e((Tn,), F32, dev)
        lib.l2norm_fwd(h3, y, Tn, hb, 1e-12, norm_out=nrm)
        logits = _e((Tn, K), BF, dev)
        lib.gemm(y, wn, logits, M=Tn, N=K, K=hb)
        if tape is not None:
            tape.update(x=x, pre1=pre1, h1=h1, pre2=pre2, h2=h2, y=y, nrm=nrm)
        return logits

    def _head_bwd(self, tape: dict, dlogits: torch.Tensor) -> torch.Tensor:
        dev = self.device
        W, G = self.towers[("trunk", "param")], self.towers[("trunk", "grad")]
        Tn = dlogits.shape[0]
        hh, hb, K, D = self.tc.head_hidden, self.tc.head_bottleneck, self.tc.head_out_dim, self.D
        dy = _e((Tn, hb), F32, dev)
        dgrad(dlogits, self.head_wn, dy, Tn)
        dWn = torch.zeros((K, hb), dtype=F32, device=dev)
        wgrad(dlogits, tape["y"], dWn, Tn)
        lib.weight_norm_bwd(W.extra["last_v"], W.extra["last_g"], self.head_vnorm, dWn, G.extra["last_v"],
                            G.extra["last_g"], K, hb)
        dh3 = _e((Tn, hb), BF, dev)
        lib.l2norm_bwd(tape["y"], tape["nrm"], dy, dh3, Tn, hb)
        m0, m2, m4 = W.extra["mlp0"], W.extra["mlp2"], W.extra["mlp4"]
        g0, g2, g4 = G.extra["mlp0"], G.extra["mlp2"], G.extra["mlp4"]
        lib.cast_colsum(dh3, None, g4.b, Tn, hb)
        dh2 = _e((Tn, hh), BF, dev)
        dgrad(dh3, m4.w, dh2, Tn)
        wgrad(dh3, tape["h2"], g4.w, Tn)
        dpre2 = _e((Tn, hh), BF, dev)
        lib.gelu_bwd(tape["pre2"], dh2, dpre2, g2.b, Tn, hh)
        dh1 = _e((Tn, hh), BF, dev)
        dgrad(dpre2, m2.w, dh1, Tn)
        wgrad(dpre2, tape["h1"], g2.w, Tn)
        dpre1 = _e((Tn, hh), BF, dev)
        lib.gelu_bwd(tape["pre1"], dh1, dpre1, g0.b, Tn, hh)
        dx = _e((Tn, D), BF, dev)
        dgrad(dpre1, m0.w, dx, Tn)
        wgrad(dpre1, tape["x"], g0.w, Tn)
        return dx

    # -------------------------------------------------------------- objective 2: SSL (vtp.py:365-386,410-484)
    def split_masks(self, mask_indices: torch.Tensor, masks_weight: torch.Tensor, B: int, HW: int) -> Dict[str, torch.Tensor]:
        """Per-image-group mask lists for TrainConfig.ssl_chunk (data dependent, so it synchronises): call it once per
        batch in the input pipeline and pass the result on as batch keys `mask_indices@i` / `masks_weight@i`; the step
        itself then contains no data-dependent shape and can be captured in a CUDA graph."""
        chunk = self.tc.ssl_chunk if 0 < self.tc.ssl_chunk < B else B
        out = {}
        if chunk == B:
            return out
        img = mask_indices // HW
        for i, b0 in enumerate(range(0, B, chunk)):
            b1 = min(B, b0 + chunk)
            bc = b1 - b0
            s0 = (img >= b0) & (img < b1)
            s1 = (img >= B + b0) & (img < B + b1)
            out[f"mask_indices@{i}"] = torch.cat([mask_indices[s0] - b0 * HW, mask_indices[s1] - (B + b0 - bc) * HW])
            out[f"masks_weight@{i}"] = torch.cat([masks_weight[s0], masks_weight[s1]])
        return out

    def ssl_fwd_bwd(self, global_crops, local_crops, mask_indices, masks_weight, weight: float = 1.0, mask_groups=None):
        """global_crops [2B,3,H,W] (view-major), local_crops [n_local*B,3,h,w] (crop-major), mask_indices int64 flat
        indices into [2B*HW] of masked global patches (ascending), masks_weight [n_masked] = 1/(#masked in that image).
        With TrainConfig.ssl_chunk = c the B source images are processed c at a time (all their crops together): the
        teacher targets use last step's centre either way, so chunking only changes floating-point summation order."""
        import torch.distributed as dist
        dev, tc = self.device, self.tc
        K = tc.head_out_dim
        self._head_prepare()
        B2 = global_crops.shape[0]
        B = B2 // 2
        n_m = mask_indices.numel()
        csum = torch.zeros((2, K), dtype=F32, device=dev)   # Σ raw teacher logits: [cls rows, masked-patch rows]
        chunk = tc.ssl_chunk if 0 < tc.ssl_chunk < B else B
        if chunk == B:
            self._ssl_chunk(global_crops, local_crops, mask_indices, masks_weight, weight, B, csum)
        else:
            ps = self.cfg.vision_patch_size
            HW = (global_crops.shape[-2] // ps) * (global_crops.shape[-1] // ps)
            n_loc = tc.n_local_crops
            lc = local_crops.view(n_loc, B, *local_crops.shape[1:])
            if mask_groups is None or "mask_indices@0" not in mask_groups:
                mask_groups = self.split_masks(mask_indices, masks_weight, B, HW)   # synchronises (boolean indexing)
            for i, b0 in enumerate(range(0, B, chunk)):
                b1 = min(B, b0 + chunk)
                bc = b1 - b0
                g = torch.cat([global_crops[b0:b1], global_crops[B + b0:B + b1]])
                l = lc[:, b0:b1].reshape(n_loc * bc, *local_crops.shape[1:])
                self._ssl_chunk(g, l, mask_groups[f"mask_indices@{i}"], mask_groups[f"masks_weight@{i}"], weight, B, csum,
                                final_group=(b1 == B))
        # teacher centre EMA over the whole (global) batch (DINOv2 softmax_center_teacher / update_center)
        cnt = torch.empty(2, dtype=F32, device=dev)          # fill kernels, no host copy: the step is graph-capturable
        cnt[0:1].fill_(float(B2)), cnt[1:2].fill_(float(max(n_m, 1)))
        if self.world > 1:
            dist.all_reduce(csum, group=self.pg)
            dist.all_reduce(cnt, group=self.pg)
        cm = tc.center_momentum
        mean = csum / cnt[:, None]
        lib.axpby(self.center_dino, mean[0].contiguous(), cm, 1 - cm, K)
        lib.axpby(self.center_ibot, mean[1].contiguous(), cm, 1 - cm, K)

    def _ssl_chunk(self, global_crops, local_crops, mask_indices, masks_weight, weight: float, norm_B: int, csum,
                   final_group: bool = True):
        """Teacher + student forward, DINO/iBOT losses and the full backward for one group of source images; the loss
        terms are normalised by `norm_B` (the whole per-GPU batch) and the raw teacher-logit sums are added to csum."""
        dev, tc = self.device, self.tc
        W, G, Wt = self.towers[("trunk", "param")], self.towers[("trunk", "grad")], self.towers[("trunk", "teacher")]
        D, K = self.D, tc.head_out_dim
        n_loc = tc.n_local_crops
        B2 = global_crops.shape[0]
        B = B2 // 2
        n_m = mask_indices.numel()
        # ---------------- teacher (no grad): get_teacher_forward_outputs vtp.py:410-450
        xt, (_, T, gh, gw) = E.trunk_forward(Wt, global_crops, "bf16")
        HW = gh * gw
        xnt = E.norm(xt, B2 * T, D, Wt.norm_w, None, Wt.eps, "bf16", want="f32")
        ar = torch.arange(B2, device=dev, dtype=torch.long)
        cls_rows = ar * T
        swapped = torch.cat([cls_rows[B:], cls_rows[:B]])                       # cat(chunk[1], chunk[0])
        m_rows = (mask_indices // HW) * T + 1 + mask_indices % HW
        Tt = B2 + n_m
        tin = _e((Tt, D), BF, dev)
        lib.gather_rows(xnt, tin, torch.cat([swapped, m_rows]), D)
        tlog = self._head_fwd(Wt, self.head_wn_t, tin, None)
        # centre statistics (sums of raw teacher logits), then centred + sharpened softmax in place
        lib.cast_colsum(tlog, None, csum[0], B2, K)
        if n_m:
            lib.cast_colsum(tlog[B2:], None, csum[1], n_m, K)
        lib.dino_teacher_probs(tlog, self.center_dino, B2, K, tc.teacher_temp)
        if n_m:
            lib.dino_teacher_probs(tlog[B2:], self.center_ibot, n_m, K, tc.teacher_temp)
        del xt, xnt
        # ---------------- student: get_student_ssl_outputs vtp.py:452-484
        tp_g, tp_l = {}, {}
        xg, _ = E.trunk_forward(W, global_crops, "bf16", mask_idx=mask_indices, tape=tp_g,
                                drop=self._drop(tc.ssl_drop_rate))
        xl, (Bl, Tl, _, _) = E.trunk_forward(W, local_crops, "bf16", tape=tp_l, drop=self._drop(tc.ssl_drop_rate))
        xng = E.norm(xg, B2 * T, D, W.norm_w, None, W.eps, "bf16", want="f32", tape=tp_g)
        xnl = E.norm(xl, Bl * Tl, D, W.norm_w, None, W.eps, "bf16", want="f32", tape=tp_l)
        l_rows = torch.arange(Bl, device=dev, dtype=torch.long) * Tl
        Ts = Bl + B2 + n_m
        sin_ = _e((Ts, D), BF, dev)
        lib.gather_rows(xnl, sin_[:Bl], l_rows, D)
        lib.gather_rows(xng, sin_[Bl:], torch.cat([cls_rows, m_rows]), D)
        htape = {}
        slog = self._head_fwd(W, self.head_wn, sin_, htape)
        # ---------------- losses (DINOv2 DINOLoss / iBOTPatchLoss, see oracle.dino_ibot_loss)
        n_terms = 2 + 2 * n_loc
        bidx = torch.arange(B, device=dev, dtype=torch.int32)
        t0 = torch.cat([bidx.repeat(n_loc), torch.arange(B2, device=dev, dtype=torch.int32),
                        B2 + torch.arange(n_m, device=dev, dtype=torch.int32)])
        t1 = torch.cat([(B + bidx).repeat(n_loc), torch.full((B2 + n_m,), -1, device=dev, dtype=torch.int32)])
        wl = weight / (norm_B * n_terms)
        wrow = torch.cat([torch.full((Bl,), wl, device=dev), torch.full((B2,), wl, device=dev),
                          masks_weight.to(F32) * (weight / norm_B)])
        lib.dino_student_ce(slog[:Bl], tlog, t0[:Bl], t1[:Bl], wrow[:Bl], Bl, K, tc.student_temp, self.loss_acc[1:2])
        lib.dino_student_ce(slog[Bl:Bl + B2], tlog, t0[Bl:Bl + B2], t1[Bl:Bl + B2], wrow[Bl:Bl + B2], B2, K,
                            tc.student_temp, self.loss_acc[2:3])
        if n_m:
            lib.dino_student_ce(slog[Bl + B2:], tlog, t0[Bl + B2:], t1[Bl + B2:], wrow[Bl + B2:], n_m, K,
                                tc.student_temp, self.loss_acc[3:4])
        del tlog
        # ---------------- backward: head -> scatter to the two trunk passes
        dsin = self._head_bwd(htape, slog)
        del slog, htape
        if final_group:
            self._reduce_bucket("head")  # DINO head gradient is final: all-reduce under the trunk backward
        dl32 = torch.zeros((Bl * Tl, D), dtype=F32, device=dev)
        lib.scatter_add_rows(dsin[:Bl], dl32, l_rows, D)
        dxl = _e((Bl * Tl, D), BF, dev)
        lib.cast_colsum(dl32, dxl, None, Bl * Tl, D)
        trunk_backward(W, G, tp_l, dxl, dl32.zero_())
        del dl32, dxl, xl, xnl, tp_l
        dg32 = torch.zeros((B2 * T, D), dtype=F32, device=dev)
        lib.scatter_add_rows(dsin[Bl:], dg32, torch.cat([cls_rows, m_rows]), D)
        dxg = _e((B2 * T, D), BF, dev)
        lib.cast_colsum(dg32, dxg, None, B2 * T, D)
        trunk_backward(W, G, tp_g, dxg, dg32.zero_())

    # -------------------------------------------------------------- optimiser (+ EMA teacher, vtp.py:388-401)
    def allreduce_grads(self):
        """Collective C3: whatever bucket has not been started yet (always the trunk), then wait for all of them; the
        sum is averaged by grad_scale = 1/world inside the fused optimiser.  fp32 on the wire (exact accumulation)."""
        if self.world > 1:
            import torch.distributed as dist
            if not self._started:        # "end" mode: nothing in flight — one call over the whole flat buffer
                dist.all_reduce(self.store.g, group=self.pg)
                return
            for which in ("text", "head", "decoder", "trunk"):
                self._reduce_bucket(which, final=True)
            for w in self._pending:
                w.wait()                 # the compute stream waits for NCCL's stream; the host does not block
            self._pending = []

    def set_schedules(self, lr=None, weight_decay=None, teacher_momentum=None):
        """Per-step schedules for the learning rate, weight decay and EMA teacher momentum: `schedules.CosineSchedule`
        objects (the reference's CosineScheduler, text_utils.py:160-207) or plain sequences, indexed by the optimiser
        step (0-based) and held at their last value afterwards.  They live on the device; the optimiser looks them up
        with its own step counter, also inside a captured graph.  None keeps the constant from TrainConfig."""
        from .schedules import as_table, pad_tables
        given = [(i, as_table(s)) for i, s in enumerate((lr, weight_decay, teacher_momentum)) if s is not None]
        tabs = [None, None, None]
        n = 0
        if given:
            padded = pad_tables([t for _, t in given])
            n = int(padded[0].size)
            for (i, _), t in zip(given, padded):
                tabs[i] = torch.from_numpy(t).to(self.device)
        self._sched = (tabs[0], tabs[1], tabs[2], n)
        if self._graph is not None:
            raise RuntimeError("set_schedules() after capture_step(): capture again (table pointers are part of the graph)")

    def scheduled_values(self) -> Dict[str, float]:
        """{step, lr, weight_decay, teacher_momentum} the LAST optimiser step used (synchronises)."""
        h = self.hyper.cpu()
        return {"step": int(h[0]), "lr": float(h[3]), "weight_decay": float(h[4]), "teacher_momentum": float(h[5])}

    def optimizer_step(self):
        st, tc = self.store, self.tc
        self.step_count += 1
        lr_t, wd_t, mom_t, n_t = self._sched
        lib.hyper_tick(self.hyper, tc.beta1, tc.beta2, lr_t, wd_t, mom_t, n_t)
        for start, end, decay, teacher in st.regions:
            n = end - start
            lib.adamw_step(st.p[start:end], st.g[start:end], st.m[start:end], st.v[start:end], st.pb[start:end],
                           st.tp[start:end] if teacher else None, st.tpb[start:end] if teacher else None, n,
                           lr=tc.lr, beta1=tc.beta1, beta2=tc.beta2, eps=tc.eps, wd=tc.weight_decay if decay else 0.0,
                           step=self.step_count, grad_scale=1.0 / self.world, ema_momentum=tc.teacher_momentum,
                           hyper=self.hyper)

    # -------------------------------------------------------------- CUDA graph of the whole step
    def capture_step(self, batch: Dict[str, torch.Tensor], warmup: int = 2):
        """Capture ONE full training step (three objectives, collectives, optimiser + EMA) into a CUDA graph that
        `replay_step` launches with a single call: ~2 300 kernel launches per VTP-Small step cost ~200 ms of host time,
        which is exposed whenever the caller synchronises per step (reading the loss).  The step state that changes from
        step to step (Adam bias corrections, scheduled lr / wd / momentum, teacher centres) lives on the device, so the
        replay needs no host scalar.  `warmup` REAL steps run on `batch` first (they train; lazy initialisation and the
        allocator settle), then one step is captured without executing.  Batches given to `replay_step` must have the
        shapes of `batch` (incl. the number of masked patches)."""
        if self._graph is not None:
            raise RuntimeError("a step graph exists already")
        self._static = {k: v.to(self.device).clone() for k, v in batch.items()}
        B = batch["global_crops"].shape[0] // 2
        if 0 < self.tc.ssl_chunk < B and "mask_indices@0" not in self._static:
            ps = self.cfg.vision_patch_size
            HW = (batch["global_crops"].shape[-2] // ps) * (batch["global_crops"].shape[-1] // ps)
            self._static.update(self.split_masks(self._static["mask_indices"], self._static["masks_weight"], B, HW))
        graph = StepGraph(self.device)
        graph.capture(lambda: self.train_step(self._static), warmup)
        self.step_count -= 1                      # the capture did not execute
        self.graph_launches = graph.launches      # kernels of ours inside one replay
        self._graph = graph
        return self

    def replay_step(self, batch: Optional[Dict[str, torch.Tensor]] = None) -> torch.Tensor:
        """One training step by graph replay.  `batch` (device or pinned-host tensors) is copied into the graph's static
        input buffers first; None re-uses their current contents.  Returns the loss vector like train_step."""
        if self._graph is None:
            raise RuntimeError("capture_step() first")
        if batch is not None and batch is not self._static:
            if any("@" in k for k in self._static) and "mask_indices@0" not in batch:
                gc, ps = self._static["global_crops"], self.cfg.vision_patch_size
                B, HW = gc.shape[0] // 2, (gc.shape[-2] // ps) * (gc.shape[-1] // ps)
                batch = dict(batch)
                batch.update(self.split_masks(batch["mask_indices"].to(self.device), batch["masks_weight"].to(self.device), B, HW))
            for k, v in self._static.items():
                if batch[k].shape != v.shape:
                    raise ValueError(f"replay_step: '{k}' has shape {tuple(batch[k].shape)}, the graph was captured for {tuple(v.shape)}")
                v.copy_(batch[k], non_blocking=True)
        self._graph.replay()
        self.step_count += 1
        return self.loss_acc

    def release_graph(self):
        """Destroy the captured step graph and its static inputs.  REQUIRED before `dist.destroy_process_group()` in a
        multi-rank job: NCCL does not tear a communicator down while a CUDA graph that captured its collectives is alive
        (the 2-GPU run of round 2 hung in destroy_process_group until the graph was released first)."""
        if self._graph is not None:
            self._graph.release()
            self._graph = None
            self._static = None
            import gc
            gc.collect()
            torch.cuda.synchronize(self.device)

    @property
    def static_batch(self) -> Dict[str, torch.Tensor]:
        """The graph's input buffers (fill them directly — e.g. H2D copies on a side stream — and call replay_step())."""
        return self._static

    def check_exchange(self):
        """Raise if the peer-memory contrastive exchange reported a barrier time-out (synchronises)."""
        if self.peer is not None:
            self.peer.check()

    def train_step(self, batch: Dict[str, torch.Tensor]) -> torch.Tensor:
        """One full 3-objective step. Returns the device tensor of accumulated loss terms
        [clip, dino_local, dino_global, ibot, rec_l1, lpips, -, -] (read it with .cpu() to synchronise).  A NaN in slot 0
        with clip_exchange == "p2p" means the peer-memory barrier timed out (a rank never arrived): the step's update
        is invalid — `check_exchange()` raises in that case."""
        tc = self.tc
        self.loss_acc.zero_()
        self._started = set()
        if tc.w_clip:
            self.clip_fwd_bwd(batch["image"], batch["text"], tc.w_clip)
        self._reduce_bucket("text")      # text tower, clip projection, logit scale: final — reduce under the SSL objective
        if tc.w_ssl:
            self.ssl_fwd_bwd(batch["global_crops"], batch["local_crops"], batch["mask_indices"], batch["masks_weight"],
                             tc.w_ssl, mask_groups=batch)
        if tc.w_rec:
            img = batch["rec_image"]
            nB = img.shape[0]
            rc = tc.rec_chunk if 0 < tc.rec_chunk < nB else nB
            for b0 in range(0, nB, rc):
                self.rec_fwd_bwd(img[b0:b0 + rc], tc.w_rec, norm_B=nB, final_group=(b0 + rc >= nB))
        self.allreduce_grads()
        self.optimizer_step()
        return self.loss_acc
