"""Linear probing of a VTP trunk on the device (tools/test_linear_probing_hf.py of the reference).

A grid of fp32 linear classifiers, one per (n last blocks, learning rate), is trained on frozen trunk features with
SGD-momentum and a cosine schedule, then scored by top-1 accuracy.  One training step is the trunk forward, the feature
assembly read in place from the residual stream after each of the last max(n) blocks (`vtp_probe_features`), one
bf16x3 GEMM per n-group with every classifier of the group side by side along N, the per-classifier cross-entropy with
its gradient operand (`vtp_probe_ce`), one dW GEMM per group and the fused SGD update that also refreshes the next
forward's weight operand (`vtp_probe_sgd`).  The step reads no host scalar, so after one eager step it is captured
into a CUDA graph and replayed; nothing in it synchronises the host.

Layout: classifier i of a group with K = (n+1)·D inputs keeps its C classes in Cp = ceil8(C) rows (padding rows stay 0);
the flat fp32 buffers p / g / momentum hold every group's [G_n·Cp, K] weights, then all biases [G·Cp].
The features X [B, (max(n)+1)·D] are cls_{L-max(n)+1} | … | cls_L | mean of the patch rows of block L; group n reads
columns [(max(n)-n)·D, (max(n)+1)·D) (create_linear_input, linear_probing_hf.py:137-152).

    python -m vtp_b200.probe --model_path DIR --imagenet_root ROOT [--batch_size 128 --epochs 10 --epoch_length 1250]
    torchrun --nproc_per_node=8 -m vtp_b200.probe ... --use_ddp
"""
from __future__ import annotations

import argparse
import json
import os
from dataclasses import dataclass
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import engine as E
from . import lib
from .graphs import StepGraph

F32, BF = torch.float32, torch.bfloat16

IMAGENET_DEFAULT_MEAN = (0.485, 0.456, 0.406)
IMAGENET_DEFAULT_STD = (0.229, 0.224, 0.225)
CROP_SIZE, RESIZE_SIZE = 224, 256
DEFAULT_LEARNING_RATES = (1e-5, 2e-5, 5e-5, 1e-4, 2e-4, 5e-4, 1e-3, 2e-3, 5e-3, 1e-2, 2e-2, 5e-2, 0.1)
MOMENTUM = 0.9


def scale_lr(lr: float, batch_size: int, world: int = 1) -> float:
    """linear_probing_hf.py:216-218."""
    return lr * (batch_size * world) / 256.0


def classifier_key(n: int, lr: float) -> str:
    """linear_probing_hf.py:242 (lr already scaled)."""
    return f"classifier_{n}_blocks_avgpool_True_lr_{lr:.5f}".replace(".", "_")


@dataclass
class Classifier:
    key: str
    n: int
    lr: float        # scaled learning rate of the param group that trains it
    created: int     # creation index (its initial weights are the created-th draw)


def plan_classifiers(n_last_blocks_list: Sequence[int], learning_rates: Sequence[float], batch_size: int,
                     world: int = 1) -> Tuple[List[Classifier], int]:
    """The classifiers that train, in the reference's ModuleDict order, and how many were created.

    linear_probing_hf.py:233-246 stores classifier (n, lr) under a key that formats the scaled lr to 5 decimals, so two
    lrs can share a key (at world 1 and batch 128: 5e-6 and 1e-5 -> `0_00001`).  The ModuleDict then keeps the later
    classifier at the earlier key's position, and the earlier one — still in the optimiser, never given a gradient —
    does not train.  This is reproduced: 24 classifiers at world 1 / batch 128, 26 at world 8."""
    order: List[Classifier] = []
    slot: Dict[str, int] = {}
    created = 0
    for n in n_last_blocks_list:
        for base in learning_rates:
            lr = scale_lr(base, batch_size, world)
            c = Classifier(classifier_key(n, lr), int(n), lr, created)
            created += 1
            if c.key in slot:
                order[slot[c.key]] = c
            else:
                slot[c.key] = len(order)
                order.append(c)
    return order, created


def lr_table(lrs: Sequence[float], max_iter: int) -> np.ndarray:
    """fp32 [max_iter, len(lrs)]: row t = the lr of every param group at optimiser step t, recorded from torch's own
    SGD + CosineAnnealingLR(T_max=max_iter, eta_min=0) as linear_probing_hf.py:486-488,291 steps them."""
    params = [torch.nn.Parameter(torch.zeros(1)) for _ in lrs]
    opt = torch.optim.SGD([{"params": [p], "lr": lr} for p, lr in zip(params, lrs)], momentum=MOMENTUM, weight_decay=0)
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, max_iter, eta_min=0)
    rows = np.empty((max_iter, len(lrs)), dtype=np.float64)
    for t in range(max_iter):
        rows[t] = [g["lr"] for g in opt.param_groups]
        opt.step()      # no gradients: a no-op that keeps the scheduler's step-order check satisfied
        sched.step()
    return rows.astype(np.float32)


def initial_weights(n_last_blocks_list: Sequence[int], learning_rates: Sequence[float], in_dim: Dict[int, int],
                    num_classes: int, seed: int) -> List[Tuple[torch.Tensor, torch.Tensor]]:
    """(weight, bias) of every created classifier, drawn like linear_probing_hf.py:158-166 after torch.manual_seed(seed):
    nn.Linear's own initialisation (which consumes the CPU generator), then weight ~ N(0, 0.01) and bias = 0.  The global
    generator state is restored afterwards."""
    out = []
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)
        for n in n_last_blocks_list:
            for _ in learning_rates:
                lin = torch.nn.Linear(in_dim[n], num_classes)
                lin.weight.data.normal_(mean=0.0, std=0.01)
                lin.bias.data.zero_()
                out.append((lin.weight.data, lin.bias.data))
    return out


@dataclass
class _Group:
    n: int
    g0: int      # first classifier
    G: int       # classifiers in the group
    K: int       # (n+1)·D
    xcol: int    # first column of X it reads
    woff: int    # offset of its weights in the flat buffers


class LinearProbe:
    """The reference's linear-probe grid on the device.

    model: a VTPModel on the GPU (frozen).  precision "bf16" runs the trunk like the reference under bf16 autocast,
    "fp32" like it in fp32; the classifiers are fp32-accurate either way (bf16x3 GEMMs).  world > 1 (default: the
    torch.distributed world size) averages the gradient over ranks with one all-reduce per step, as DDP does."""

    def __init__(self, model, num_classes: int, n_last_blocks_list: Sequence[int] = (1, 4),
                 learning_rates: Sequence[float] = DEFAULT_LEARNING_RATES, batch_size: int = 128, max_iter: int = 12500,
                 world: Optional[int] = None, seed: int = 0, precision: str = "bf16", use_graph: bool = True,
                 process_group=None):
        import torch.distributed as dist

        if precision not in ("bf16", "fp32"):
            raise NotImplementedError(f"precision {precision!r}: the probe runs the trunk in 'bf16' or 'fp32' (no fp16 path)")
        self.dist = dist.is_available() and dist.is_initialized()
        self.world = int(world) if world is not None else (dist.get_world_size(process_group) if self.dist else 1)
        self.pg = process_group
        self.model, self.mode, self.use_graph = model, precision, use_graph
        cfg = model.config
        self.D, depth = cfg.vision_embed_dim, cfg.vision_depth
        ns = tuple(int(n) for n in n_last_blocks_list)
        if len(set(ns)) != len(ns) or not all(1 <= n <= depth for n in ns):
            raise ValueError(f"n_last_blocks_list {ns}: distinct block counts in [1, {depth}] expected")
        self.nmax = max(ns)
        self.KX = (self.nmax + 1) * self.D
        self.C, self.Cp = int(num_classes), (int(num_classes) + 7) // 8 * 8
        self.B, self.max_iter = int(batch_size), int(max_iter)
        self.classifiers, n_created = plan_classifiers(ns, learning_rates, batch_size, self.world)
        self.keys = [c.key for c in self.classifiers]
        G, Cp, D = len(self.classifiers), self.Cp, self.D
        self.G = G
        self.groups: List[_Group] = []
        off = 0
        for n in ns:
            idx = [i for i, c in enumerate(self.classifiers) if c.n == n]
            K = (n + 1) * D
            self.groups.append(_Group(n, idx[0], len(idx), K, (self.nmax - n) * D, off))
            off += len(idx) * Cp * K
        self.bias_off = off
        dev = model.trunk.cls_token.device
        if dev.type != "cuda":
            raise lib.VtpError("LinearProbe needs the model on the CUDA device (there is no CPU path)")
        self.device = dev
        total = off + G * Cp
        p = torch.zeros(total, dtype=F32)
        init = initial_weights(ns, learning_rates, {n: (n + 1) * D for n in ns}, self.C, seed)
        for grp in self.groups:
            for j in range(grp.G):
                w, b = init[self.classifiers[grp.g0 + j].created]
                p[grp.woff:grp.woff + grp.G * Cp * grp.K].view(grp.G, Cp, grp.K)[j, :self.C] = w
                p[self.bias_off:].view(G, Cp)[grp.g0 + j, :self.C] = b
        self.p = p.to(dev)
        self.g = torch.zeros_like(self.p)
        self.buf = torch.zeros_like(self.p)
        self.wb = []
        for grp in self.groups:
            wb = torch.empty((grp.G * Cp, 3 * grp.K), dtype=BF, device=dev)
            lib.split3(self.weight(grp), wb, grp.G * Cp, grp.K, b_side=True)
            self.wb.append(wb)
        self.lr_tab = torch.from_numpy(lr_table([c.lr for c in self.classifiers], self.max_iter)).to(dev)
        self.hyper = torch.zeros(8, dtype=F32, device=dev)      # [0] = optimiser steps taken (vtp_hyper_tick)
        self.loss_acc = torch.zeros(G, dtype=F32, device=dev)
        self.step_count = 0
        self._graph = StepGraph(dev, enabled=use_graph)
        self._static: Optional[Tuple[torch.Tensor, torch.Tensor]] = None

    # ------------------------------------------------------------------ buffers
    def weight(self, grp: _Group, buf: Optional[torch.Tensor] = None) -> torch.Tensor:
        t = self.p if buf is None else buf
        return t[grp.woff:grp.woff + grp.G * self.Cp * grp.K].view(grp.G * self.Cp, grp.K)

    def bias(self, buf: Optional[torch.Tensor] = None) -> torch.Tensor:
        return (self.p if buf is None else buf)[self.bias_off:]

    # ------------------------------------------------------------------ device stages
    def features(self, images: torch.Tensor) -> torch.Tensor:
        """X fp32 [B, (max(n)+1)·D] of a batch of normalised images (the trunk runs in self.mode)."""
        m = self.model
        m._check_image(images)
        W = m._pack("trunk", self.mode)
        B = images.shape[0]
        ps = m.config.vision_patch_size
        T = (images.shape[-2] // ps) * (images.shape[-1] // ps) + 1
        X = torch.empty((B, self.KX), dtype=F32, device=images.device)
        first, D = len(W.blocks) - self.nmax, self.D

        def tap(li: int, x: torch.Tensor) -> None:
            j = li - first
            if j >= 0:
                lib.probe_features(x, B, T, D, W.norm_w, W.norm_b, W.eps, X, cls_col=j * D,
                                   mean_col=self.nmax * D if j == self.nmax - 1 else -1)

        E.trunk_forward(W, images, self.mode, hook=tap)
        return X

    def logits(self, X: torch.Tensor) -> torch.Tensor:
        """Z fp32 [B, G·Cp]: every classifier's logits (classifier i in columns [i·Cp, i·Cp + C))."""
        B = X.shape[0]
        Z = torch.empty((B, self.G * self.Cp), dtype=F32, device=X.device)
        for grp, wb in zip(self.groups, self.wb):
            A = torch.empty((B, 3 * grp.K), dtype=BF, device=X.device)
            lib.split3(X[:, grp.xcol:], A, B, grp.K, b_side=False, ldx=self.KX)
            c0 = grp.g0 * self.Cp
            lib.gemm(A, wb, Z[:, c0:], M=B, N=grp.G * self.Cp, K=3 * grp.K, lda=3 * grp.K, ldb=3 * grp.K,
                     ldo=self.G * self.Cp, bias=self.bias()[c0:c0 + grp.G * self.Cp], round_bf16=False)
        return Z

    def classifier_step(self, X: torch.Tensor, labels: torch.Tensor) -> None:
        """Forward, loss, backward and SGD update of every classifier on features X [B, KX] and int64 labels [B]."""
        B, G, Cp = X.shape[0], self.G, self.Cp
        if X.dtype != F32 or X.dim() != 2 or X.shape[1] != self.KX or not X.is_contiguous() or X.device != self.device:
            raise ValueError(f"classifier_step: X must be contiguous fp32 [B, {self.KX}] on {self.device}, "
                             f"got {X.dtype} {tuple(X.shape)} on {X.device}")
        if labels.dtype != torch.int64 or labels.shape != (B,) or not labels.is_contiguous() or labels.device != self.device:
            raise ValueError(f"classifier_step: labels must be contiguous int64 [{B}] on {self.device}, "
                             f"got {labels.dtype} {tuple(labels.shape)} on {labels.device}")
        lib.hyper_tick(self.hyper, 0.0, 0.0)
        Z = self.logits(X)
        dZ3 = torch.empty((3 * B, G * Cp), dtype=BF, device=X.device)
        lib.probe_ce(Z, B, G, self.C, Cp, labels, self.loss_acc, dZ3, self.bias(self.g))
        X3 = torch.empty((3 * B, self.KX), dtype=BF, device=X.device)     # rows [X_hi; X_lo; X_hi]
        lib.split3(X, X3, 1, B * self.KX, b_side=True)
        for grp in self.groups:
            c0 = grp.g0 * Cp
            lib.gemm(dZ3[:, c0:], X3[:, grp.xcol:], self.weight(grp, self.g), M=grp.G * Cp, N=grp.K, K=3 * B,
                     lda=G * Cp, ldb=self.KX, ldo=grp.K, a_mn=True, b_mn=True, round_bf16=False)
        if self.world > 1:
            import torch.distributed as dist
            dist.all_reduce(self.g, group=self.pg)
        self.sgd()

    def sgd(self) -> None:
        """The SGD-momentum update of every parameter from self.g at the step hyper[0] (already advanced)."""
        gs = 1.0 / self.world
        for grp, wb in zip(self.groups, self.wb):
            lib.probe_sgd(self.weight(grp), self.weight(grp, self.g), self.weight(grp, self.buf), grp.G * self.Cp * grp.K,
                          row_len=grp.K, rows_per_cls=self.Cp, cls0=grp.g0, lr_table=self.lr_tab, hyper=self.hyper,
                          momentum=MOMENTUM, grad_scale=gs, pb=wb)
        lib.probe_sgd(self.bias(), self.bias(self.g), self.bias(self.buf), self.G * self.Cp, row_len=1,
                      rows_per_cls=self.Cp, cls0=0, lr_table=self.lr_tab, hyper=self.hyper, momentum=MOMENTUM,
                      grad_scale=gs)

    # ------------------------------------------------------------------ public API
    def train_step(self, images: torch.Tensor, labels: torch.Tensor) -> None:
        """One optimiser step on a batch (device or pinned host tensors of the constructor's batch size).  Does not
        synchronise; the first step runs eagerly, later ones replay a CUDA graph of the whole step (same kernels, same
        results)."""
        if self.step_count >= self.max_iter:
            raise RuntimeError(f"max_iter = {self.max_iter} optimiser steps taken (the cosine schedule ends there)")
        if images.shape[0] != self.B or labels.shape != (self.B,):
            raise ValueError(f"train_step: batch of {images.shape[0]} images / labels {tuple(labels.shape)}, "
                             f"the probe was built for batch_size {self.B}")
        if self._static is None:
            self._static = (torch.empty(images.shape, dtype=F32, device=self.device),
                            torch.empty((self.B,), dtype=torch.int64, device=self.device))
        img, lab = self._static
        if tuple(images.shape) != tuple(img.shape):
            raise ValueError(f"train_step: images {tuple(images.shape)}, earlier steps used {tuple(img.shape)}")
        img.copy_(images, non_blocking=True)
        lab.copy_(labels, non_blocking=True)
        self._graph(lambda: self.classifier_step(self.features(img), lab))
        self.step_count += 1

    def take_losses(self) -> torch.Tensor:
        """Per-classifier sum of the batch-mean losses since the last call (a device tensor [G], then zeroed)."""
        out = self.loss_acc.clone()
        self.loss_acc.zero_()
        return out

    def evaluate(self, batches: Iterable[Tuple[torch.Tensor, torch.Tensor]]) -> Dict[str, float]:
        """{key: top-1 accuracy in %} over (images, labels) batches of any size (linear_probing_hf.py:302-345); counts
        and the total are summed over ranks."""
        counts = torch.zeros(self.G, dtype=torch.int64, device=self.device)
        total = 0
        for images, labels in batches:
            images = images.to(self.device, non_blocking=True)
            labels = labels.to(self.device, torch.int64, non_blocking=True).contiguous()
            Z = self.logits(self.features(images))
            lib.probe_correct(Z, images.shape[0], self.G, self.C, self.Cp, labels, counts)
            total += images.shape[0]
        if self.world > 1:
            import torch.distributed as dist
            tot = torch.tensor([total], dtype=torch.int64, device=self.device)
            dist.all_reduce(counts, group=self.pg)
            dist.all_reduce(tot, group=self.pg)
            total = int(tot.item())
        return {k: 100.0 * int(c) / total for k, c in zip(self.keys, counts.cpu().tolist())}

    def state_dict(self) -> Dict[str, torch.Tensor]:
        """The classifiers under the reference's AllClassifiers keys (classifiers_dict.<key>.linear.weight / .bias), CPU."""
        sd = {}
        bias = self.bias().view(self.G, self.Cp).cpu()
        for grp in self.groups:
            w = self.weight(grp).view(grp.G, self.Cp, grp.K).cpu()
            for j in range(grp.G):
                key = self.keys[grp.g0 + j]
                sd[f"classifiers_dict.{key}.linear.weight"] = w[j, :self.C].clone()
                sd[f"classifiers_dict.{key}.linear.bias"] = bias[grp.g0 + j, :self.C].clone()
        return sd

    def release(self) -> None:
        """Drop the captured step graph (required before torch.distributed.destroy_process_group())."""
        self._graph.release()


# ---------------------------------------------------------------------------------------------------------- CLI
def build_parser() -> argparse.ArgumentParser:
    """The reference's flags (linear_probing_hf.py:558-583) plus --seed for the classifier initialisation."""
    ap = argparse.ArgumentParser(description="Linear probing evaluation of a VTP checkpoint on the H100 path")
    ap.add_argument("--model_path", type=str, required=True, help="VTP checkpoint directory (config.json + safetensors)")
    ap.add_argument("--imagenet_root", type=str, required=True, help="dataset root with train/ and val/ ImageFolders")
    ap.add_argument("--output_dir", type=str, default="./linear_probing_results")
    ap.add_argument("--batch_size", type=int, default=128, help="batch size per GPU")
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--epoch_length", type=int, default=1250, help="optimiser steps per epoch")
    ap.add_argument("--num_workers", type=int, default=8)
    ap.add_argument("--device", type=str, default="cuda:0", help="device (ignored with --use_ddp)")
    ap.add_argument("--precision", type=str, default="bf16", choices=["fp32", "fp16", "bf16"])
    ap.add_argument("--use_ddp", action="store_true", help="data parallel over the ranks started by torchrun")
    ap.add_argument("--local_rank", type=int, default=None)
    ap.add_argument("--seed", type=int, default=0, help="torch.manual_seed before the classifiers are created")
    return ap


def make_transforms(crop: int = CROP_SIZE, resize: int = RESIZE_SIZE):
    """(train, eval) torchvision pipelines of linear_probing_hf.py:87-102."""
    from torchvision import transforms as Tv

    norm = Tv.Normalize(mean=IMAGENET_DEFAULT_MEAN, std=IMAGENET_DEFAULT_STD)
    bic = Tv.InterpolationMode.BICUBIC
    train = Tv.Compose([Tv.RandomResizedCrop(crop, interpolation=bic), Tv.RandomHorizontalFlip(), Tv.ToTensor(), norm])
    val = Tv.Compose([Tv.Resize(resize, interpolation=bic), Tv.CenterCrop(crop), Tv.ToTensor(), norm])
    return train, val


class _Forever(torch.utils.data.Sampler):
    """Endless index stream over a sampler, advancing its epoch (set_epoch) at every pass."""

    def __init__(self, sampler):
        self.sampler = sampler

    def __iter__(self):
        epoch = 0
        while True:
            if hasattr(self.sampler, "set_epoch"):
                self.sampler.set_epoch(epoch)
            yield from iter(self.sampler)
            epoch += 1

    def __len__(self):
        return 1 << 62


def run(args) -> Dict[str, object]:
    import torch.distributed as dist
    from torch.utils.data import DataLoader, DistributedSampler, RandomSampler
    from torchvision.datasets import ImageFolder

    from .model import VTPModel

    if args.precision == "fp16":
        raise NotImplementedError("--precision fp16: the trunk runs in bf16 or fp32 only")
    if args.use_ddp:
        if not dist.is_initialized():
            dist.init_process_group(backend="nccl")
        local = args.local_rank if args.local_rank is not None else int(os.environ.get("LOCAL_RANK", 0))
        torch.cuda.set_device(local % torch.cuda.device_count())
        device = torch.device("cuda", local % torch.cuda.device_count())
    else:
        device = torch.device(args.device)
    main = not dist.is_initialized() or dist.get_rank() == 0
    os.makedirs(args.output_dir, exist_ok=True)
    model = VTPModel.from_pretrained(args.model_path).to(device).eval()
    train_tf, val_tf = make_transforms()
    train_ds = ImageFolder(os.path.join(args.imagenet_root, "train"), transform=train_tf)
    val_ds = ImageFolder(os.path.join(args.imagenet_root, "val"), transform=val_tf)
    if args.use_ddp:
        train_s, val_s = DistributedSampler(train_ds, shuffle=True), DistributedSampler(val_ds, shuffle=False)
    else:
        train_s, val_s = RandomSampler(train_ds), None
    train_dl = DataLoader(train_ds, batch_size=args.batch_size, sampler=_Forever(train_s), num_workers=args.num_workers,
                          pin_memory=True, drop_last=True)
    val_dl = DataLoader(val_ds, batch_size=2 * args.batch_size, sampler=val_s, shuffle=False,
                        num_workers=args.num_workers, pin_memory=True)
    probe = LinearProbe(model, len(train_ds.classes), batch_size=args.batch_size,
                        max_iter=args.epochs * args.epoch_length, seed=args.seed, precision=args.precision)
    best, best_key, acc = 0.0, "", {}
    it = iter(train_dl)
    for epoch in range(args.epochs):
        for _ in range(args.epoch_length):
            images, labels = next(it)
            probe.train_step(images.to(device, non_blocking=True), labels.to(device, non_blocking=True))
        loss = float(probe.take_losses().sum()) / max(args.epoch_length, 1)
        acc = probe.evaluate(val_dl)
        cur_key = max(acc, key=acc.get)
        if acc[cur_key] > best:
            best, best_key = acc[cur_key], cur_key
        if main:
            print(f"epoch {epoch}: train loss {loss:.4f}, best accuracy {acc[cur_key]:.2f}% ({cur_key})", flush=True)
    results = {"best_accuracy": best, "best_classifier": best_key, "all_accuracies": acc}
    if main:
        path = os.path.join(args.output_dir, "linear_probing_results.json")
        with open(path, "w") as f:
            json.dump(results, f, indent=2)
        print(f"results: {path}")
    probe.release()
    if args.use_ddp:
        dist.destroy_process_group()
    return results


def main(argv=None):
    return run(build_parser().parse_args(argv))


if __name__ == "__main__":
    main()
