"""Zero-shot classification on the device (tools/test_zero_shot_hf.py of the reference).

The classifier is the reference's prompt ensemble: every class name is put into every template, each prompt goes through
the CLIP text tower, the per-prompt features are L2-normalised, averaged over the templates and normalised again.  The
text tower is causal and pools at the end-of-text token (`text_pool_type='argmax'`), so a prompt's feature depends only
on its tokens 0..EOT: prompts are sorted by length into buckets and each bucket runs at L = min(ceil8(max EOT + 1),
context_length) instead of the full 77 tokens (bit-identical features, a fraction of the work).  `vtp_zs_class_embed`
turns the length-sorted features into the fp32 classifier in place.

Evaluation (`ZeroShotEvaluator`) runs per batch: the image tower's unnormalised CLIP feature, `vtp_zs_image_operand`
(a = 100 · x / max(‖x‖, eps) in fp32, as the reference's F.normalize under CUDA autocast), the logits GEMM (bf16x3 with
fp32 out in fp32 mode; bf16 operands and bf16 out in bf16 mode, autocast's matmul) and `vtp_zs_rank`, which writes each
target's rank and adds the top-k hits to int64 device counters.  From the second batch of a shape on, the whole batch
is one CUDA graph replay; the host reads the counters once, in `result()`.

    python -m vtp_b200.zero_shot --model_path DIR --data_path VAL_DIR [--precision bf16] [--prompts prompts.json]
"""
from __future__ import annotations

import argparse
import ast
import json
import os
from concurrent.futures import ThreadPoolExecutor
from typing import Callable, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import engine as E
from . import lib
from .graphs import StepGraph

F32, BF = torch.float32, torch.bfloat16
IMAGENET_DEFAULT_MEAN = (0.485, 0.456, 0.406)
IMAGENET_DEFAULT_STD = (0.229, 0.224, 0.225)
REFERENCE_SCRIPT = "test_zero_shot_hf.py"


def _mode(precision: str) -> str:
    if precision in ("bf16", "bfloat16"):
        return "bf16"
    if precision in ("fp32", "float32"):
        return "fp32"
    raise NotImplementedError(f"precision {precision!r}: zero-shot runs in 'bf16' or 'fp32' (no fp16 path)")


def _ceil8(n: int) -> int:
    return (n + 7) // 8 * 8


# ---------------------------------------------------------------------------------------------------------- prompts
def template_fn(t: Union[str, Callable[[str], str]]) -> Callable[[str], str]:
    """A template as the reference's callables, or a str.format string with {c} for the class name."""
    if callable(t):
        return t
    return lambda c, _t=t: _t.format(c=c)


def _joined_to_format(node: ast.AST) -> str:
    """`lambda c: f'a photo of a {c}.'` -> 'a photo of a {c}.' (literal braces doubled)."""
    if not isinstance(node, ast.Lambda) or not isinstance(node.body, ast.JoinedStr):
        raise ValueError(f"template is not a lambda returning an f-string: {ast.dump(node)[:80]}")
    arg = node.args.args[0].arg
    out = []
    for v in node.body.values:
        if isinstance(v, ast.Constant):
            out.append(str(v.value).replace("{", "{{").replace("}", "}}"))
        elif isinstance(v, ast.FormattedValue) and isinstance(v.value, ast.Name) and v.value.id == arg \
                and v.conversion == -1 and v.format_spec is None:
            out.append("{c}")
        else:
            raise ValueError("template f-string uses something other than the class name")
    return "".join(out)


def read_reference_prompts(path: str) -> Tuple[List[str], List[str]]:
    """IMAGENET_CLASSNAMES and OPENAI_IMAGENET_TEMPLATES (as format strings) parsed out of the reference's
    tools/test_zero_shot_hf.py with `ast`; the file is not executed."""
    with open(path, encoding="utf-8") as f:
        tree = ast.parse(f.read(), filename=path)
    found: Dict[str, ast.AST] = {}
    for node in tree.body:
        if isinstance(node, ast.Assign) and len(node.targets) == 1 and isinstance(node.targets[0], ast.Name):
            found[node.targets[0].id] = node.value
    if "IMAGENET_CLASSNAMES" not in found or "OPENAI_IMAGENET_TEMPLATES" not in found:
        raise ValueError(f"{path} does not define IMAGENET_CLASSNAMES and OPENAI_IMAGENET_TEMPLATES")
    classnames = list(ast.literal_eval(found["IMAGENET_CLASSNAMES"]))
    tmpl = found["OPENAI_IMAGENET_TEMPLATES"]
    if not isinstance(tmpl, (ast.Tuple, ast.List)):
        raise ValueError("OPENAI_IMAGENET_TEMPLATES is not a tuple or list literal")
    return classnames, [_joined_to_format(e) for e in tmpl.elts]


def find_reference_script(bpe_path: Optional[str] = None) -> Optional[str]:
    """The reference's tools/test_zero_shot_hf.py, looked for where `find_bpe_file` looks for the vocabulary: next to an
    explicit vocabulary file or $VTP_BPE_PATH, in a reference checkout on sys.path, then the working directory."""
    dirs: List[str] = []
    for p in (bpe_path, os.environ.get("VTP_BPE_PATH")):
        if p:
            dirs.append(os.path.dirname(os.path.abspath(p)))
    try:
        import importlib.util

        spec = importlib.util.find_spec("vtp.tokenizers")
        for loc in (spec.submodule_search_locations if spec and spec.submodule_search_locations else []):
            root = os.path.dirname(os.path.dirname(loc))
            dirs += [os.path.join(root, "tools"), root]
    except (ImportError, ValueError, AttributeError):
        pass
    dirs += [os.path.join(os.getcwd(), "tools"), os.getcwd()]
    for d in dirs:
        c = os.path.join(d, REFERENCE_SCRIPT)
        if os.path.exists(c):
            return os.path.abspath(c)
    return None


def load_prompts(prompts: Optional[str] = None, bpe_path: Optional[str] = None) -> Tuple[List[str], List[str]]:
    """(classnames, templates): from a JSON file {"classnames": [...], "templates": ["... {c} ...", ...]}, or else from
    the reference's script (read, not run)."""
    if prompts:
        with open(prompts, encoding="utf-8") as f:
            d = json.load(f)
        return list(d["classnames"]), list(d["templates"])
    script = find_reference_script(bpe_path)
    if script is None:
        raise FileNotFoundError(
            "no class names / templates: pass --prompts FILE (JSON with 'classnames' and 'templates' using {c}), or put "
            f"the reference's tools/{REFERENCE_SCRIPT} where the BPE vocabulary is looked for (next to --bpe_path or "
            "$VTP_BPE_PATH, a reference checkout on sys.path, or ./tools)")
    return read_reference_prompts(script)


# ---------------------------------------------------------------------------------------------------------- text side
def eot_positions(ids: torch.Tensor) -> np.ndarray:
    """The position the text tower pools at: the argmax of each row's ids (the end-of-text token)."""
    return ids.argmax(dim=-1).numpy()


def bucket_plan(eot: np.ndarray, context_length: int, max_rows: int = 4096) -> List[Tuple[np.ndarray, int]]:
    """Prompts grouped by L = min(ceil8(eot + 1), context_length), each group cut into buckets of at most max_rows.
    Returns [(prompt indices, L)] in ascending L; every prompt appears exactly once."""
    eot = np.asarray(eot, dtype=np.int64)
    Ls = np.minimum((eot + 8) // 8 * 8, context_length)
    order = np.argsort(Ls, kind="stable")
    plan = []
    for L in np.unique(Ls):
        idx = order[Ls[order] == L]
        for s in range(0, len(idx), max_rows):
            plan.append((idx[s:s + max_rows], int(L)))
    return plan


def encode_prompts(model, ids: torch.Tensor, precision: str, *, out: Optional[torch.Tensor] = None, row0: int = 0,
                   max_rows: int = 4096) -> Tuple[torch.Tensor, np.ndarray]:
    """Unnormalised text features of the prompts `ids` (int64 [N, context_length], host), each encoded only up to its
    end token.  The features land length-sorted in out[row0 : row0 + N] (allocated when out is None); returns
    (out, row_of) with prompt i at row row_of[i].  Launches are eager (this runs once per classifier)."""
    mode = _mode(precision)
    if not model.config.train_clip:
        raise RuntimeError("CLIP not enabled. Set train_clip=True in config.")
    ctx, vocab = model.config.text_context_length, model.config.text_vocab_size
    if ids.dtype != torch.int64 or ids.dim() != 2 or ids.shape[1] != ctx:
        raise ValueError(f"expected int64 token ids of shape (N, {ctx}), got {ids.dtype} {tuple(ids.shape)}")
    if ids.numel() and (int(ids.max()) >= vocab or int(ids.min()) < 0):
        raise ValueError(f"token ids outside the text tower's vocabulary [0, {vocab})")
    ids = ids.cpu()
    dev = model.trunk.cls_token.device
    W = model._pack("text", mode)
    N = ids.shape[0]
    if out is None:
        out = torch.empty((row0 + N, W.extra["proj"].N), dtype=BF if mode == "bf16" else F32, device=dev)
    row_of = np.empty(N, dtype=np.int32)
    r = row0
    with torch.no_grad():
        for idx, L in bucket_plan(eot_positions(ids), ctx, max_rows):
            f = E.text_forward(W, ids[torch.from_numpy(idx), :L].contiguous().to(dev), mode)
            out[r:r + len(idx)].copy_(f)
            row_of[idx] = np.arange(r, r + len(idx), dtype=np.int32)
            r += len(idx)
    return out, row_of


def build_zero_shot_classifier(model, tokenizer, classnames: Sequence[str], templates: Sequence, num_classes_per_batch: int = 10,
                               device=None, use_tqdm: bool = True, *, precision: str = "fp32",
                               chunk_prompts: int = 8192, max_rows: int = 4096) -> torch.Tensor:
    """test_zero_shot_hf.py:342-394: the fp32 classifier [E, C] (column c = class c's normalised template mean).

    templates: callables or str.format strings with {c}.  tokenizer: any list[str] -> int64 [N, L] callable.
    num_classes_per_batch and device are accepted for the reference's signature and change nothing (every step is
    row-independent; prompts are batched by length and the model's device is used).  Tokenization of the next chunk
    of chunk_prompts prompts runs on a worker thread while the current chunk is encoded."""
    mode = _mode(precision)
    fns = [template_fn(t) for t in templates]
    C, T = len(classnames), len(fns)
    if C == 0 or T == 0:
        raise ValueError("need at least one class name and one template")
    dev = model.trunk.cls_token.device
    per = max(1, chunk_prompts // T)
    chunks = [(c0, min(C, c0 + per)) for c0 in range(0, C, per)]

    def tokenize(ch):
        return tokenizer([fn(c) for c in classnames[ch[0]:ch[1]] for fn in fns])

    bar = None
    if use_tqdm:
        try:
            from tqdm import tqdm

            bar = tqdm(total=C, desc="Building classifier", unit="class")
        except ImportError:
            pass
    W = model._pack("text", mode)
    feats = torch.empty((C * T, W.extra["proj"].N), dtype=BF if mode == "bf16" else F32, device=dev)
    row_of = np.empty(C * T, dtype=np.int32)
    with ThreadPoolExecutor(max_workers=1) as pool:
        nxt = pool.submit(tokenize, chunks[0])
        for i, ch in enumerate(chunks):
            ids = nxt.result()
            if i + 1 < len(chunks):
                nxt = pool.submit(tokenize, chunks[i + 1])
            p0 = ch[0] * T
            _, rows = encode_prompts(model, torch.as_tensor(ids), precision, out=feats, row0=p0, max_rows=max_rows)
            row_of[p0:p0 + len(rows)] = rows
            if bar is not None:
                bar.update(ch[1] - ch[0])
    if bar is not None:
        bar.close()
    out = torch.empty((_ceil8(C), feats.shape[1]), dtype=F32, device=dev)
    lib.zs_class_embed(feats, out, C, T, row_of=torch.from_numpy(row_of).to(dev))
    return out[:C].t().contiguous()


# ---------------------------------------------------------------------------------------------------------- image side
def accuracy_from_ranks(ranks: np.ndarray, topk: Sequence[int] = (1, 5)) -> List[float]:
    """test_zero_shot_hf.py:312-316 and :439-440 over all rows: 100 · #{rank < k} / n."""
    ranks = np.asarray(ranks)
    n = ranks.size
    return [float((ranks < k).sum()) / n * 100 for k in topk]


class _Step:
    """Device buffers of one batch shape (the graph's static inputs and outputs)."""

    def __init__(self, B: int, H: int, W: int, E: int, Cp: int, mode: str, dev, use_graph: bool):
        act = BF if mode == "bf16" else F32
        self.x = torch.empty((B, 3, H, W), dtype=act, device=dev)
        self.t = torch.empty(B, dtype=torch.int64, device=dev)
        self.a = torch.empty((B, E), dtype=act, device=dev)
        self.a3 = torch.empty((B, 3 * E), dtype=BF, device=dev) if mode == "fp32" else None
        self.logits = torch.empty((B, Cp), dtype=act, device=dev)
        self.ranks = torch.empty(B, dtype=torch.int32, device=dev)
        self.graph = StepGraph(dev, enabled=use_graph)


class ZeroShotEvaluator:
    """Top-k accuracy of a zero-shot classifier, accumulated on the device.

    classifier: fp32 [E, C] (as build_zero_shot_classifier returns it); its GEMM operand stays resident ([Cp, 3E]
    bf16x3 in fp32 mode, [Cp, E] bf16 in bf16 mode, Cp = ceil8(C)).  precision: "fp32" or "bf16" for the image tower
    and the logits, as the reference's autocast."""

    def __init__(self, model, classifier: torch.Tensor, precision: str = "fp32", topk: Sequence[int] = (1, 5),
                 use_graph: bool = True):
        self.mode = _mode(precision)
        self.model, self.topk, self.use_graph = model, tuple(int(k) for k in topk), use_graph
        if not 1 <= len(self.topk) <= lib.ZS_MAX_K:
            raise ValueError(f"topk: 1..{lib.ZS_MAX_K} values")
        self.device = model.trunk.cls_token.device
        if self.device.type != "cuda":
            raise lib.VtpError("ZeroShotEvaluator needs the model on the CUDA device (there is no CPU path)")
        if model.visual_proj is None:
            raise RuntimeError("CLIP not enabled. Set train_clip=True in config.")
        if classifier.dim() != 2 or not classifier.is_floating_point():
            raise ValueError(f"classifier must be a float [E, C] tensor, got {classifier.dtype} {tuple(classifier.shape)}")
        Ed, C = classifier.shape
        if Ed % 8:
            raise ValueError(f"classifier width E = {Ed} must be a multiple of 8")
        self.E, self.C, self.Cp = Ed, C, _ceil8(C)
        w = torch.zeros((self.Cp, Ed), dtype=F32, device=self.device)
        w[:C] = classifier.to(self.device, F32).t()
        if self.mode == "fp32":
            self.w_op = torch.empty((self.Cp, 3 * Ed), dtype=BF, device=self.device)
            lib.split3(w, self.w_op, self.Cp, Ed, b_side=True)
        else:
            self.w_op = torch.empty((self.Cp, Ed), dtype=BF, device=self.device)
            lib.cast_f32_to_bf16(w, self.w_op, w.numel())
        self.counts = torch.zeros(len(self.topk), dtype=torch.int64, device=self.device)
        self.n = 0
        self._ranks: List[torch.Tensor] = []
        self._steps: Dict[tuple, _Step] = {}

    # ------------------------------------------------------------------ the device step
    def _run(self, st: _Step) -> None:
        m = self.model
        saved = m.compute_mode
        try:
            m.compute_mode = self.mode
            f = m.get_clip_image_feature(st.x, normalize=False)
        finally:
            m.compute_mode = saved
        if f.shape[1] != self.E:
            raise ValueError(f"image features have width {f.shape[1]}, the classifier {self.E}")
        self.head(st, f.contiguous())

    def head(self, st: _Step, f: torch.Tensor) -> None:
        """The zero-shot head on unnormalised image features f [B, E]: operand, logits GEMM, ranks and hit counts."""
        B = f.shape[0]
        lib.zs_image_operand(f, st.a, 100.0)
        if self.mode == "fp32":
            lib.split3(st.a, st.a3, B, self.E, b_side=False)
            lib.gemm(st.a3, self.w_op, st.logits, M=B, N=self.Cp, K=3 * self.E, round_bf16=False)
        else:
            lib.gemm(st.a, self.w_op, st.logits, M=B, N=self.Cp, K=self.E)
        lib.zs_rank(st.logits, self.C, st.t, st.ranks, self.counts, self.topk)

    @torch.no_grad()
    def add(self, images: torch.Tensor, targets: torch.Tensor) -> None:
        """Score one batch: ImageNet-normalised fp32 or bf16 images [B,3,H,W] and int64 targets [B] (host, pinned or
        device).  Enqueues only.  In bf16 mode the images are rounded to bf16 first, as the reference's input cast."""
        if images.dim() != 4 or images.shape[1] != 3 or images.dtype not in (F32, BF):
            raise ValueError(f"add: fp32 or bf16 images [B,3,H,W] expected, got {images.dtype} {tuple(images.shape)}")
        B, _, H, W = images.shape
        if targets.dtype != torch.int64 or tuple(targets.shape) != (B,):
            raise ValueError(f"add: int64 targets [{B}] expected, got {targets.dtype} {tuple(targets.shape)}")
        key = (B, H, W)
        st = self._steps.get(key)
        if st is None:
            st = self._steps[key] = _Step(B, H, W, self.E, self.Cp, self.mode, self.device, self.use_graph)
        st.x.copy_(images, non_blocking=True)
        st.t.copy_(targets, non_blocking=True)
        st.graph(lambda: self._run(st))
        self.n += B
        self._ranks.append(st.ranks.clone())

    # ------------------------------------------------------------------ results
    def ranks(self) -> torch.Tensor:
        """Device int32 [N]: the rank of each image's target among the class logits (C for a target outside [0, C))."""
        return torch.cat(self._ranks) if self._ranks else torch.empty(0, dtype=torch.int32, device=self.device)

    def counts_host(self) -> List[int]:
        return [int(c) for c in self.counts.cpu().tolist()]

    def result(self) -> Tuple[float, ...]:
        """(top-k accuracy in percent for each k), as test_zero_shot_hf.py:434-440: float hit count / n * 100."""
        if self.n == 0:
            raise ValueError("no images were added")
        return tuple(float(c) / self.n * 100 for c in self.counts_host())

    def close(self) -> None:
        for st in self._steps.values():
            st.graph.release()


def evaluate(model, classifier: torch.Tensor, dataloader, device, precision: str = "fp32") -> Tuple[float, float]:
    """test_zero_shot_hf.py:401-441: (top1, top5) in percent."""
    ev = ZeroShotEvaluator(model, classifier, precision=precision, topk=(1, 5))
    dev = ev.device
    for images, targets in dataloader:
        ev.add(images.to(dev, non_blocking=True), targets.to(dev, non_blocking=True))
    top1, top5 = ev.result()
    ev.close()
    return top1, top5


# ---------------------------------------------------------------------------------------------------------- CLI
def build_parser() -> argparse.ArgumentParser:
    """The reference's flags (test_zero_shot_hf.py:473-486) plus --bpe_path and --prompts."""
    ap = argparse.ArgumentParser(description="Zero-shot ImageNet evaluation of a VTP checkpoint on the H100 path")
    ap.add_argument("--model_path", type=str, required=True, help="VTP checkpoint directory (config.json + safetensors)")
    ap.add_argument("--data_path", type=str, required=True, help="ImageFolder root of the evaluation images")
    ap.add_argument("--batch_size", type=int, default=128, help="batch size for evaluation")
    ap.add_argument("--num_workers", type=int, default=8, help="number of dataloader workers")
    ap.add_argument("--device", type=str, default="cuda:0", help="device (e.g. cuda:0)")
    ap.add_argument("--precision", type=str, default="fp32", choices=["fp32", "fp16", "bf16"])
    ap.add_argument("--bpe_path", type=str, default=None, help="BPE vocabulary (bpe_simple_vocab_16e6.txt.gz)")
    ap.add_argument("--prompts", type=str, default=None,
                    help="JSON {\"classnames\": [...], \"templates\": [\"a photo of a {c}.\", ...]}; default: read from "
                         f"the reference's tools/{REFERENCE_SCRIPT}")
    return ap


def make_transform(image_size: int):
    """test_zero_shot_hf.py:455-459."""
    from torchvision import transforms as Tv

    return Tv.Compose([Tv.Resize((image_size, image_size)), Tv.ToTensor(),
                       Tv.Normalize(mean=list(IMAGENET_DEFAULT_MEAN), std=list(IMAGENET_DEFAULT_STD))])


def run(args) -> Dict[str, float]:
    from torch.utils.data import DataLoader
    from torchvision.datasets import ImageFolder

    from .model import VTPModel
    from .text_tokenizer import BPETokenizer, find_bpe_file

    if args.precision == "fp16":
        raise NotImplementedError("--precision fp16: zero-shot runs in bf16 or fp32 only")
    device = torch.device(args.device)
    print("=" * 60)
    print("Zero-Shot ImageNet Evaluation (VTP HuggingFace)")
    print("=" * 60)
    print(f"Model path: {args.model_path}")
    print(f"Data path: {args.data_path}")
    print(f"Device: {device}")
    print(f"Precision: {args.precision}")
    print(f"Batch size: {args.batch_size}")
    print()
    classnames, templates = load_prompts(args.prompts, args.bpe_path)
    print("Loading model...")
    model = VTPModel.from_pretrained(args.model_path).to(device).eval()
    image_size = model.config.image_size
    context_length = model.config.text_context_length
    print(f"Image size: {image_size}")
    print(f"Context length: {context_length}")
    print("Loading tokenizer...")
    tokenizer = BPETokenizer(bpe_path=find_bpe_file(args.bpe_path), context_length=context_length)
    print(f"Loading ImageNet validation: {args.data_path}")
    dataset = ImageFolder(root=args.data_path, transform=make_transform(image_size))
    if len(dataset.classes) != len(classnames):
        raise ValueError(f"the dataset has {len(dataset.classes)} classes but there are {len(classnames)} class names")
    loader = DataLoader(dataset, batch_size=args.batch_size, shuffle=False, num_workers=args.num_workers,
                        pin_memory=True)
    num_samples = len(dataset)
    print(f"Number of samples: {num_samples}")
    if num_samples != 50000:
        print(f"  [Warning] Expected 50000 samples for ImageNet validation, got {num_samples}")
    print()
    print("Building zero-shot classifier...")
    classifier = build_zero_shot_classifier(model, tokenizer, classnames, templates, num_classes_per_batch=10,
                                            device=device, use_tqdm=True, precision=args.precision)
    print()
    print("Running evaluation...")
    top1, top5 = evaluate(model, classifier, loader, device=device, precision=args.precision)
    print()
    print("=" * 60)
    print("Results:")
    print(f"  ImageNet Zero-Shot Top-1 Accuracy: {top1:.2f}%")
    print(f"  ImageNet Zero-Shot Top-5 Accuracy: {top5:.2f}%")
    print("=" * 60)
    return {"top1": top1, "top5": top5}


def main(argv=None):
    return run(build_parser().parse_args(argv))


if __name__ == "__main__":
    main()
