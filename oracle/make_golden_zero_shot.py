"""TEST INFRASTRUCTURE ONLY — golden run of the REAL reference's zero-shot tool (tools/test_zero_shot_hf.py) on CPU:

    python -m oracle.make_golden_zero_shot   ->  tests/golden/zero_shot_prompts.{json,npz}, tests/golden/zero_shot_tiny.{npz,json}

zero_shot_prompts: the reference's 1 000 class names (duplicates included) and its 80 templates as str.format strings
with {c}, plus the reference tokenizer's ids of all 80 000 prompts (class-major, c*80 + t), each row SOT .. EOT as
ragged uint16 with int64 offsets.  The GPU tests and the benchmark need the real prompt lengths but have no vocabulary.

zero_shot_tiny: the reference's own `build_zero_shot_classifier` and `evaluate` (imported from the script) on a seeded
tiny reference VTPModel (the "tiny" geometry with text_vocab_size 49408 so the real ids fit; the state-dict spec is
stored for `seeded_state_dict`), 48 classes x 80 templates (the first 40 classes and the 8 with the longest prompts,
so the 24-token bucket is covered) and 96 seeded 64x64 images.  Row i's target is the class at fp64 rank
[0,0,1,2,4,5,6,30][i % 8], so hits and misses at k = 1 and 5 both occur.  Three runs: fp32, fp64 (`model.double()`,
fp64 images) and bf16 under CPU autocast.  Stored per run: the unnormalised text features of the first 8 templates of
every class, the classifier [E, 48], the logits [96, 48], each row's target rank, the top-1 / top-5 accuracies; plus
the dtypes seen along the bf16 flow and the fp32-vs-fp64 (and bf16-vs-fp64) gaps that serve as tolerances.

CPU autocast differs from CUDA's in one place that matters here: `aten::norm` falls through under AutocastCPU, so
F.normalize of a bf16 feature stays bf16 on the CPU, while under CUDA autocast the norm runs in fp32 and the features
come out fp32.  In the bf16 run the model's two feature methods are therefore wrapped so that their normalisation
follows CUDA's policy, x / x.float().norm(dim=-1, keepdim=True).clamp_min(1e-12); everything else is the reference's
own code.
"""
from __future__ import annotations

import importlib.util
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_harness as rh  # noqa: E402
from oracle.seeded import seeded_images, seeded_state_dict  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
N_FIRST, N_LONG, N_IMG, SIZE = 40, 8, 96, 64
RANK_OF_TARGET = [0, 0, 1, 2, 4, 5, 6, 30]
N_TF_TEMPLATES = 8   # text features are stored for the first 8 templates of each class (the gaps cover all 80)


def load_zero_shot_module():
    rh.import_reference()
    path = os.path.join(rh.REF_ROOT, "tools", "test_zero_shot_hf.py")
    spec = importlib.util.spec_from_file_location("ref_zero_shot_hf", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod, path


def cuda_norm_policy(model):
    """Wrap get_clip_{image,text}_feature so that normalize=True divides by an fp32 norm (CUDA autocast's policy)."""
    for name in ("get_clip_image_feature", "get_clip_text_feature"):
        orig = getattr(model, name)

        def wrapped(x, normalize=True, _orig=orig):
            f = _orig(x, normalize=False)
            return f / f.float().norm(dim=-1, keepdim=True).clamp_min(1e-12) if normalize else f

        setattr(model, name, wrapped)


def ranks_of(logits: np.ndarray, targets: np.ndarray) -> np.ndarray:
    """#{j : l_j ahead of l_t}: NaN first, then larger, ties to the lower index (the rule of vtp_zs_rank)."""
    out = np.empty(len(targets), dtype=np.int64)
    C = logits.shape[1]
    for i, t in enumerate(targets):
        if not 0 <= t < C:
            out[i] = C
            continue
        l, lt = logits[i], logits[i, t]
        j = np.arange(C)
        if np.isnan(lt):
            ahead = np.isnan(l) & (j < t)
        else:
            ahead = np.isnan(l) | (l > lt) | ((l == lt) & (j < t))
        out[i] = int(ahead.sum())
    return out


def main():
    mod, script = load_zero_shot_module()
    from vtp.models.vtp_hf import VTPConfig, VTPModel
    from vtp.tokenizers import get_tokenizer
    from vtp_b200.zero_shot import read_reference_prompts

    torch.set_num_threads(os.cpu_count())
    classnames = list(mod.IMAGENET_CLASSNAMES)
    templates_fmt = read_reference_prompts(script)[1]
    assert len(classnames) == 1000 and len(templates_fmt) == 80
    tok = get_tokenizer("ViT-B-32", context_length=77)
    texts = [t(c) for c in classnames for t in mod.OPENAI_IMAGENET_TEMPLATES]
    assert texts == [t.format(c=c) for c in classnames for t in templates_fmt]
    ids = tok(texts).numpy()
    eot = ids.argmax(1)
    lens = eot + 1
    offsets = np.zeros(len(ids) + 1, dtype=np.int64)
    offsets[1:] = np.cumsum(lens)
    flat = np.concatenate([ids[i, :lens[i]] for i in range(len(ids))]).astype(np.uint16)
    assert int(ids.max()) < 65536
    np.savez_compressed(os.path.join(OUT, "zero_shot_prompts.npz"), ids=flat, offsets=offsets)
    with open(os.path.join(OUT, "zero_shot_prompts.json"), "w") as f:
        json.dump({"classnames": classnames, "templates": templates_fmt, "context_length": 77,
                   "eot_token": int(ids.max()), "max_len": int(lens.max()), "mean_len": float(lens.mean())}, f, indent=0)

    # ---- tiny model run
    class_max = lens.reshape(1000, 80).max(1)
    longest = [int(c) for c in np.argsort(-class_max, kind="stable") if c >= N_FIRST][:N_LONG]
    sel = list(range(N_FIRST)) + sorted(longest)
    names = [classnames[c] for c in sel]
    kw = dict(vision_embed_dim=128, vision_depth=2, vision_num_heads=2, text_embed_dim=128, text_num_heads=2,
              text_depth=2, decoder_embed_dim=128, decoder_num_heads=2, decoder_depth=2, text_vocab_size=49408,
              image_size=SIZE)
    cfg = VTPConfig(**kw)
    spec = {k: list(v.shape) for k, v in VTPModel(cfg).state_dict().items()}
    x = seeded_images(N_IMG, SIZE, SIZE, seed=7)

    def model_for(dtype):
        m = VTPModel(cfg).eval()
        m.load_state_dict(seeded_state_dict(spec, seed=0))
        return m.double() if dtype == torch.float64 else m

    sel_ids = ids.reshape(1000, 80, 77)[sel].reshape(-1, 77)
    runs = {}
    targets = np.zeros(N_IMG, dtype=np.int64)
    dtypes_seen = {}
    input_dtype = mod.get_input_dtype
    for tag in ("fp64", "fp32", "bf16"):
        dt = torch.float64 if tag == "fp64" else torch.float32
        m = model_for(dt)
        if tag == "bf16":
            cuda_norm_policy(m)
        prec = "bf16" if tag == "bf16" else "fp32"
        ctx = mod.get_autocast_context(prec, device_type="cpu")
        with torch.no_grad(), ctx():
            clf = mod.build_zero_shot_classifier(m, tok, names, mod.OPENAI_IMAGENET_TEMPLATES, num_classes_per_batch=10,
                                                 device=torch.device("cpu"), use_tqdm=False)
            tf = m.get_clip_text_feature(torch.from_numpy(sel_ids), normalize=False)
        imgs = x.to(torch.float64 if tag == "fp64" else (torch.bfloat16 if tag == "bf16" else torch.float32))
        with torch.inference_mode(), ctx():
            fi = m.get_clip_image_feature(imgs, normalize=True)
            logits = 100.0 * fi @ clf
        if tag == "bf16":
            dtypes_seen = {"text_feature": str(tf.dtype), "classifier": str(clf.dtype), "image_feature": str(fi.dtype),
                           "logits": str(logits.dtype)}
        if tag == "fp64":
            order = np.argsort(-logits.numpy(), axis=1, kind="stable")
            targets = np.array([order[i, RANK_OF_TARGET[i % 8]] for i in range(N_IMG)], dtype=np.int64)
        loader = [(imgs[i:i + 32], torch.from_numpy(targets[i:i + 32])) for i in range(0, N_IMG, 32)]
        mod.get_input_dtype = (lambda p: torch.float64) if tag == "fp64" else input_dtype
        top1, top5 = mod.evaluate(m, clf, loader, torch.device("cpu"), prec)
        lg = logits.double().numpy()
        runs[tag] = dict(text_feat=tf.double().numpy(), classifier=clf.double().numpy(), logits=lg,
                         ranks=ranks_of(lg, targets), top1=top1, top5=top5)
    out = {"class_index": np.asarray(sel, dtype=np.int64), "targets": targets}
    for tag, r in runs.items():
        out[f"text_feat_{tag}"] = r["text_feat"].reshape(len(sel), 80, -1)[:, :N_TF_TEMPLATES].astype(np.float32)
        for k in ("classifier", "logits"):
            out[f"{k}_{tag}"] = r[k].astype(np.float64 if tag == "fp64" else np.float32)
        out[f"ranks_{tag}"] = r["ranks"]
    gaps = {k: float(np.abs(runs["fp32"][k] - runs["fp64"][k]).max()) for k in ("text_feat", "classifier", "logits")}
    gaps_bf16 = {k: float(np.abs(runs["bf16"][k] - runs["fp64"][k]).max()) for k in ("text_feat", "classifier", "logits")}
    np.savez_compressed(os.path.join(OUT, "zero_shot_tiny.npz"), **out)
    meta = {"config": kw, "spec": spec, "seed": 0, "image_seed": 7, "n_images": N_IMG, "image_size": SIZE,
            "classes": sel, "rank_of_target": RANK_OF_TARGET,
            "counts": {tag: {"top1": r["top1"], "top5": r["top5"]} for tag, r in runs.items()},
            "bf16_dtypes": dtypes_seen, "gap_fp32_fp64": gaps, "gap_bf16_fp64": gaps_bf16, "torch": torch.__version__}
    with open(os.path.join(OUT, "zero_shot_tiny.json"), "w") as f:
        json.dump(meta, f, indent=1)
    print("prompts: max len", int(lens.max()), "mean", float(lens.mean()), "; tiny:", meta["counts"], gaps, gaps_bf16,
          dtypes_seen)


if __name__ == "__main__":
    main()
