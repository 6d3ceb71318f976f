"""TEST INFRASTRUCTURE ONLY — golden run of the REAL reference's linear probe (tools/test_linear_probing_hf.py) on CPU:

    python -m oracle.make_golden_probe      ->  tests/golden/probe_tiny.{npz,json}

The reference's own `setup_linear_classifiers`, `train_one_epoch` (one call per step, so every step's loss is seen) and
`evaluate` run on seeded fixed taps in place of a trunk: per step, 4 cls tokens [B, D] and patch tokens [B, HW, D]
(`oracle/probe_taps.py`, regenerated bit for bit by the tests).  D = 64, C = 37 (padding to 40 is exercised), B = 128, world 1
(24 classifiers: two scaled lrs collide), 30 steps, a cosine schedule over those 30 steps, then a held-out set of 256
rows.  The same run is repeated in fp64 (modules and features `.double()`): its distance from the fp32 run is the
tolerance yardstick.

Stored (the file stays small, so the weights are stored in part): the key list, every step's loss per classifier, the
final biases, the final weights of classes 0..15 and C-1 of every classifier (all input columns), the L2 norm of every
final weight row, the held-out accuracies, per held-out row and classifier whether the reference predicted the label and
its top-2 logit margin; and the fp32-vs-fp64 gaps of each of those.
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

from oracle.probe_taps import B, C, D, HW, N_EVAL, ROWS, SEED, STEPS, TAP_SEED, linear_input, probe_taps  # noqa: E402


def load_probe_module():
    rh.import_reference()
    path = os.path.join(rh.REF_ROOT, "tools", "test_linear_probing_hf.py")
    spec = importlib.util.spec_from_file_location("ref_linear_probing_hf", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def run(mod, dtype):
    if dtype == torch.float64:
        mod.create_linear_input = lambda x, use_n_blocks, use_avgpool: linear_input(x, use_n_blocks)
    sample, _ = probe_taps(0, 1, dtype)
    torch.manual_seed(SEED)
    clf, groups = mod.setup_linear_classifiers(sample, (1, 4), mod.DEFAULT_LEARNING_RATES, B, C, torch.device("cpu"))
    clf = clf.to(dtype)
    opt = torch.optim.SGD(groups, momentum=0.9, weight_decay=0)
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, STEPS, eta_min=0)
    crit = torch.nn.CrossEntropyLoss()
    keys = list(clf.classifiers_dict.keys())
    losses = np.zeros((STEPS, len(keys)))
    for t in range(STEPS):
        feats, labels = probe_taps(t, B, dtype)
        with torch.no_grad():
            out = clf(feats)
            losses[t] = [crit(out[k], labels).item() for k in keys]
        mod.train_one_epoch(lambda _: feats, clf, opt, sched, crit, [(torch.zeros(1), labels)], t, 1, torch.device("cpu"))
    feats, labels = probe_taps(-1, N_EVAL, dtype)
    acc = mod.evaluate(lambda _: feats, clf, [(torch.zeros(1), labels)], torch.device("cpu"))
    with torch.no_grad():
        out = clf(feats)
    correct = np.stack([(out[k].argmax(1) == labels).numpy() for k in keys])
    top2 = np.stack([out[k].topk(2, dim=1).values.double().numpy() for k in keys])
    w = {k: clf.classifiers_dict[k].linear.weight.detach().double().numpy() for k in keys}
    b = np.stack([clf.classifiers_dict[k].linear.bias.detach().double().numpy() for k in keys])
    return keys, losses, acc, correct, top2[..., 0] - top2[..., 1], w, b


def main():
    mod = load_probe_module()
    k32, l32, a32, c32, m32, w32, b32 = run(mod, torch.float32)
    k64, l64, a64, _, _, w64, b64 = run(mod, torch.float64)
    assert k32 == k64 and len(k32) == 24
    out = {"loss": l32.astype(np.float32), "bias": b32.astype(np.float32),
           "acc": np.asarray([a32[k] for k in k32]), "correct": c32, "margin": m32.astype(np.float32),
           "row_norm": np.stack([np.linalg.norm(w32[k], axis=1) for k in k32]),
           "gap_loss": np.abs(l32 - l64).max(axis=0), "gap_bias": np.abs(b32 - b64).max(axis=1),
           "gap_weight": np.asarray([np.abs(w32[k] - w64[k]).max() for k in k32]),
           "gap_margin": np.asarray([0.0])}
    for i, k in enumerate(k32):
        out[f"w{i}"] = w32[k][ROWS].astype(np.float32)
    # the logits' fp32-vs-fp64 distance on the held-out set bounds which rows may flip
    feats64, _ = probe_taps(-1, N_EVAL, torch.float64)
    gm = 0.0
    for i, k in enumerate(k32):
        n = int(k.split("_")[1])
        x = linear_input(feats64, n).numpy()
        gm = max(gm, float(np.abs(x @ (w32[k] - w64[k]).T + (b32[i] - b64[i])).max()))
    out["gap_margin"] = np.asarray([gm])
    path = os.path.join(ROOT, "tests", "golden", "probe_tiny")
    np.savez_compressed(path + ".npz", **out)
    meta = {"keys": k32, "D": D, "C": C, "B": B, "HW": HW, "steps": STEPS, "n_eval": N_EVAL, "seed": SEED,
            "tap_seed": TAP_SEED, "weight_rows": ROWS, "lrs": [g for g in mod.DEFAULT_LEARNING_RATES],
            "acc_fp64": [a64[k] for k in k64]}
    with open(path + ".json", "w") as f:
        json.dump(meta, f, indent=1)
    print(os.path.getsize(path + ".npz"), "bytes;", "max gaps: loss", out["gap_loss"].max(), "weight",
          out["gap_weight"].max(), "margin", gm)


if __name__ == "__main__":
    main()
