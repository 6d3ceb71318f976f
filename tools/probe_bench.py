"""Linear-probe training step (vtp_b200/probe.py) at the reference's shapes: batch 128 per GPU, 224x224 images, 1 000
classes, the default grid of 24 classifiers (n = 1 and 4 last blocks x 13 learning rates, two keys collide at world 1),
VTP-S and VTP-L trunks with seeded random weights, bf16 trunk.  GPU only; CUDA-event timing on the launching stream.

  python tools/probe_bench.py [--out /tmp/probe.json] [--models s,l] [--reps 20]

Rows per model:
  step_ms      one whole training step by CUDA-graph replay (trunk forward + features + classifiers + SGD); img/s = B/step
  features_ms  trunk forward with the in-place feature taps (vtp_probe_features), eager launches
  classifier_ms  forward GEMMs + cross-entropy + dW GEMMs (classifier step minus its SGD), eager launches
  sgd_ms       the fused SGD-momentum update of every classifier, eager launches
  torch_classifier_ms  the same classifier part restated in eager torch as the reference runs it: G fp32 nn.Linear
               (TF32 off) on the assembled features, CrossEntropyLoss summed over classifiers, autograd, SGD(momentum
               0.9, foreach) and CosineAnnealingLR.step(); the reference's per-step loss.item() is included
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from vtp_b200 import probe as P
from vtp_b200.config import preset
from vtp_b200.model import VTPModel

ap = argparse.ArgumentParser()
ap.add_argument("--out", default=None)
ap.add_argument("--models", default="s,l")
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--batch", type=int, default=128)
a = ap.parse_args()

q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                   capture_output=True, text=True).stdout.splitlines()
gpu = q[0].strip() if q else torch.cuda.get_device_name()


def time_ms(fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def torch_classifier_step(probe, X, labels):
    """The eager reference formulation of the classifier part, built once per probe."""
    torch.backends.cuda.matmul.allow_tf32 = False
    sd = probe.state_dict()
    mods, groups = [], []
    for c in probe.classifiers:
        k = f"classifiers_dict.{c.key}.linear."
        lin = torch.nn.Linear(sd[k + "weight"].shape[1], probe.C).cuda()
        lin.weight.data.copy_(sd[k + "weight"])
        lin.bias.data.copy_(sd[k + "bias"])
        mods.append((c.n, lin))
        groups.append({"params": lin.parameters(), "lr": c.lr})
    opt = torch.optim.SGD(groups, momentum=0.9, weight_decay=0)
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, probe.max_iter, eta_min=0)
    crit = torch.nn.CrossEntropyLoss()
    D, nmax = probe.D, probe.nmax

    def step():
        loss = sum(crit(lin(X[:, (nmax - n) * D:]), labels) for n, lin in mods)
        opt.zero_grad()
        loss.backward()
        opt.step()
        sched.step()
        loss.item()
    return step


rows = []
for name in a.models.split(","):
    cfg = preset(name, train_clip=False, train_reconstruction=False)
    torch.manual_seed(0)
    m = VTPModel(cfg).cuda().eval()
    B = a.batch
    n_steps = 4 * a.reps + 20
    probe = P.LinearProbe(m, 1000, batch_size=B, max_iter=n_steps)
    x = torch.randn(B, 3, 224, 224, device="cuda")
    y = torch.randint(0, 1000, (B,), device="cuda")
    step_ms = time_ms(lambda: probe.train_step(x, y), a.reps)
    X = probe.features(x)
    feat_ms = time_ms(lambda: probe.features(x), a.reps)
    sgd_ms = time_ms(probe.sgd, a.reps)
    cls_ms = time_ms(lambda: probe.classifier_step(X, y), a.reps) - sgd_ms
    probe.release()
    ref_step = torch_classifier_step(probe, X, y)
    torch_ms = time_ms(ref_step, a.reps)
    row = dict(model=name, gpu=gpu, batch=B, image=224, classes=1000, classifiers=probe.G,
               step_ms=round(step_ms, 3), img_per_s=round(B / step_ms * 1e3, 1), features_ms=round(feat_ms, 3),
               classifier_ms=round(cls_ms, 3), sgd_ms=round(sgd_ms, 3), torch_classifier_ms=round(torch_ms, 3),
               classifier_speedup=round(torch_ms / (cls_ms + sgd_ms), 2))
    print(json.dumps(row), flush=True)
    rows.append(row)
    del probe, m, ref_step
    torch.cuda.empty_cache()
if a.out:
    with open(a.out, "w") as f:
        json.dump(rows, f, indent=1)
