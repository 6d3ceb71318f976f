"""Zero-shot classification (vtp_b200/zero_shot.py) at the reference's shapes.  GPU only; CUDA-event timing on the
launching stream; every shape is warmed before it is timed.  Inputs come from the fixtures and seeds only.

  python tools/zero_shot_bench.py [--out /tmp/zs.json] [--models s,b,l] [--reps 5]

Classifier build, per text-tower geometry (VTP-S / B / L, seeded weights), over the 80 000 prompts of the fixture
(1 000 ImageNet classes x 80 templates, tokenised by the reference tokenizer; tests/golden/zero_shot_prompts.*):
  bucketed_ms   text tower on length buckets (each prompt up to its end token) + vtp_zs_class_embed
  full_ms       text tower on full 77-token rows in batches of 800 prompts (the reference's 10 classes x 80 templates)
                + vtp_zs_class_embed; the bucketed and full-length features are checked bit-identical first
  tokenize_ms   host BPE tokenization of the 80 000 prompts (the reference vocabulary at $VTP_BPE_PATH, else the
                16 000-merge prefix of it in tests/golden/bpe_prefix.txt.gz)
Evaluation, batch 128 at 256x256 on the VTP-L image tower:
  eval_batch_ms  one whole batch by CUDA-graph replay (image tower + zero-shot head)
  head_ms        the zero-shot head alone (vtp_zs_image_operand + logits GEMM + vtp_zs_rank), eager launches
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from oracle.seeded import seeded_images, seeded_state_dict
from vtp_b200 import engine as E
from vtp_b200 import lib
from vtp_b200 import zero_shot as Z
from vtp_b200.config import preset
from vtp_b200.model import VTPModel

ap = argparse.ArgumentParser()
ap.add_argument("--out", default=None)
ap.add_argument("--models", default="s,b,l")
ap.add_argument("--reps", type=int, default=5)
a = ap.parse_args()

q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                   text=True).stdout.splitlines()
gpu = q[0].strip() if q else torch.cuda.get_device_name()


def time_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def fixture():
    with open(os.path.join(ROOT, "tests", "golden", "zero_shot_prompts.json")) as f:
        meta = json.load(f)
    z = np.load(os.path.join(ROOT, "tests", "golden", "zero_shot_prompts.npz"))
    flat, off = z["ids"].astype(np.int64), z["offsets"]
    ids = np.zeros((len(off) - 1, 77), dtype=np.int64)
    for i in range(len(off) - 1):
        ids[i, :off[i + 1] - off[i]] = flat[off[i]:off[i + 1]]
    return meta, torch.from_numpy(ids)


def model(name, **over):
    m = VTPModel(preset(name, **over))
    m.load_state_dict(seeded_state_dict({k: list(v.shape) for k, v in m.state_dict().items()}, seed=0))
    return m.cuda().eval()


meta, ids = fixture()
C, T = len(meta["classnames"]), len(meta["templates"])
rows = []
from vtp_b200.text_tokenizer import BPETokenizer

# the reference vocabulary when $VTP_BPE_PATH names it, else the 16 000-merge prefix of it that the tests carry
vocab = os.environ.get("VTP_BPE_PATH") or os.path.join(ROOT, "tests", "golden", "bpe_prefix.txt.gz")
tok = BPETokenizer(bpe_path=vocab, context_length=77)
texts = [t.format(c=c) for c in meta["classnames"] for t in meta["templates"]]
t0 = time.perf_counter()
tok(texts)
tok_ms = (time.perf_counter() - t0) * 1e3
print(json.dumps({"tokenize_ms": tok_ms, "vocabulary": os.path.basename(vocab), "prompts": len(texts)}), flush=True)

for name in a.models.split(","):
    m = model(name)
    for mode in ("bf16", "fp32"):
        W = m._pack("text", mode)
        Ed = W.extra["proj"].N
        cls = torch.empty(((C + 7) // 8 * 8, Ed), device="cuda")

        def bucketed():
            feats, row_of = Z.encode_prompts(m, ids, mode)
            lib.zs_class_embed(feats, cls, C, T, row_of=torch.from_numpy(row_of).cuda())
            return feats, row_of

        ids_dev = ids.cuda()

        def full():
            feats = torch.empty((C * T, Ed), dtype=torch.bfloat16 if mode == "bf16" else torch.float32, device="cuda")
            for s in range(0, C * T, 800):
                feats[s:s + 800].copy_(E.text_forward(W, ids_dev[s:s + 800], mode))
            lib.zs_class_embed(feats, cls, C, T)
            return feats

        fb, row_of = bucketed()
        ff = full()
        identical = bool(torch.equal(fb[torch.from_numpy(row_of).long().cuda()], ff))
        del fb, ff
        r = {"model": name, "mode": mode, "E": Ed, "identical": identical, "gpu": gpu}
        if identical:
            r["bucketed_ms"] = time_ms(bucketed, a.reps)
            r["full_ms"] = time_ms(full, a.reps)
            r["speedup"] = r["full_ms"] / r["bucketed_ms"]
        r["tokenize_ms"] = tok_ms
        rows.append(r)
        print(json.dumps(r), flush=True)
    del m
    torch.cuda.empty_cache()

# evaluation step on the VTP-L image tower
m = model("l")
x = seeded_images(128, 256, 256, seed=3).cuda()
tg = torch.randint(0, C, (128,), generator=torch.Generator().manual_seed(4)).cuda()
clf = torch.nn.functional.normalize(torch.randn(m.text_projection.shape[0], C, generator=torch.Generator().manual_seed(5)),
                                    dim=0).cuda()
for mode in ("bf16", "fp32"):
    ev = Z.ZeroShotEvaluator(m, clf, precision=mode)
    step = lambda: ev.add(x, tg)
    step()
    step()                                            # the capture
    r = {"model": "l", "mode": mode, "batch": 128, "image": 256, "gpu": gpu, "eval_batch_ms": time_ms(step, a.reps * 4)}
    st = next(iter(ev._steps.values()))
    saved = m.compute_mode
    m.compute_mode = mode
    f = m.get_clip_image_feature(st.x, normalize=False)
    m.compute_mode = saved

    def head():
        ev.head(st, f)

    r["head_ms"] = time_ms(head, a.reps * 20)
    rows.append(r)
    print(json.dumps(r), flush=True)
    ev.close()

if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rows, f, indent=1)
