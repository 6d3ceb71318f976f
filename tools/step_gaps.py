"""Dev tool: where one training step's wall time goes ON THE DEVICE with real concurrency and warm caches.
Runs the benchmark step under torch.profiler (CUPTI kernel records), then prints: step time by CUDA events without the
profiler, summed kernel time, idle time between kernels (host-launch bubbles), host enqueue time, and a per-kernel table.
  python tools/step_gaps.py [--model small] [--batch 256] [--out /tmp/step_gaps.json]"""
import argparse
import collections
import json
import os
import re
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from vtp_b200 import lib
from vtp_b200.config import preset
from vtp_b200.memory import suggest_chunks
from vtp_b200.synthetic import make_batch, to_device
from vtp_b200.train import TrainConfig, VTPTrainer

ap = argparse.ArgumentParser()
ap.add_argument("--model", default="small")
ap.add_argument("--batch", type=int, default=256)
ap.add_argument("--out", default=None)
ap.add_argument("--graph", action="store_true", help="profile the CUDA-graph replay of the step")
a = ap.parse_args()
dev = torch.device("cuda")
cfg = preset(a.model)
sc, rc = suggest_chunks(cfg, a.batch, head_out_dim=65536, lpips=True)
tr = VTPTrainer(cfg, TrainConfig(ssl_chunk=sc, rec_chunk=rc), device=dev)
tr.enable_lpips(seed=0, chunk=32)
b = to_device(make_batch(a.batch, vocab=cfg.text_vocab_size), dev, non_blocking=False)
step = tr.train_step
if a.graph:
    tr.capture_step(b)
    step = lambda batch: tr.replay_step(batch)
for _ in range(3):
    step(b)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
l0 = lib.LAUNCHES
e0.record()
c0 = time.perf_counter()
for _ in range(3):
    step(b)
host_ms = (time.perf_counter() - c0) / 3 * 1e3
e1.record()
torch.cuda.synchronize()
step_ms = e0.elapsed_time(e1) / 3
launches = (lib.LAUNCHES - l0) // 3
from torch.profiler import ProfilerActivity, profile

with profile(activities=[ProfilerActivity.CUDA]) as prof:
    step(b)
    torch.cuda.synchronize()
ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
ks = sorted(((e.time_range.start, e.time_range.end, e.name) for e in ev), key=lambda t: t[0])
busy, idle, cur_end = 0.0, 0.0, None
gaps = []
for s, e, n in ks:
    if cur_end is None:
        cur_end = e
        busy += e - s
        continue
    if s > cur_end:
        idle += s - cur_end
        gaps.append((s - cur_end, n))
        busy += e - s
        cur_end = e
    else:
        if e > cur_end:
            busy += e - cur_end
            cur_end = e
span = ks[-1][1] - ks[0][0] if ks else 0.0
agg = collections.defaultdict(lambda: [0, 0.0])
for s, e, n in ks:
    n = re.sub(r"\(.*$", "", n)
    n = re.sub(r"^void ", "", n)
    agg[n][0] += 1
    agg[n][1] += (e - s)
tot = sum(v[1] for v in agg.values())
rows = sorted(agg.items(), key=lambda kv: -kv[1][1])
print(f"step (CUDA events, no profiler): {step_ms:.1f} ms   host enqueue {host_ms:.1f} ms   vtp launches/step {launches}")
print(f"profiled step: span {span / 1e3:.1f} ms, device busy {busy / 1e3:.1f} ms, idle between kernels {idle / 1e3:.1f} ms "
      f"({100 * idle / max(span, 1):.1f} %), {len(ks)} device activities, summed kernel time {tot / 1e3:.1f} ms")
print("| kernel | n | total ms | share | avg us |\n|---|---:|---:|---:|---:|")
for n, (c, t) in rows[:45]:
    print(f"| `{n[:90]}` | {c} | {t / 1e3:.2f} | {100 * t / tot:.1f}% | {t / c:.1f} |")
gaps.sort(reverse=True)
print("largest idle gaps (us, before kernel):", [(round(g, 1), re.sub(r"\(.*$", "", n)[:40]) for g, n in gaps[:12]])
if a.out:
    json.dump({"step_ms": step_ms, "host_enqueue_ms": host_ms, "launches": launches, "span_ms": span / 1e3, "busy_ms": busy / 1e3,
               "idle_ms": idle / 1e3, "kernels": [{"name": n, "n": c, "ms": t / 1e3} for n, (c, t) in rows]}, open(a.out, "w"))
