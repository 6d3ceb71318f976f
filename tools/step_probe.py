"""Dev tool: run each objective of the training step separately at a given batch with timing + memory (GPU only)."""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from vtp_b200 import lib, memory
from vtp_b200.config import preset
from vtp_b200.synthetic import make_batch, to_device
from vtp_b200.train import TrainConfig, VTPTrainer

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=256)
ap.add_argument("--model", default="small")
ap.add_argument("--prototypes", type=int, default=65536)
ap.add_argument("--reps", type=int, default=2)
ap.add_argument("--image-size", type=int, default=256)
ap.add_argument("--local-size", type=int, default=96)
a = ap.parse_args()
dev = torch.device("cuda")
cfg = preset(a.model)
t0 = time.time()
tr = VTPTrainer(cfg, TrainConfig(head_out_dim=a.prototypes), device=dev)
print(f"trainer built in {time.time()-t0:.1f}s, params {tr.store.n/1e6:.1f}M", flush=True)
b = to_device(make_batch(a.batch, image_size=a.image_size, local_size=a.local_size, vocab=cfg.text_vocab_size), dev,
              non_blocking=False)
# memory.train_step_bytes estimate (no LPIPS: this probe does not enable it), printed beside each measured peak
est = memory.train_step_bytes(cfg, a.batch, image=a.image_size, local=a.local_size, head_out_dim=a.prototypes, lpips=False)
base = est["persistent"] + est["inputs"]
print(f"batch ready {time.time()-t0:.1f}s", flush=True)


def timed(name, fn, est_bytes):
    for i in range(a.reps):
        torch.cuda.synchronize()
        l0 = lib.LAUNCHES
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        c0 = time.perf_counter()
        fn()
        cpu_ms = (time.perf_counter() - c0) * 1e3   # host time to enqueue everything (>= GPU time means launch-bound)
        e1.record()
        torch.cuda.synchronize()
        print(f"{name:10s} rep{i}: {e0.elapsed_time(e1):8.1f} ms  host enqueue {cpu_ms:7.1f} ms  launches {lib.LAUNCHES-l0:5d}  "
              f"peak mem {torch.cuda.max_memory_allocated()/2**30:.1f} GiB (estimate {est_bytes/2**30:.1f})", flush=True)


timed("clip", lambda: tr.clip_fwd_bwd(b["image"], b["text"], 1.0), base + est["clip"])
timed("rec", lambda: tr.rec_fwd_bwd(b["rec_image"], 1.0), base + est["rec"])
timed("ssl", lambda: tr.ssl_fwd_bwd(b["global_crops"], b["local_crops"], b["mask_indices"], b["masks_weight"], 1.0),
      base + est["ssl"])
timed("optimizer", lambda: tr.optimizer_step(), est["peak"])
timed("full step", lambda: tr.train_step(b), est["peak"])
print("losses", tr.loss_acc.cpu().tolist())
