"""Cost of the photometric augmentations (vtp_crop_augment, csrc/data.cu) on one GPU.

  python tools/data_bench.py [--rounds 3] [--steps 10] [--batch 128] [--out /tmp/data_bench.json]

1. Kernel time: device time of vtp_crop_augment (stats + apply kernel, CUDA events over 20 launches after 3 warm-ups),
   the stats kernel's share (torch.profiler, a separate pass), and vtp_crop_resize_norm on the same crops, against the
   HBM bound of the 12 B per output pixel written (3.35 TB/s, H100 SXM data sheet).  Shapes: 256 source images -> 512
   global crops at 256² + 2 048 local crops at 96²; 64 images -> 128 global crops at 512² + 512 local crops at 192².
   Tables: the DINOv2 recipe as TrainBatchPipeline samples it, and every stage on (jitter, grayscale, blur, solarise).
2. Step time: the VTP-Small graph step fed by TrainBatchPipeline (256², 8 local crops at 96²), photometric augmentation
   on and off in alternating rounds within this one call, so the spread between rounds of the same arm is measured
   alongside the difference between arms.  The pipeline prepares step i + 1 on its side stream under step i.
The card's name and power limit are read in the same call."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from vtp_b200 import lib
from vtp_b200.data import PhotometricAug, TrainBatchPipeline, photometric_params, random_resized_crop_boxes

HBM_BPS = 3.35e12
ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--batch", type=int, default=128)
ap.add_argument("--out", default="/tmp/data_bench.json")
a = ap.parse_args()
dev = "cuda"
res = {"gpu": torch.cuda.get_device_name(0)}
try:
    res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                        capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError) as e:
    res["power_limit"] = f"unread ({e})"
print(res, flush=True)


def crops(B, N, S, scale, rng):
    H, W = S + S // 8, S + S // 4
    src = torch.randint(0, 256, (B, H, W, 3), dtype=torch.uint8, device=dev)
    boxes = torch.from_numpy(random_resized_crop_boxes(rng, N, H, W, scale)).to(dev)
    idx = torch.from_numpy(np.tile(np.arange(B, dtype=np.int32), N // B)).to(dev)
    flips = torch.from_numpy((rng.random(N) < 0.5).astype(np.uint8)).to(dev)
    return src, idx, boxes, flips, torch.empty(N, 3, S, S, device=dev), torch.empty(N, device=dev)


def events(fn, reps=20, warm=3):
    for _ in range(warm):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def stats_share(fn, reps=20):
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    tot = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            tot[ev.name] = tot.get(ev.name, 0.0) + ev.device_time_total
    stats = sum(v for k, v in tot.items() if "crop_augment_stats" in k) / reps / 1e3
    apply = sum(v for k, v in tot.items() if "crop_augment_kernel" in k) / reps / 1e3
    return stats, apply


aug = PhotometricAug()
kern = []
for B, S, Sl in ((256, 256, 96), (64, 512, 192)):
    rng = np.random.default_rng(0)
    for name, N, size, scale, tables in (
            ("global", 2 * B, S, (0.32, 1.0),
             {"recipe": np.concatenate([photometric_params(rng, B, aug, aug.blur_p[0], 0.0),
                                        photometric_params(rng, B, aug, aug.blur_p[1], aug.solarize_p)])}),
            ("local", 8 * B, Sl, (0.05, 0.32), {"recipe": photometric_params(rng, 8 * B, aug, aug.blur_p[2], 0.0)})):
        tables["all_on"] = photometric_params(rng, N, PhotometricAug(jitter_p=1.0, gray_p=1.0), 1.0, 1.0)
        src, idx, boxes, flips, out, ws = crops(B, N, size, scale, rng)
        bound_ms = N * size * size * 12 / HBM_BPS * 1e3
        plain = events(lambda: lib.crop_resize_norm(src, idx, boxes, flips, out))
        for tname, t in tables.items():
            prm = torch.from_numpy(t).to(dev)
            fn = lambda: lib.crop_augment(src, idx, boxes, flips, prm, ws, out)
            ms = events(fn)
            st_ms, ap_ms = stats_share(fn)
            row = dict(images=B, crops=name, N=N, S=size, table=tname, augment_ms=round(ms, 4),
                       stats_kernel_ms=round(st_ms, 4), apply_kernel_ms=round(ap_ms, 4), crop_resize_norm_ms=round(plain, 4),
                       hbm_bound_ms=round(bound_ms, 4), share_of_hbm_bound=round(bound_ms / ms, 3),
                       write_gbs=round(N * size * size * 12 / ms / 1e6, 1))
            kern.append(row)
            print(json.dumps(row), flush=True)
        del src, out
res["kernels"] = kern
for B, S, Sl in ((256, 256, 96), (64, 512, 192)):
    tot = [sum(r["augment_ms"] for r in kern if r["images"] == B and r["table"] == "recipe"),
           sum(r["hbm_bound_ms"] for r in kern if r["images"] == B and r["table"] == "recipe")]
    res[f"recipe_{B}_images_ms"] = {"augment": round(tot[0], 3), "hbm_bound": round(tot[1], 3)}

# ------------------------------------------------------------------------------------------------------ step time
from vtp_b200.config import preset
from vtp_b200.memory import suggest_chunks
from vtp_b200.train import TrainConfig, VTPTrainer

torch.cuda.empty_cache()
cfg = preset("small")
B = a.batch
ssl_chunk, rec_chunk = suggest_chunks(cfg, B, head_out_dim=65536, lpips=False)
tr = VTPTrainer(cfg, TrainConfig(head_out_dim=65536, ssl_chunk=ssl_chunk, rec_chunk=rec_chunk))
src = torch.randint(0, 256, (B, 288, 320, 3), dtype=torch.uint8).pin_memory()
ids = torch.randint(1, cfg.text_vocab_size - 2, (B, 77), dtype=torch.long).pin_memory()
pipes = {arm: TrainBatchPipeline(dev, n_local=8, seed=0, photometric=PhotometricAug() if arm == "on" else None)
         for arm in ("off", "on")}
for p in pipes.values():
    p.submit(src, ids)
tr.capture_step(pipes["off"].get(), warmup=2)
pipes["off"].submit(src, ids)
times = {"off": [], "on": []}
for r in range(a.rounds):
    for arm in ("off", "on"):
        p = pipes[arm]
        for _ in range(2):                       # settle this arm's queue
            tr.replay_step(p.get())
            p.submit(src, ids)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.steps):
            batch = p.get()
            p.submit(src, ids)
            tr.replay_step(batch)
        torch.cuda.synchronize()
        times[arm].append((time.perf_counter() - t0) * 1e3 / a.steps)
        print(f"round {r} {arm}: {times[arm][-1]:.1f} ms/step", flush=True)
for p in pipes.values():
    p.get()
    p.close()
res["step"] = {"model": "VTP-Small", "batch": B, "image": 256, "local": "8 x 96", "lpips": False, "graph": True,
               "ms_per_step": {k: [round(x, 2) for x in v] for k, v in times.items()},
               "median_ms": {k: round(float(np.median(v)), 2) for k, v in times.items()}}
print(json.dumps(res, indent=1))
with open(a.out, "w") as f:
    json.dump(res, f, indent=1)
