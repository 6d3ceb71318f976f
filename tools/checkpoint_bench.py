"""Cost of saving and resuming a training run (VTPTrainer.save_checkpoint / load_checkpoint) on one GPU.

  python tools/checkpoint_bench.py [--presets small,large] [--dir /tmp] [--batch 4]

Per preset (head_out_dim 65 536, LPIPS on): a trainer captures its step graph (one warm-up step at --batch source images),
saves a checkpoint into a fresh directory under --dir and loads it back into itself, graph still captured.  Prints one
JSON line per preset: bytes written, expected bytes (12 B per parameter + 4 B per teacher parameter + the two centres,
from memory.param_count), save and load seconds (wall clock around each call, both synchronise the trainer's stream).
The load reads the files just written, so they are likely in the page cache: it measures deserialisation and the host to
device copies rather than the disk.  The directory is removed afterwards.  The card's name and power limit are read in the
same call."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from vtp_b200.config import preset
from vtp_b200.memory import param_count
from vtp_b200.synthetic import make_batch, to_device
from vtp_b200.train import TrainConfig, VTPTrainer

ap = argparse.ArgumentParser()
ap.add_argument("--presets", default="small,large")
ap.add_argument("--dir", default=tempfile.gettempdir())
ap.add_argument("--batch", type=int, default=4)
a = ap.parse_args()

gpu = torch.cuda.get_device_name(0)
try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError) as e:
    power = f"unread ({e})"

for name in a.presets.split(","):
    cfg = preset(name)
    tc = TrainConfig()
    tr = VTPTrainer(cfg, tc)
    tr.enable_lpips()
    tr.capture_step(to_device(make_batch(a.batch, vocab=cfg.text_vocab_size), "cuda"), warmup=1)
    root = tempfile.mkdtemp(prefix="vtp_ckpt_", dir=a.dir)
    path = os.path.join(root, "ck")
    try:
        t0 = time.perf_counter()
        tr.save_checkpoint(path)
        t_save = time.perf_counter() - t0
        written = sum(os.path.getsize(os.path.join(path, f)) for f in os.listdir(path))
        t0 = time.perf_counter()
        tr.load_checkpoint(path)
        t_load = time.perf_counter() - t0
        tr.replay_step()                       # the graph runs on from the loaded state
        torch.cuda.synchronize()
    finally:
        shutil.rmtree(root, ignore_errors=True)
    n = param_count(cfg, tc.head_out_dim, tc.head_hidden, tc.head_bottleneck)
    print(json.dumps({"preset": name, "gpu": gpu, "power_limit": power, "params": n["total"],
                      "teacher_params": n["teacher"], "bytes_written": written,
                      "bytes_expected": n["total"] * 12 + n["teacher"] * 4 + 2 * tc.head_out_dim * 4,
                      "save_s": round(t_save, 3), "load_s": round(t_load, 3),
                      "save_GBps": round(written / t_save / 1e9, 2), "load_GBps": round(written / t_load / 1e9, 2)}),
          flush=True)
    tr.release_graph()
    del tr
    torch.cuda.empty_cache()
