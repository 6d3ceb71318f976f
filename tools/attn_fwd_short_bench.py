"""Attention forward at the 256² step's shapes (128 < HW <= 256): CUDA-event timing of vtp_attention_fwd, head_dim 64,
at the exact batch sizes of one trunk / decoder call.  GPU only.

  python tools/attn_fwd_short_bench.py [--reps 20] [--rounds 3]

Each shape: 3 warm-up launches, then `rounds` windows of `reps` launches; the median window is reported.
TFLOP/s counts the two patch-by-patch matmuls, 4·B·H·(T-1)²·64.  The HBM floor is the bytes one call must move
(read qkv, write O and lse) at the 3.35 TB/s of the H100 SXM data sheet."""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from vtp_b200 import lib

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--rounds", type=int, default=3)
a = ap.parse_args()

SHAPES = [  # (model, B, H, T, prefix): VTP-Small trunk / decoder at 176 images, VTP-Large's 66
    ("VTP-Small", 176, 6, 257, 1), ("VTP-Small", 176, 6, 256, 0),
    ("VTP-Large", 66, 16, 257, 1), ("VTP-Large", 66, 16, 256, 0),
]
HBM_BPS = 3.35e12

q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                   capture_output=True, text=True).stdout.splitlines()
rows = []
for model, B, H, T, prefix in SHAPES:
    qkv = torch.randn(B * T, 3 * H * 64, device="cuda").to(torch.bfloat16)
    out = torch.empty(B * T, H * 64, device="cuda", dtype=torch.bfloat16)
    lse = torch.empty(B, H, T, device="cuda")
    fn = lambda: lib.attention_fwd(qkv, out, B, T, H, prefix=prefix, lse=lse)
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(a.rounds):
        torch.cuda.synchronize()
        e0.record()
        for _ in range(a.reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / a.reps)
    ms = statistics.median(times)
    HW = T - prefix
    tf = 4 * B * H * HW * HW * 64 / ms / 1e9
    floor_ms = (qkv.numel() * 2 + out.numel() * 2 + lse.numel() * 4) / HBM_BPS * 1e3
    rows.append({"model": model, "B": B, "H": H, "T": T, "prefix": prefix, "ms": round(ms, 4),
                 "ms_windows": [round(t, 4) for t in times], "tflops": round(tf, 1),
                 "hbm_floor_ms": round(floor_ms, 4), "hbm_floor_share": round(floor_ms / ms, 3)})
    print(f"{model:9s} B={B:3d} H={H:2d} T={T}: {ms:7.4f} ms  {tf:6.1f} TFLOP/s  HBM floor {floor_ms:.4f} ms "
          f"({floor_ms / ms:.0%})", flush=True)
print(json.dumps({"gpu": q[0].strip() if q else torch.cuda.get_device_name(), "rows": rows}))
