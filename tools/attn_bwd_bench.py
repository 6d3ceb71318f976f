"""Attention backward at the 256² training step's shapes: CUDA-event timing of vtp_attention_bwd (20 launches after 3
warm-ups) for T = 257 / prefix 1 (encoders) and T = 256 / prefix 0 (decoder), B = 176 with 6 heads (VTP-Small) and
B = 66 with 16 heads (VTP-Large), with RoPE.  GPU only.

  python tools/attn_bwd_bench.py [--repeats 5] [--out /tmp/attn_bwd.json]

TFLOP/s counts the five algorithmic patch GEMMs, 10·B·H·(T−1)²·64.  The HBM floor is the bytes the op must move,
read qkv, O and dO and write dqkv: 8·B·T·H·64·2 bytes, at the 3.35 TB/s of the H100 SXM data sheet; `frac_of_hbm_floor`
is that time over the measured time.  Each shape is timed `--repeats` times; min, median and max are reported."""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from vtp_b200 import lib

BF = torch.bfloat16
HBM_BPS = 3.35e12
ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--repeats", type=int, default=5)
ap.add_argument("--out", default=None)
a = ap.parse_args()

q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                   capture_output=True, text=True).stdout.splitlines()
gpu = q[0].strip() if q else torch.cuda.get_device_name()


def time_ms(fn):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(a.reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / a.reps


rows = []
for B, H, model in ((176, 6, "VTP-Small"), (66, 16, "VTP-Large")):
    for T, prefix in ((257, 1), (256, 0)):
        HW = T - prefix
        g = torch.Generator(device="cuda").manual_seed(T)
        qkv = (torch.randn(B * T, 3 * H * 64, device="cuda", generator=g) * 1.2).to(BF)
        dout = torch.randn(B * T, H * 64, device="cuda", generator=g).to(BF)
        ang = torch.rand(HW, 64, device="cuda", generator=g) * 6.28
        rope = (torch.sin(ang).to(BF), torch.cos(ang).to(BF))
        o = torch.empty(B * T, H * 64, device="cuda", dtype=BF)
        lse = torch.empty(B, H, T, device="cuda")
        lib.attention_fwd(qkv, o, B, T, H, prefix=prefix, lse=lse)
        dqkv = torch.empty_like(qkv)
        ms = sorted(time_ms(lambda: lib.attention_bwd(qkv, o, dout, lse, dqkv, B, T, H, prefix=prefix, rope=rope))
                    for _ in range(a.repeats))
        med = statistics.median(ms)
        tf = 10 * B * H * HW * HW * 64 / med / 1e9
        floor_ms = 8 * B * T * H * 64 * 2 / HBM_BPS * 1e3
        rows.append({"model": model, "B": B, "H": H, "T": T, "prefix": prefix, "ms_min": round(ms[0], 4),
                     "ms_median": round(med, 4), "ms_max": round(ms[-1], 4), "tflops": round(tf, 1),
                     "frac_of_hbm_floor": round(floor_ms / med, 3)})
        print(f"{model:9s} B={B:3d} H={H:2d} T={T}: {med:7.3f} ms (min {ms[0]:.3f}, max {ms[-1]:.3f})  "
              f"{tf:6.1f} TFLOP/s  {floor_ms / med:6.1%} of the HBM floor", flush=True)
        del qkv, dout, o, lse, dqkv

res = {"gpu": gpu, "rows": rows}
print(json.dumps(res))
if a.out:
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
