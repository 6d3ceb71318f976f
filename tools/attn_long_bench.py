"""Attention forward and backward at long sequences (images above 256x256): CUDA-event timing of vtp_attention_fwd on
the launching stream, head_dim 64, one cls prefix token, VTP-Small (6 heads) and VTP-Large (16 heads) head counts.
T = 257 runs the single-pass short kernel, for comparison; every larger T runs the streaming kernel of
attention_long.cu.  Also times the fp32 accuracy-mode tiled kernel at T = 1025.  GPU only.

  python tools/attn_long_bench.py [--out /tmp/attn_long.json]

TFLOP/s counts the two patch-by-patch matmuls only, 4·B·H·(T-1)²·64 (the cls row and column are not counted); the
share of peak is against the 989 TFLOP/s dense bf16 figure of the H100 SXM data sheet.  B is chosen so that every
shape launches about 16 waves of 128-row query tiles on the card's SMs.

Backward rows time the training entry points at the same shapes: vtp_attention_bwd (single pass, "short", T = 257
only) and vtp_attention_bwd_long (streaming, "long", every T; δ workspace included).  Their TFLOP/s counts the five
algorithmic patch GEMMs, 10·B·H·(T-1)²·64; the streaming kernels recompute S and dP (7 GEMMs in all), and the two
recomputed GEMMs are NOT counted.  bwd_over_fwd is the backward time over the forward time at the same shape."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from vtp_b200 import lib

BF = torch.bfloat16
PEAK_BF16 = 989e12
ap = argparse.ArgumentParser()
ap.add_argument("--out", default=None)
ap.add_argument("--reps", type=int, default=20)
a = ap.parse_args()

q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                   capture_output=True, text=True).stdout.splitlines()
gpu = q[0].strip() if q else torch.cuda.get_device_name()
sms = torch.cuda.get_device_properties(0).multi_processor_count


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


rows, bwd_rows = [], []
for H, model in ((6, "VTP-Small"), (16, "VTP-Large")):
    for T in (257, 577, 1025, 2305, 4097):
        HW = T - 1
        B = max(1, -(-16 * sms // (-(-HW // 128) * H)))
        qkv = torch.randn(B * T, 3 * H * 64, device="cuda").to(BF)
        out = torch.empty(B * T, H * 64, device="cuda", dtype=BF)
        ms = time_ms(lambda: lib.attention_fwd(qkv, out, B, T, H, prefix=1))
        tf = 4 * B * H * HW * HW * 64 / ms / 1e9
        rows.append({"model": model, "H": H, "T": T, "B": B, "kernel": "short" if HW <= 256 else "long",
                     "ms": round(ms, 4), "tflops": round(tf, 1), "frac_of_bf16_peak": round(tf * 1e12 / PEAK_BF16, 3)})
        print(f"{model:9s} H={H:2d} T={T:5d} B={B:4d}: {ms:8.3f} ms  {tf:6.1f} TFLOP/s  "
              f"{tf * 1e12 / PEAK_BF16:6.1%} of 989", flush=True)
        lse = torch.empty(B, H, T, device="cuda")
        lib.attention_fwd(qkv, out, B, T, H, prefix=1, lse=lse)
        dout = torch.randn(B * T, H * 64, device="cuda").to(BF)
        dqkv = torch.empty_like(qkv)
        delta = torch.empty(B, H, T, device="cuda")
        kernels = {"long": lambda: lib.attention_bwd_long(qkv, out, dout, lse, delta, dqkv, B, T, H, prefix=1)}
        if HW <= 256:
            kernels = {"short": lambda: lib.attention_bwd(qkv, out, dout, lse, dqkv, B, T, H, prefix=1), **kernels}
        for kern, fn in kernels.items():
            mb = time_ms(fn)
            tb = 10 * B * H * HW * HW * 64 / mb / 1e9
            bwd_rows.append({"model": model, "H": H, "T": T, "B": B, "kernel": kern, "ms": round(mb, 4),
                             "tflops": round(tb, 1), "frac_of_bf16_peak": round(tb * 1e12 / PEAK_BF16, 3),
                             "bwd_over_fwd": round(mb / ms, 2)})
            print(f"  backward {kern:5s}: {mb:8.3f} ms  {tb:6.1f} TFLOP/s  {tb * 1e12 / PEAK_BF16:6.1%} of 989  "
                  f"{mb / ms:5.2f}x forward", flush=True)
        del qkv, out, lse, dout, dqkv, delta

f32 = []
for H in (6, 16):
    T, B = 1025, 8
    qkv = torch.randn(B * T, 3 * H * 64, device="cuda")
    out = torch.empty(B * T, H * 64, device="cuda")
    ms = time_ms(lambda: lib.attention_fwd_f32(qkv, out, B, T, H))
    f32.append({"H": H, "T": T, "B": B, "ms": round(ms, 3), "tflops": round(4 * B * H * T * T * 64 / ms / 1e9, 2)})
    print(f"fp32 tiled H={H:2d} T={T} B={B}: {ms:8.3f} ms", flush=True)

res = {"gpu": gpu, "rows": rows, "bwd_rows": bwd_rows, "f32_tiled": f32}
print(json.dumps(res))
if a.out:
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
