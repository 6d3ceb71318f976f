"""FID on the device (vtp_b200/fid.py) at pytorch-fid's batch of 50, with seeded stand-in Inception weights (the same
shapes and FLOPs as pytorch-fid's).  GPU only; CUDA-event timing on the launching stream, the per-stage split from a
separate torch.profiler run.

  python tools/fid_bench.py [--out /tmp/fid.json] [--reps 10]

Rows:
  forward        FIDInception.accumulate on B uint8 256x256 images (resize, 94 convs, pools, moments): ms, img/s, and
                 the split by kernel family (resize, im2col = vtp_fid_im2col3 + vtp_split3, gemm, pool, moments) with
                 the model FLOPs (2·M·N·taps·Cin per conv, the unsplit product) and the bf16x3 operand bytes written by
                 im2col / split3, both computed from the shapes here
  frechet        host frechet_distance on 2048² covariances (scipy sqrtm), ms
  recon_eval     ReconstructionEvaluator.add (graph replay, PNGs written to a temporary directory) at B = 32 on 256²
                 with the VTP-S model, without and with rFID: img/s
  torch_tf32     the reference network (oracle/fid_inception.py) in eager fp32 torch with cuDNN's default TF32
                 convolutions, what pytorch-fid runs: ms and img/s at the same B
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from vtp_b200 import fid, lib

ap = argparse.ArgumentParser()
ap.add_argument("--out", default=None)
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--batch", type=int, default=50)
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


def shape_counts():
    """(model FLOPs, im2col / split3 operand bytes) per image, from the conv shapes."""
    sizes = {"Conv2d_1a_3x3": 299, "Conv2d_2a_3x3": 149, "Conv2d_2b_3x3": 147, "Conv2d_3b_1x1": 73, "Conv2d_4a_3x3": 73}
    flops = opbytes = 0
    for name, (ci, co, kh, kw, s, ph, pw) in fid.CONVS.items():
        if name in sizes:
            H = sizes[name]
        else:
            blk = name.split(".")[0]
            H = 35 if blk in ("Mixed_5b", "Mixed_5c", "Mixed_5d", "Mixed_6a") else (17 if blk < "Mixed_7a" else 8)
            if blk == "Mixed_7a":
                H = 17
        Ho, Wo = lib.fid_conv_out(H, H, kh, kw, s, ph, pw)
        M = Ho * Wo
        flops += 2 * M * co * kh * kw * ci
        opbytes += M * (96 if ci == 3 else kh * kw * 3 * ci) * 2
    return flops, opbytes


B = a.batch
net = fid.FIDInception.random_init(0)
st = fid.FIDStatistics()
u8 = torch.randint(0, 256, (B, 256, 256, 3), dtype=torch.uint8, device="cuda")
fwd_ms = time_ms(lambda: net.accumulate(u8, st, B), a.reps)
flops, opbytes = shape_counts()

from torch.profiler import ProfilerActivity, profile

with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(3):
        net.accumulate(u8, st, B)
    torch.cuda.synchronize()
split = {"resize": 0.0, "im2col": 0.0, "gemm": 0.0, "pool": 0.0, "moments": 0.0, "other": 0.0}
for ev in prof.key_averages():
    n, t = ev.key, ev.device_time_total / 1e3 / 3   # ms per forward
    if t <= 0:
        continue
    k = ("resize" if "fid_resize" in n else "im2col" if ("im2col3" in n or "split3" in n) else "gemm" if "gemm_kernel" in n
         else "pool" if "fid_pool" in n else "moments" if "fid_moments" in n else "other")
    split[k] += t
gemm_ms = split["gemm"]
row_fwd = dict(gpu=gpu, row="forward", batch=B, image=256, ms=round(fwd_ms, 3), img_per_s=round(B / fwd_ms * 1e3, 1),
               split_ms={k: round(v, 3) for k, v in split.items()},
               model_gflop_per_img=round(flops / 1e9, 3), gemm_tflops_model=round(flops * B / gemm_ms / 1e9, 1) if gemm_ms else None,
               operand_mb_per_img=round(opbytes / 1e6, 1),
               im2col_TBps_written=round(opbytes * B / split["im2col"] / 1e9, 3) if split["im2col"] else None)
print(json.dumps(row_fwd), flush=True)

rng = np.random.default_rng(0)
X = rng.normal(size=(2304, 2048))
Y = rng.normal(size=(2304, 2048)) * 1.1
m1, s1, m2, s2 = X.mean(0), np.cov(X, rowvar=False), Y.mean(0), np.cov(Y, rowvar=False)
t = time.perf_counter()
fid.frechet_distance(m1, s1, m2, s2)
row_fr = dict(gpu=gpu, row="frechet", dims=2048, ms=round((time.perf_counter() - t) * 1e3, 1))
print(json.dumps(row_fr), flush=True)

from vtp_b200.config import preset
from vtp_b200.model import VTPModel
from vtp_b200.recon_eval import ReconstructionEvaluator

torch.manual_seed(0)
m = VTPModel(preset("s", train_clip=False)).cuda().eval()
x = torch.randn(32, 3, 256, 256, device="cuda")
rec_rows = {}
for label, fnet in (("without_rfid", None), ("with_rfid", net)):
    with tempfile.TemporaryDirectory() as tmp:
        ev = ReconstructionEvaluator(m, save_dir=tmp, batch_size=32, fid=fnet)
        for _ in range(2):
            ev.add(x)
        ev.flush()
        torch.cuda.synchronize()
        t = time.perf_counter()
        n = max(4, a.reps)
        for _ in range(n):
            ev.add(x)
        ev.flush()
        torch.cuda.synchronize()
        rec_rows[label] = round(32 * n / (time.perf_counter() - t), 1)
        # the device step alone (graph replay, no PNG copy or writer)
        st_ = ev._steps[(32, 256, 256)]
        rec_rows[label + "_step_ms"] = round(time_ms(st_.graph.replay, a.reps), 3)
        ev.close()
row_rec = dict(gpu=gpu, row="recon_eval", model="s", batch=32, image=256, img_per_s=rec_rows)
print(json.dumps(row_rec), flush=True)
del m

from oracle.fid_inception import features as oracle_features
from oracle.fid_inception import fid_inception

n32 = fid_inception(fid.random_weights(0), dtype=torch.float32, device="cuda")
img = u8.permute(0, 3, 1, 2).float() / 255
tf_ms = time_ms(lambda: oracle_features(n32, img), a.reps)
row_tf = dict(gpu=gpu, row="torch_tf32", batch=B, cudnn_allow_tf32=torch.backends.cudnn.allow_tf32, ms=round(tf_ms, 3),
              img_per_s=round(B / tf_ms * 1e3, 1))
print(json.dumps(row_tf), flush=True)
if a.out:
    with open(a.out, "w") as f:
        json.dump([row_fwd, row_fr, row_rec, row_tf], f, indent=1)
