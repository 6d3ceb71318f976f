"""Reconstruction evaluation (vtp_b200/recon_eval.py) at the reference's evaluation shape: 256x256 images, batch 50 per
GPU, VTP-S and VTP-L with seeded random weights, bf16 encoder and fp32 decoder, LPIPS with seeded random VGG16 / lin
weights (the same shapes and FLOPs as the released ones).  GPU only; CUDA-event timing on the launching stream.

  python tools/recon_eval_bench.py [--out /tmp/recon.json] [--models s,l] [--reps 10]

Rows per model:
  encdec_ms     encode (bf16) + decode (fp32), eager launches
  metrics_ms    kernels 1-3 (vtp_recon_pixels with uint8 and LPIPS-input outputs, vtp_recon_ssim, vtp_recon_finalise)
  metrics_TBps  their HBM bytes over their time: per value of the 3·H·W·B pixel grid, the pixel pass reads 4 + 4 B and
                writes 2 + 8 B, the SSIM pass reads 4 + 4 B (halo re-reads are counted once), against 3.35 TB/s
  lpips_ms      LPIPSMetric on the batch (both images of every pair through VGG16, bf16x3 convolutions)
  step_ms       ReconstructionEvaluator.add by CUDA-graph replay without / with LPIPS (no PNGs); img/s = B / step
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from vtp_b200 import lib
from vtp_b200.config import preset
from vtp_b200.lpips import LPIPSMetric
from vtp_b200.model import VTPModel
from vtp_b200.recon_eval import ReconstructionEvaluator

ap = argparse.ArgumentParser()
ap.add_argument("--out", default=None)
ap.add_argument("--models", default="s,l")
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--batch", type=int, default=50)
ap.add_argument("--size", type=int, default=256)
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


B, S = a.batch, a.size
lp_metric = LPIPSMetric.random_init(0)
rows = []
for name in a.models.split(","):
    cfg = preset(name, train_clip=False)
    torch.manual_seed(0)
    m = VTPModel(cfg).cuda().eval()
    x = torch.randn(B, 3, S, S, device="cuda")

    def encdec():
        m.compute_mode = "bf16"
        lat = m.get_reconstruction_latents(x)
        m.compute_mode = "fp32"
        return m.get_latents_decoded_images(lat)

    encdec_ms = time_ms(encdec, a.reps)
    rec = encdec().contiguous()
    m.compute_mode = None
    ev = ReconstructionEvaluator(m, lpips=lp_metric)
    sub, div = ev.sub, ev.div
    sse = torch.empty(B, 16, dtype=torch.float64, device="cuda")
    part = torch.empty(B, lib.recon_ssim_tiles(S, S), dtype=torch.float64, device="cuda")
    u8 = torch.empty(2, B, S, S, 3, dtype=torch.uint8, device="cuda")
    lp = torch.empty(B, 2, 3, S, S, device="cuda")
    ps, ss = torch.empty(B, dtype=torch.float64, device="cuda"), torch.empty(B, device="cuda")
    acc = torch.zeros(8, dtype=torch.float64, device="cuda")

    def metrics():
        lib.recon_pixels(x, rec, sub, div, sse, u8_ref=u8[0], u8_rec=u8[1], lp=lp)
        lib.recon_ssim(x, rec, sub, div, part)
        lib.recon_finalise(sse, part, None, S, S, ps, ss, None, acc)

    metrics_ms = time_ms(metrics, 10 * a.reps)
    nbytes = 3 * S * S * B * (4 + 4 + 2 + 8 + 4 + 4)
    lpips_ms = time_ms(lambda: lp_metric.parts(lp), a.reps)
    ev_plain = ReconstructionEvaluator(m, lpips=None)
    step_plain = time_ms(lambda: ev_plain.add(x), a.reps)
    step_lp = time_ms(lambda: ev.add(x), a.reps)
    ev_plain.close()
    ev.close()
    row = dict(model=name, gpu=gpu, batch=B, image=S, encdec_ms=round(encdec_ms, 3),
               encdec_img_per_s=round(B / encdec_ms * 1e3, 1), metrics_ms=round(metrics_ms, 4),
               metrics_TBps=round(nbytes / metrics_ms / 1e9, 3), metrics_share_of_3p35=round(nbytes / metrics_ms / 1e9 / 3.35, 3),
               lpips_ms=round(lpips_ms, 3), step_ms=round(step_plain, 3), img_per_s=round(B / step_plain * 1e3, 1),
               step_lpips_ms=round(step_lp, 3), img_per_s_lpips=round(B / step_lp * 1e3, 1))
    print(json.dumps(row), flush=True)
    rows.append(row)
    del m, ev, ev_plain
    torch.cuda.empty_cache()
if a.out:
    with open(a.out, "w") as f:
        json.dump(rows, f, indent=1)
