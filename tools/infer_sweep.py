"""Config 5 of BASELINE.json: encode+decode inference throughput sweep (bf16 autocast mode).  GPU only.  (Latents parity
against the reference lives in tests/test_model_gpu.py — tools never touch oracle/.)
  python tools/infer_sweep.py --model large --batches 1,8,64,256 [--graphs] [--image-size 512]
--graphs also times CUDA-graph replays (VTPModel.enable_cuda_graphs) — the small-batch serving path.
--image-size N (a multiple of 16, default 256) times N x N images and adds the card's name and power limit, read in
the same run, to the JSON line."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from vtp_b200.config import preset
from vtp_b200.flops import encode_decode_flops
from vtp_b200.model import VTPModel

ap = argparse.ArgumentParser()
ap.add_argument("--model", default="large")
ap.add_argument("--batches", default="1,8,64,256")
ap.add_argument("--graphs", action="store_true")
ap.add_argument("--image-size", type=int, default=256)
a = ap.parse_args()
cfg = preset(a.model)
torch.manual_seed(0)
m = VTPModel(cfg).cuda()
fl = encode_decode_flops(cfg, a.image_size)
out = {"model": a.model, "gflop_per_image": fl / 1e9, "rows": []}
if a.image_size != 256:
    import subprocess

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.splitlines()
    out.update(image_size=a.image_size, gpu=q[torch.cuda.current_device()].strip() if q else torch.cuda.get_device_name())
for B in [int(b) for b in a.batches.split(",")]:
    x = torch.randn(B, 3, a.image_size, a.image_size, device="cuda")
    with torch.autocast("cuda", dtype=torch.bfloat16):
        for _ in range(3):
            rec = m.get_latents_decoded_images(m.get_reconstruction_latents(x))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 10 if B >= 8 else 30
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            rec = m.get_latents_decoded_images(m.get_reconstruction_latents(x))
        e1.record()
        torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    row = {"batch": B, "ms": ms, "img_per_s": B / ms * 1e3, "tflops": fl * B / ms / 1e9}
    if a.graphs:
        m.enable_cuda_graphs()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            for _ in range(2):
                rec_g = m.get_latents_decoded_images(m.get_reconstruction_latents(x))
            torch.cuda.synchronize()
            e0.record()
            for _ in range(reps):
                rec_g = m.get_latents_decoded_images(m.get_reconstruction_latents(x))
            e1.record()
            torch.cuda.synchronize()
        m.enable_cuda_graphs(False)
        row["ms_graphs"] = e0.elapsed_time(e1) / reps
        row["graphs_equal_eager"] = bool(torch.equal(rec_g, rec))
    out["rows"].append(row)
    print(f"{a.model} B={B:4d}: {ms:8.2f} ms  {B / ms * 1e3:9.1f} img/s  {fl * B / ms / 1e9:7.1f} TFLOP/s"
          + (f"   graphs: {row['ms_graphs']:8.2f} ms" if a.graphs else ""), flush=True)
print(json.dumps(out))
