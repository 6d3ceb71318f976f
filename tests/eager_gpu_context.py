"""NOT a test (not collected): context number for DESIGN.md — the reference ALGORITHM as eager PyTorch on the same H100.

The reference is pure PyTorch (SURVEY.md §0: "the bar on the GPU is PyTorch eager on the same H100"): this script runs the
3-objective step of oracle/train_step.py — the reference's towers restated functionally + the restated losses + autograd +
torch.optim.AdamW + EMA — on `cuda` under `torch.autocast(bfloat16)` with `F.scaled_dot_product_attention` (flash) for the
attention, i.e. what a user gets from the reference's modules on this GPU: cuBLAS / cuDNN / SDPA kernels, one launch per
op.  It lives under tests/ because it executes oracle/ (test infrastructure); nothing in the product imports it.

    python tests/eager_gpu_context.py [--model small] [--batches 32,64,128] [--steps 3]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import torch.nn.functional as F

from oracle import vtp_oracle as vo
from oracle.train_step import OracleTrainer
from vtp_b200.config import preset
from vtp_b200.lpips import random_weights
from vtp_b200.model import VTPModel
from vtp_b200.synthetic import make_batch

ap = argparse.ArgumentParser()
ap.add_argument("--model", default="small")
ap.add_argument("--batches", default="32,64,128")
ap.add_argument("--steps", type=int, default=3)
ap.add_argument("--prototypes", type=int, default=65536)
ap.add_argument("--device", default="cuda", help="cpu only for a dry run of this script")
a = ap.parse_args()
DEV = a.device

cfg = preset(a.model)
sd_cpu = {k: v.detach().clone() for k, v in VTPModel(cfg).state_dict().items()}
lp_cpu = random_weights(0)                 # CPU generator: before the default device changes
torch.set_default_device(DEV)          # every tensor the oracle creates (arange, zeros, ...) lands on the GPU
vo.sdpa = lambda q, k, v, mode, causal=False: F.scaled_dot_product_attention(q, k, v, is_causal=causal)   # flash SDPA
sd = {k: v.to(DEV) for k, v in sd_cpu.items()}
K, D = a.prototypes, cfg.vision_embed_dim
g = torch.Generator(device=DEV).manual_seed(0)
hsd = {"mlp.0.weight": torch.randn(2048, D, generator=g) * 0.02, "mlp.0.bias": torch.zeros(2048),
       "mlp.2.weight": torch.randn(2048, 2048, generator=g) * 0.02, "mlp.2.bias": torch.zeros(2048),
       "mlp.4.weight": torch.randn(256, 2048, generator=g) * 0.02, "mlp.4.bias": torch.zeros(256),
       "last_layer.weight_g": torch.ones(K, 1), "last_layer.weight_v": torch.randn(K, 256, generator=g) * 0.02}
dims = dict(vision_depth=cfg.vision_depth, vision_num_heads=cfg.vision_num_heads, text_depth=cfg.text_depth,
            text_num_heads=cfg.text_num_heads, decoder_depth=cfg.decoder_depth, decoder_num_heads=cfg.decoder_num_heads)
lp = tuple([t.to(DEV) for t in part] for part in lp_cpu)
rows = []
for B in [int(b) for b in a.batches.split(",")]:
    try:
        tr = OracleTrainer(sd, hsd, dims, n_local=8, mode="fp32", lpips=lp)
        torch.set_default_device("cpu")
        batch = make_batch(B, vocab=cfg.text_vocab_size)
        torch.set_default_device(DEV)
        batch = {k: v.to(DEV) for k, v in batch.items()}
        with torch.autocast(DEV, dtype=torch.bfloat16):
            tr.step(batch)                      # warm-up (cuDNN autotune, allocator)
            if DEV == "cuda":
                torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.steps):
                losses = tr.step(batch)         # float(loss) inside synchronises every step
            if DEV == "cuda":
                torch.cuda.synchronize()
        dt = (time.perf_counter() - t0) / a.steps
        rows.append({"batch": B, "ms_per_step": dt * 1e3, "img_per_s": B / dt, "peak_mem_GiB": (torch.cuda.max_memory_allocated() / 2**30 if DEV == "cuda" else 0.0),
                     "loss": {k: round(v, 4) for k, v in losses.items()}})
        print(f"eager PyTorch (autocast bf16, SDPA) {a.model} batch {B}: {dt * 1e3:.1f} ms/step = {B / dt:.1f} img/s, "
              f"peak {rows[-1]['peak_mem_GiB']:.1f} GiB", flush=True)
        del tr, batch
        if DEV == "cuda":
            torch.cuda.empty_cache()
    except torch.OutOfMemoryError:
        print(f"batch {B}: out of memory", flush=True)
        torch.cuda.empty_cache()
        break
print(json.dumps({"model": a.model, "what": "oracle/train_step.py on cuda, torch.autocast(bf16), F.scaled_dot_product_attention, "
                  "torch.optim.AdamW; same crops / prototypes / losses (incl. LPIPS) as bench.py", "rows": rows}))
