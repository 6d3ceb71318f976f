"""Achieved HBM bandwidth of the memory-bound kernels of the hot path at the bench workload's shapes (VTP-Small, 256
images/GPU -> M = 131 584 token rows of the SSL student pass), CUDA-event timed on the launching stream, against the
measured copy bandwidth in MEASURED_PEAKS.json.  Every working set exceeds the 126 MB L2, so no flush is needed.

  python tools/hbm_kernels_bench.py [--out /tmp/hbm_kernels.json]

`bytes` = ALGORITHMIC bytes (each tensor read or written once), so GB/s is a lower bound of the DRAM rate."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from vtp_b200 import lib

BF, F32 = torch.bfloat16, torch.float32
ap = argparse.ArgumentParser()
ap.add_argument("--out", default="/tmp/hbm_kernels.json")
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--once", action="store_true", help="launch every kernel once, no timing (for ncu --set full)")
a = ap.parse_args()
dev = "cuda"
peak = 6562.6
try:
    with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")) as f:
        peak = json.load(f)["hbm_gbs"]
except Exception:
    pass

M, D, Hs = 2 * 256 * 257, 384, 1024
rows = []


def timeit(name, fn, nbytes, note=""):
    try:
        _timeit(name, fn, nbytes, note)
    except Exception as e:  # keep going: one bad call must not lose the other rows
        rows.append({"kernel": name, "error": str(e)[:200]})
        print(f"{name:34s} FAILED: {e}", flush=True)


def _timeit(name, fn, nbytes, note=""):
    if a.once:
        fn()
        torch.cuda.synchronize()
        return
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(a.reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / a.reps * 1e3
    gbs = nbytes / us / 1e3
    rows.append({"kernel": name, "us": round(us, 2), "bytes": int(nbytes), "GBps": round(gbs, 1), "frac_of_peak": round(gbs / peak, 3),
                 "note": note})
    print(f"{name:34s} {us:9.1f} us  {nbytes / 1e6:9.1f} MB  {gbs:8.1f} GB/s  {gbs / peak:6.1%}  {note}", flush=True)


x32 = torch.randn(M, D, device=dev)
w = torch.ones(D, device=dev)
bln = torch.zeros(D, device=dev)
ybf = torch.empty(M, D, dtype=BF, device=dev)
rstd = torch.empty(M, device=dev)
mean = torch.empty(M, device=dev)
timeit("norm_fwd rms fp32->bf16", lambda: lib.norm_fwd(x32, ybf, w, None, 1e-5, M, D, y_mode=lib.OUT_BF16, rstd=rstd),
       M * D * 6, "layers/normalization.py:17-22")
timeit("norm_fwd ln fp32->bf16", lambda: lib.norm_fwd(x32, ybf, w, bln, 1e-6, M, D, y_mode=lib.OUT_BF16, rstd=rstd, mean=mean),
       M * D * 6)
g = torch.zeros(M, D, device=dev)
dy = torch.randn(M, D, device=dev).to(BF)
dw, db = torch.zeros(D, device=dev), torch.zeros(D, device=dev)
gb = torch.empty(M, D, dtype=BF, device=dev)
cs = torch.zeros(D, device=dev)
timeit("norm_bwd rms (+gb, colsum)", lambda: lib.norm_bwd(x32, rstd, None, w, dy, g, dw, None, M, D, gb_out=gb, g_colsum=cs),
       M * D * (4 + 2 + 4 + 4 + 2), "x, dy read; g read+write; bf16 copy written")
pre = torch.randn(M, 2 * Hs, device=dev).to(BF)
hid = torch.empty(M, Hs, dtype=BF, device=dev)
timeit("swiglu_fwd", lambda: lib.swiglu_fwd(pre, hid, M, Hs), M * Hs * 6, "layers/ffn.py:77-81")
dhid = torch.randn(M, Hs, device=dev).to(BF)
dpre = torch.empty_like(pre)
dbias = torch.zeros(2 * Hs, device=dev)
timeit("swiglu_bwd (+bias grad)", lambda: lib.swiglu_bwd(pre, dhid, dpre, dbias, M, Hs), M * Hs * 10)
qkv = torch.randn(M, 3 * D, device=dev).to(BF)
from vtp_b200.rope import rope_periods, rope_sincos
sin, cos = rope_sincos(16, 16, rope_periods(64).to(BF))
sin, cos = sin.to(dev).contiguous(), cos.to(dev).contiguous()
timeit("rope_fwd (q,k in place)", lambda: lib.rope_fwd(qkv, sin, cos, M, 257, 1, D), M * 2 * D * 4, "layers/attention.py:70-89")
cs3 = torch.zeros(3 * D, device=dev)
timeit("cast_colsum bf16 [M,3D]", lambda: lib.cast_colsum(qkv, None, cs3, M, 3 * D), M * 3 * D * 2)
img = torch.randn(512, 3, 256, 256, device=dev)
col = torch.empty(512 * 256, 768, dtype=BF, device=dev)
timeit("patchify 512x3x256x256", lambda: lib.patchify(img, col, 16), img.numel() * 6, "layers/embeddings.py:61-70 input side")
n = 100_000_000
p, gg, m1, v1 = (torch.zeros(n, device=dev) for _ in range(4))
pb = torch.zeros(n, dtype=BF, device=dev)
tp, tpb = torch.zeros(n, device=dev), torch.zeros(n, dtype=BF, device=dev)
timeit("adamw + bf16 copy + EMA teacher", lambda: lib.adamw_step(p, gg, m1, v1, pb, tp, tpb, n, lr=1e-4, beta1=0.9, beta2=0.95,
                                                                  eps=1e-8, wd=0.05, step=1, ema_momentum=0.994),
       n * (4 * 4 * 2 - 4 + 2 + 4 * 2 + 2), "p,m,v r/w; g read+zeroed; bf16 copies; teacher r/w")
del p, gg, m1, v1, pb, tp, tpb
# DINO / iBOT loss kernels at the bench shape: K = 65 536 prototypes, rows = cls + masked-patch tokens of 256 source images
K, Rt = 65536, 4096
tl = (torch.randn(Rt, K, device=dev) * 2).to(BF)
center = torch.zeros(K, device=dev)
timeit("dino_teacher_probs [4096, 65536]", lambda: lib.dino_teacher_probs(tl, center, Rt, K, 0.07), Rt * K * 4,
       "centred + sharpened teacher softmax, in place")
sl = (torch.randn(Rt, K, device=dev) * 2).to(BF)
t0 = torch.arange(Rt, device=dev, dtype=torch.int32)
t1 = torch.full((Rt,), -1, device=dev, dtype=torch.int32)
wrow = torch.full((Rt,), 1.0 / Rt, device=dev)
lacc = torch.zeros(1, device=dev)
timeit("dino_student_ce [4096, 65536]", lambda: lib.dino_student_ce(sl, tl, t0, t1, wrow, Rt, K, 0.1, lacc), Rt * K * 6,
       "student log-softmax CE + gradient in place, one teacher row each")
del tl, sl
rec = torch.randn(256, 3, 256, 256, device=dev)
u8 = torch.empty(256, 256, 256, 3, dtype=torch.uint8, device=dev)
sub = torch.tensor([-2.1179, -2.0357, -1.8044], device=dev)
div = torch.tensor([4.3668, 4.4643, 4.4444], device=dev)
timeit("image_to_u8 256x3x256x256", lambda: lib.image_to_u8(rec, sub, div, u8), rec.numel() * 5, "vtp_tokenizer.py:106-119")
# GEMMs whose roofline is HBM (SURVEY §8d): bottleneck D->64 and proj_out + PixelShuffle store
xn = torch.randn(M, D, device=dev).to(BF)
wb = torch.randn(64, D, device=dev).to(BF)
tok = torch.empty(256 * 2 * 256, 64, dtype=BF, device=dev)
timeit("GEMM bottleneck N=64 (+cls drop)", lambda: lib.gemm(xn, wb, tok, M=M, N=64, K=D, rr_group=257, rr_skip=-1),
       M * D * 2 + tok.numel() * 2, "vision_transformer_bottleneck.py:66-79")
Md = 256 * 256
xd = torch.randn(Md, D, device=dev).to(BF)
wo = torch.randn(768, D, device=dev).to(BF)
bo = torch.zeros(768, device=dev)
out_img = torch.empty(256, 3, 256, 256, dtype=BF, device=dev)
timeit("GEMM proj_out + PixelShuffle bf16", lambda: lib.gemm(xd, wo, out_img, M=Md, N=768, K=D, bias=bo, pixel_shuffle=(16, 16, 16, 3),
                                                            ldo=256),
       Md * D * 2 + out_img.numel() * 2, "pixel_decoder.py:157-160")
os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
with open(a.out, "w") as f:
    json.dump({"peak_GBps": peak, "peak_source": "MEASURED_PEAKS.json hbm_gbs (copy read+write)", "M": M, "D": D, "rows": rows}, f, indent=1)
