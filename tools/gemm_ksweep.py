"""Dev tool: the GEMM's fixed cost per output tile, from a sweep over K at fixed M x N (GPU only).

The persistent GEMM gives each SM ceil(tiles / SMs) tiles one after another, so a launch takes `waves` tile times.  Timing
`lib.gemm` at several K and fitting the time per tile-wave as  a + b*K  separates what every tile costs whatever its K
(intercept a: pipeline fill, accumulator hand-off, epilogue that the mainloop does not hide) from the mainloop's own rate
(slope b -> 2*128*BN*SMs / b FLOP/s).  Shapes: the bench.py roofline call (FFN fc1, M = 131 584, N = 2048, bias, bf16
out), the same M at N = 384 (proj / fc2 dgrad width), and one LPIPS layer (conv2_1: 32 images, 128 x 128, 128 output
channels, bias + ReLU, implicit 3x3 conv; K = 9 * C_in).
  python tools/gemm_ksweep.py [--out ksweep.json]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from vtp_b200 import lib

BF = torch.bfloat16
BM = 128


def card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:  # the card name from torch is still recorded
        q = f"nvidia-smi unavailable ({e})"
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": q}


def time_ms(fn, warmup=3, reps=20) -> float:
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def fit(ks, ts):
    n = len(ks)
    mk, mt = sum(ks) / n, sum(ts) / n
    b = sum((k - mk) * (t - mt) for k, t in zip(ks, ts)) / sum((k - mk) ** 2 for k in ks)
    return mt - b * mk, b


def sweep(name, run, M, N, ks, nsm):
    """run(K) -> a callable doing one launch at that K.  Returns the per-K table and the a + b*K fit (microseconds)."""
    BN = 64 if N <= 64 else 128
    tiles = -(-M // BM) * -(-N // BN)
    waves = -(-tiles // nsm)
    rows = []
    for K in ks:
        ms = time_ms(run(K))
        rows.append({"K": K, "ms": ms, "us_per_wave": ms * 1e3 / waves, "tflops": 2.0 * M * N * K / (ms * 1e-3) / 1e12})
    a, b = fit([r["K"] for r in rows], [r["us_per_wave"] for r in rows])
    res = {"shape": name, "M": M, "N": N, "BN": BN, "tiles": tiles, "waves": waves, "rows": rows, "a_us": a, "b_us_per_k": b,
           "mainloop_tflops": 2.0 * BM * BN * nsm / (b * 1e-6) / 1e12}
    for r in rows:
        r["a_share"] = a / r["us_per_wave"]
    print(f"\n{name}: M={M} N={N} BN={BN} tiles={tiles} waves={waves}")
    print("|   K |     ms | us/wave | TFLOP/s | a / tile time |\n|---:|---:|---:|---:|---:|")
    for r in rows:
        print(f"| {r['K']:4d} | {r['ms']:6.3f} | {r['us_per_wave']:7.3f} | {r['tflops']:7.1f} | {100 * r['a_share']:5.1f} % |")
    print(f"fit: a = {a:.3f} us per tile, b = {b * 1e3:.3f} ns per unit K  ->  mainloop {res['mainloop_tflops']:.0f} TFLOP/s")
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda")
    nsm = torch.cuda.get_device_properties(dev).multi_processor_count
    info = card()
    print(f"{info['device']} | {info['nvidia_smi']} | {nsm} SMs")
    g = torch.Generator(device=dev).manual_seed(0)
    results = []
    M = 2 * 256 * 257  # fc1 rows of the SSL student pass at batch 256 (bench.py roofline call)
    kmax = 3072
    A = torch.randn(M, kmax, device=dev, generator=g).to(BF)
    for N in (2048, 384):
        W = torch.randn(N, kmax, device=dev, generator=g).to(BF)
        bias = torch.zeros(N, device=dev)
        out = torch.empty(M, N, device=dev, dtype=BF)
        run = lambda K: (lambda: lib.gemm(A, W, out, M=M, N=N, K=K, lda=kmax, ldb=kmax, bias=bias))
        results.append(sweep(f"linear N={N}", run, M, N, [64, 128, 384, 768, 1536, 3072], nsm))
        del W, out
    del A
    Bimg, hw, co = 32, 128, 128  # LPIPS conv2_1 (C_in = 64 there); C_in swept to vary K = 9 * C_in
    Mc = Bimg * hw * hw
    y = torch.empty(Bimg, hw, hw, co, device=dev, dtype=BF)
    bias = torch.zeros(co, device=dev)
    xs = {ci: torch.randn(Bimg, hw, hw, ci, device=dev, generator=g).to(BF) for ci in (64, 128, 256, 512)}
    ws = {ci: (torch.randn(co, 9 * ci, device=dev, generator=g) * 0.05).to(BF) for ci in xs}
    run = lambda K: (lambda: lib.gemm(xs[K // 9], ws[K // 9], y, M=Mc, N=co, K=K, lda=K // 9, ldb=K, bias=bias,
                                      act=lib.ACT_RELU, ldo=co, conv=(K // 9, hw, hw)))
    results.append(sweep(f"conv3x3 {Bimg}x{hw}x{hw} -> {co} (bias+ReLU)", run, Mc, co, [9 * c for c in xs], nsm))
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": info, "sms": nsm, "sweeps": results}, f, indent=1)


if __name__ == "__main__":
    main()
