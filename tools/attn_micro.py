"""Times hipie_attention_tc at the three shapes the ViT-H blocks run, as the engine calls it (fp16 q / k / v^T planes, output as
the fp16 + e4m3 planes of the proj GEMM), plus the bf16x3 mode at the global shape:
  global 64-wide grid (1024^2 inputs): B 8, 16 heads, T 4096
  80-wide grid (1280^2 inputs):        B 8, 16 heads, T 6400
  14 x 14 windows:                     B 200 windows, 16 heads, T 196
CUDA events around 10 launches, median of 5 such windows after 3 warm-up launches; TFLOP/s are algorithmic (4 B H T^2 hd).
Prints the card name, power limit and SM clocks first: the numbers mean nothing without them.
Usage: python tools/attn_micro.py [repo root whose hipie_b200 to time; default: this tool's tree]"""
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.abspath(sys.argv[1]) if len(sys.argv) > 1 else os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from hipie_b200 import ops  # noqa: E402

dev = torch.device("cuda:0")
H, hd = 16, 80
E = H * hd


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name(dev)


def inputs(B, T, gh, gw, win):
    g = torch.Generator(device="cuda").manual_seed(0)
    qk = torch.randn(B * T, 2 * E, device=dev, generator=g)
    v = torch.randn(B * T, E, device=dev, generator=g)
    if win:
        vt = torch.zeros(E, B, 200, device=dev)
        vt[:, :, :T] = v.t().reshape(E, B, T)
        vt = vt.view(E, B * 200)
    else:
        vt = v.t().contiguous()
    rel = dict(rel_h=torch.randn(B, H, T, gh, device=dev, generator=g), rel_w=torch.randn(B, H, T, gw, device=dev, generator=g),
               kh=gh, kw=gw)
    return qk, vt, rel


def time_ms(fn):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    runs = []
    for _ in range(5):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(10):
            fn()
        e.record()
        torch.cuda.synchronize()
        runs.append(s.elapsed_time(e) / 10)
    return statistics.median(runs)


def main():
    print(f"card: {card()}")
    print(f"tree: {ROOT}")
    for name, B, gh, gw, win in (("global 64-wide", 8, 64, 64, False), ("80-wide", 8, 80, 80, False), ("window 14x14", 200, 14, 14, True)):
        T = gh * gw
        qk, vt, rel = inputs(B, T, gh, gw, win)
        args = (B, H, T, hd, T * 2 * E, 2 * E, T * 2 * E, 2 * E, hd ** -0.5)
        flops = 4.0 * B * H * T * T * hd
        qk16, vt16 = qk.half(), vt.half()
        q, k, v = ops.BF2(qk16[:, :E], None), ops.BF2(qk16[:, E:], None), ops.BF2(vt16, None)
        ms = time_ms(lambda: ops.attention_tc(q, k, v, *args, out_e4m3=True, f16=True, **rel))
        print(f"{name:15s} B {B:3d} T {T:5d}  f16x1 -> fp16+e4m3 planes: {ms:8.3f} ms  {flops / ms / 1e9:6.1f} TFLOP/s")
        if not win and gw == 64:
            S, Vs = ops.split(qk), ops.split(vt)
            q3, k3 = ops.BF2(S.hi[:, :E], S.lo[:, :E]), ops.BF2(S.hi[:, E:], S.lo[:, E:])
            ms = time_ms(lambda: ops.attention_tc(q3, k3, Vs, *args, prec=3, **rel))
            print(f"{name:15s} B {B:3d} T {T:5d}  bf16x3 -> bf16 hi/lo:         {ms:8.3f} ms  {flops / ms / 1e9:6.1f} TFLOP/s")
        del qk, vt, rel, qk16, vt16
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
