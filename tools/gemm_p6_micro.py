"""Times the ViT-H GEMMs of the headline step as the engine calls them: the fp16 + e4m3 split (prec 6) on proj / fc1 / fc2 and
the encoder FFNs, the two-pass fp16 mode (prec 4) on the qk linear, and a K sweep of prec 6 at M = 32768, N = 5120 fitted to
time = a + b K (a: what does not overlap the mainloop -- epilogue, pipeline fill; b: the mainloop rate).
One launch per sample after a 256 MB L2 flush, median of 7 samples after 2 warm-up launches; TFLOP/s are algorithmic (2 M N K).
Prints the card name, power limit and SM clocks first: the numbers mean nothing without them.
Usage: python tools/gemm_p6_micro.py [repo root whose hipie_b200 to time; default: this tool's tree]"""
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.abspath(sys.argv[1]) if len(sys.argv) > 1 else os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from hipie_b200 import ops  # noqa: E402

dev = torch.device("cuda:0")
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name(dev)


def timed(fn):
    for _ in range(2):
        fn()
    ts = []
    for _ in range(7):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); fn(); e.record(); torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    return sorted(ts)[len(ts) // 2]


def window_map(B=8, g=64, ws=14):
    """Rows of the 14 x 14 window layout (B x 25 windows x 196) -> token rows (B x 4096); -1 for the pad tokens of the 70 x 70 grid."""
    gp = (g + ws - 1) // ws * ws
    nw = gp // ws
    rm = torch.full((B, nw, nw, ws, ws), -1, dtype=torch.int32)
    y = torch.arange(gp).view(nw, 1, ws, 1).expand(nw, nw, ws, ws)
    x = torch.arange(gp).view(1, nw, 1, ws).expand(nw, nw, ws, ws)
    ok = (y < g) & (x < g)
    for b in range(B):
        rm[b][ok] = (b * g * g + y * g + x)[ok].int()
    return rm.reshape(-1).to(dev), B * g * g


def p6(M, N, K, **kw):
    g = torch.Generator(device="cuda").manual_seed(0)
    A = ops.split_f16_e4m3(torch.randn(M, K, device=dev, generator=g))
    W = ops.split_f16_e4m3(torch.randn(N, K, device=dev, generator=g) * 0.05, weight=True)
    return A, W, torch.randn(N, device=dev, generator=g) * 0.1


def main():
    print(f"card: {card()}")
    print(f"tree: {ROOT}")
    rows = []
    for name, M, N, K, mode in (("vit fc1 gelu->planes", 32768, 5120, 1280, "planes"),
                                ("vit fc2 +res", 32768, 1280, 5120, "res"),
                                ("vit proj +res", 32768, 1280, 1280, "res"),
                                ("vit proj win +res map", 39200, 1280, 1280, "map"),
                                ("enc ffn1 relu->planes", 174080, 2048, 256, "planes_relu"),
                                ("enc ffn2 +res", 174080, 256, 2048, "res")):
        A, W, bias = p6(M, N, K)
        if mode.startswith("planes"):
            act = ops.ACT_GELU if mode == "planes" else ops.ACT_RELU
            fn = lambda: ops.gemm(A, W, bias=bias, act=act, want_f32=False, out_e4m3=True, prec=6)
        elif mode == "res":
            x = torch.randn(M, N, device=dev)
            fn = lambda: ops.gemm(A, W, bias=bias, residual=x, out_f32=x, prec=6)
        else:
            rm, rows_out = window_map()
            x = torch.randn(rows_out, N, device=dev)
            fn = lambda: ops.gemm(A, W, bias=bias, residual=x, out_f32=x, row_map=rm, out_rows=rows_out, prec=6)
        rows.append((f"p6 {name}", M, N, K, timed(fn)))
        del A, W
    # qk of the fp16 attention mode: A one fp16 plane (the LayerNorm output), W fp16 hi + lo, output one fp16 plane
    g = torch.Generator(device="cuda").manual_seed(0)
    M, N, K = 32768, 2560, 1280
    a16 = ops.BF2(torch.randn(M, K, device=dev, generator=g).half(), None)
    w4 = ops.split_weight_f16(torch.randn(N, K, device=dev, generator=g) * 0.05)
    bias = torch.randn(N, device=dev, generator=g) * 0.1
    rows.append(("p4 vit qk ->fp16", M, N, K, timed(lambda: ops.gemm(a16, w4, bias=bias, want_f32=False, want_split=True, out_fp16=True, prec=4))))
    for name, M, N, K, ms in rows:
        print(f"{name:26s} {M:6d} x {N:5d} x {K:5d}  {ms * 1000:8.1f} us  {2.0 * M * N * K / ms / 1e9:6.1f} TFLOP/s", flush=True)
    # K sweep: fc1's output (GELU -> fp16 + e4m3 planes) at N = 5120
    M, N = 32768, 5120
    ks, ts = [640, 1280, 2560, 5120], []
    for K in ks:
        A, W, bias = p6(M, N, K)
        ts.append(timed(lambda: ops.gemm(A, W, bias=bias, act=ops.ACT_GELU, want_f32=False, out_e4m3=True, prec=6)))
        print(f"p6 K sweep {M} x {N} x {K:5d}  {ts[-1] * 1000:8.1f} us  {2.0 * M * N * K / ts[-1] / 1e9:6.1f} TFLOP/s", flush=True)
        del A, W
    b, a = np.polyfit(np.array(ks, dtype=np.float64), np.array(ts, dtype=np.float64), 1)
    print(f"p6 K sweep fit: time = {a * 1000:.1f} us + K x {b * 1000:.4f} us  (mainloop {2.0 * M * N / b / 1e9:.1f} TFLOP/s)")


if __name__ == "__main__":
    main()
