"""Isolates the GEMM epilogue / store path: tiny-K contractions whose time is all output traffic, next to plain device
memset / copy bandwidth on the same box (the denominators for the store-bound kernels: mask-embed, K=256 encoder linears)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from hipie_b200 import _lib, ops

dev = torch.device("cuda:0")


def timeit(fn, n=10):
    for _ in range(3):
        fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / n


buf = torch.empty(2 * 1024 ** 3 // 4, device=dev)
src = torch.empty_like(buf)
ms = timeit(lambda: buf.zero_())
print(f"memset 2 GiB: {ms:.3f} ms  {buf.numel()*4/ms/1e6:.0f} GB/s (write only)")
ms = timeit(lambda: buf.copy_(src))
print(f"copy   2 GiB: {ms:.3f} ms  {2*buf.numel()*4/ms/1e6:.0f} GB/s (read+write)")
ms = timeit(lambda: torch.sum(src))
print(f"read   2 GiB: {ms:.3f} ms  {buf.numel()*4/ms/1e6:.0f} GB/s (read only)")
del buf, src
for (M, N, K) in [(174080, 2048, 32), (174080, 2048, 256), (174080, 256, 256), (8 * 300, 65536, 256)]:
    a = torch.randn(M, K, device=dev)
    w = torch.randn(N, K, device=dev) * 0.05
    A, W = ops.split(a), ops.split_weight(w)
    for name, kw, obytes in [("f32", dict(), 4), ("planes", dict(want_f32=False, want_split=True), 4), ("hi only", dict(want_f32=False, want_split=True, prec=1), 2),
                             ("f32+planes", dict(want_split=True), 8)]:
        prec = kw.pop("prec", 3)
        ops.set_precision(prec)
        ms = timeit(lambda: ops.gemm(A, W, prec=prec, **kw))
        ops.set_precision(3)
        print(f"gemm {M}x{N}x{K} out={name:10s} prec{prec}: {ms:.3f} ms  out {M*N*obytes/ms/1e6:.0f} GB/s  ({2.0*M*N*K/ms/1e9:.0f} TF alg)", flush=True)
