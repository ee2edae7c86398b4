"""GPU smoke + A/B of the GEMM epilogue variants (run under `timeout`): the TMA-store epilogue against the register-store
epilogue.  Exit code 0 = every variant reproduces the baseline bit for bit on every
case and agrees with an fp64 reference."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from hipie_b200 import _lib, ops

torch.manual_seed(0)
dev = torch.device("cuda:0")
ok = True
VARIANTS = [0, 1]       # tma_store; the first is the baseline


def setv(tma):
    _lib.set_option("gemm_tma_store", tma)


cases = [(1024, 256, 256, {}), (4096, 1280, 1280, dict(act=ops.ACT_GELU, want_split=True)), (2048 + 64, 384, 512, {}),
         (1500, 136, 264, dict(want_split=True)), (1500, 130, 264, {}), (8192, 128, 256, dict(want_split=True, want_f32=False)),
         (4096, 640, 1280, dict(transposed=True, want_split=True, want_f32=False)), (32768, 1280, 1280, dict(res=True)),
         (300, 4096, 256, dict(bits_threshold=0.0)), (2400, 2048, 256, dict(act=ops.ACT_RELU, want_split=True, want_f32=False, cs=True)),
         (777, 96, 64, dict(act=ops.ACT_RELU))]
for prec in (3, 1):
    for M, N, K, kw in cases:
        a = torch.randn(M, K, device=dev)
        w = torch.randn(N, K, device=dev) * 0.05
        bias = torch.randn(N, device=dev)
        ops.set_precision(prec)
        A, W = ops.split(a), ops.split_weight(w)
        kw = dict(kw)
        res = torch.randn(M, N, device=dev) if kw.pop("res", False) else None
        cs = torch.rand(N, device=dev) + 0.5 if kw.pop("cs", False) else None
        outs = []
        for tma in VARIANTS:
            setv(tma)
            f, s, bits = ops.gemm(A, W, prec=prec, bias=bias, residual=res, colscale=cs, **kw)
            torch.cuda.synchronize()
            outs.append((f, None if s is None else (s.hi, s.lo), bits))

        def same(x, y):
            if x is None:
                return y is None
            if isinstance(x, tuple):
                return all(same(p, q) for p, q in zip(x, y))
            return torch.equal(x, y)
        sames = [all(same(x, y) for x, y in zip(outs[0], o)) for o in outs[1:]]
        f, s, bits = outs[-1]
        val = f if f is not None else (s[0].float() + (s[1].float() if s[1] is not None else 0))
        ref = a.double() @ w.double().t() + bias.double()
        if kw.get("act") == ops.ACT_GELU:
            ref = torch.nn.functional.gelu(ref)
        if kw.get("act") == ops.ACT_RELU:
            ref = torch.relu(ref)
        if cs is not None:
            ref = ref * cs.double()
        if res is not None:
            ref = ref + res.double()
        if kw.get("transposed"):
            ref = ref.t()
        err = (val.double() - ref).abs().max().item()
        tol = 2e-3 if prec == 3 else 0.5
        good = all(sames) and err < tol
        if bits is not None:
            want = (val > 0).view(M, N // 32, 32).long()
            want = (want << torch.arange(32, device=dev)).sum(-1)
            want = torch.where(want >= 2 ** 31, want - 2 ** 32, want).int()
            good = good and torch.equal(bits.view(M, N // 32), want)
        ok &= good
        print(f"prec{prec} {M}x{N}x{K} {kw}: variants==baseline {sames}, max err vs fp64 {err:.2e} {'ok' if good else 'FAIL'}", flush=True)
ops.set_precision(3)
for (M, N, K, kw) in [(32768, 5120, 1280, dict(act=ops.ACT_GELU, want_split=True, want_f32=False)), (32768, 2560, 1280, dict(want_split=True, want_f32=False)),
                      (174080, 2048, 256, dict(act=ops.ACT_RELU, want_split=True, want_f32=False)), (174080, 256, 256, dict()),
                      (174080, 384, 256, dict()), (174080, 2048, 32, dict()), (174080, 2048, 32, dict(want_split=True, want_f32=False))]:
    a = torch.randn(M, K, device=dev)
    w = torch.randn(N, K, device=dev) * 0.05
    A, W = ops.split(a), ops.split_weight(w)
    for tma in VARIANTS:
        setv(tma)
        for _ in range(3):
            ops.gemm(A, W, prec=3, **kw)
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(10):
            ops.gemm(A, W, prec=3, **kw)
        e.record()
        torch.cuda.synchronize()
        ms = s.elapsed_time(e) / 10
        print(f"time tma={tma} {M}x{N}x{K} {'planes' if kw.get('want_split') else 'f32'}: {ms:.3f} ms  {2.0*M*N*K/ms/1e9:.0f} TF alg", flush=True)
# mask-embed shape (8 x (300 x 65536 x 256), fp32 rows + bits)
me = torch.randn(8 * 300, 256, device=dev)
px = torch.randn(8 * 65536, 256, device=dev)
A, W = ops.split(me), ops.split_weight(px)
for tma in VARIANTS:
    setv(tma)
    fn = lambda: ops.gemm(A, W, M=300, N=65536, K=256, batch=8, lda=256, ldw=256, a_bstride=300 * 256, w_bstride=65536 * 256, bits_threshold=0.0, prec=3)
    for _ in range(3):
        fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(10):
        fn()
    e.record()
    torch.cuda.synchronize()
    ms = s.elapsed_time(e) / 10
    alg = 8 * ((300 * 256 + 65536 * 256) * 4 + 300 * 65536 * 4 + 300 * 65536 / 8)
    print(f"time tma={tma} mask-embed 8x(300x65536x256): {ms:.3f} ms  {alg/ms/1e6:.0f} GB/s algorithmic", flush=True)
setv(1)
print("GEMM_CHECK_OK" if ok else "GEMM_CHECK_FAIL")
sys.exit(0 if ok else 1)
