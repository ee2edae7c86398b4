"""GPU: the operand planes of the precision map (DESIGN.md 3) at the edges of fp16 and e4m3, and the range the split is accurate in.

(a) Producers, bit for bit against the host formula (tests/test_precision_planes.py: split_planes = torch .half(), clamp to
    +-448, float8_e4m3fn, slots interleaved by e4m3_slot0) on an edge-value set: every binade from 2^-30 to 2^17, fp16 and e4m3
    rounding ties with their fp32 neighbours, fp16 subnormals and the saturation / overflow points 448 ... 65520, 1e6.  Every
    producer of the plane formats carries the set: split_f16_e4m3 (both modes), the three LayerNorm kernels (gamma = 0: the
    output is exactly beta), the GEMM epilogues (W = 0: the output is exactly the bias), attention_tc (one dominant key: P is
    one-hot, the output is one V row) and row_softmax (fp16-subnormal probabilities).  Each asserts the kernel it meant to reach.
(b) Consumers on planes that hold saturated e4m3 slots, e4m3 subnormals and fp16 subnormals, against fp64 on exactly the planes
    read: only fp32 accumulation may differ.  Also the single-pass fp16 attention on fp16-subnormal probabilities.
(c) The accuracy class of prec 6 as a function of range, on the device, for the operands of tests/test_precision_planes.py.
(d) The operating range of the shipped map: one forward of the c1 configuration and one SAM vit_h image encoding with every
    prec 2 / 4 / 6 GEMM, LayerNorm and attention call recorded (synthetic weights); the tables are printed and kept as JSON in
    $HIPIE_PARITY_DIR (default: the temp directory).
"""
import json
import math
import os
import tempfile
import time
import traceback
import warnings

import pytest
import torch

from test_precision_planes import (IN_RANGE, IN_RANGE_OUTLIERS, OUT_OF_RANGE, OUTLIER_BOUND, RANGE_BOUND, range_case,
                                   split_planes)

pytestmark = pytest.mark.gpu

_T0 = time.time()
BUDGET_S = 900.0


@pytest.fixture(scope="module")
def ops(cuda):
    from hipie_b200 import ops as o
    o.set_precision(3)
    return o


# ------------------------------------------------------------------------------------------ kernel selection (as test_dispatch_branches_gpu)
def _launched(fn):
    """(fn(), names of the device kernels it launched).  A trace that holds the runtime calls but no device activity at all is
    taken once more; if the second one is empty too, the profiler cannot trace in this process (after a session that traced a
    whole model forward, as tests/test_parts_gpu.py does, torch.profiler stops delivering device activity) and the names are None."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(2):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        names = {e.key.replace(" ", "") for e in prof.key_averages()}
        if any(not n.startswith(("cuda", "Activity")) for n in names):
            return out, names
    return out, None


def _assert_ran(names, kernel, *targs, alone_of=()):
    """`kernel<targs...>` (demangled, or mangled with int / bool template arguments) was launched, and none of `alone_of`.  Every
    caller also restates the launcher's predicate for the shape it uses; without a trace (names None) that restatement is what
    remains, and the test says so in a warning."""
    if names is None:
        warnings.warn(f"no device trace in this process: {kernel}{list(targs)} asserted by the restated launcher predicate only")
        return
    def has(k, *ta):
        dem = k + ("<" + ",".join(str(t).lower() for t in ta) + ">" if ta else "(")
        man = k + ("I" + "".join(f"Lb{int(t)}E" if isinstance(t, bool) else f"Li{t}E" for t in ta) + "E" if ta else "E")
        return any(dem in n or man in n for n in names)
    shown = sorted(n[:120] for n in names if "kernel" in n)
    assert has(kernel, *targs), f"{kernel}{list(targs)} not launched; recorded: {shown}"
    for alt in alone_of:
        assert not has(*alt), f"{alt} launched as well; recorded: {shown}"


class _option:
    def __init__(self, name, value):
        self.name, self.value = name, value

    def __enter__(self):
        from hipie_b200 import _lib
        _lib.set_option(self.name, self.value)

    def __exit__(self, *exc):
        from hipie_b200 import _lib
        _lib.set_option(self.name, 1)
        return False


# ------------------------------------------------------------------------------------------ the edge-value set and the host formula
def _edge_values():
    """fp32 values at the edges of fp16 and e4m3, both signs and +-0, in a random order, padded with zeros to a multiple of 1280."""
    up = lambda x: torch.nextafter(x, torch.tensor(math.inf))
    down = lambda x: torch.nextafter(x, torch.tensor(-math.inf))
    # mantissas: exact, the e4m3 ulp and tie (3 bits), the fp16 ulp and tie (10 bits), a tie to even, the top of the binade
    mant = torch.tensor([1.0, 1 + 2 ** -3, 1 + 2 ** -4, 1.5 + 2 ** -4, 1.875 + 2 ** -4, 1 + 2 ** -10, 1 + 2 ** -11, 1 + 3 * 2 ** -11,
                         1.5 + 2 ** -11, 2 - 2 ** -11, 2 - 2 ** -12, 1 + 17 * 2 ** -16, 1 + 2 ** -11 + 9 * 2 ** -17])
    binades = torch.tensor([2.0 ** e for e in range(-30, 18)])
    base = (binades[:, None] * mant[None, :]).flatten()
    ties = (binades[:, None] * mant[None, [2, 3, 4, 6, 7, 8, 10]]).flatten()
    sub16 = (torch.arange(0, 1024, 37).double() + 0.5).float() * 2.0 ** -24          # fp16 subnormal ties
    edges = torch.tensor([448.0, 464.0, 465.0, 480.0, 896.0, 65504.0, 65519.0, 65520.0, 1e6, 2.0 ** -14, 2.0 ** -14 - 2.0 ** -24,
                          2.0 ** -24, 2.0 ** -25, 2.0 ** -6, 2.0 ** -9, 2.0 ** -10, 28.0, 29.0])
    g = torch.Generator().manual_seed(0)
    rnd = torch.exp2(torch.rand(512, generator=g) * 47 - 30) * (1 + torch.rand(512, generator=g))
    mag = torch.cat([base, up(ties), down(ties), sub16, up(sub16), down(sub16), edges, up(edges), down(edges), rnd])
    v = torch.cat([mag, -mag, torch.tensor([0.0, -0.0])])
    v = v[torch.randperm(v.numel(), generator=g)]
    pad = (-v.numel()) % 1280
    return torch.cat([v, torch.zeros(pad)])


EDGES = _edge_values()


def _host(x, weight=False):
    """Host formula of the planes of fp32 rows x: (fp16 plane, (rows, 2K) e4m3 plane as float values)."""
    h, p8 = split_planes(x.float().cpu(), weight)
    return h, p8.view(torch.float8_e4m3fn).float()


def _assert_planes(planes, want, weight=False, what=""):
    """BF2 fp16 (+ e4m3) planes == the host formula of the fp32 rows `want`, value for value (+0 == -0; a NaN never matches)."""
    h, p8 = _host(want.reshape(-1, want.shape[-1]), weight)
    got_h = planes.hi.reshape(h.shape).cpu()
    bad = (got_h.float() != h.float()).nonzero()
    assert bad.numel() == 0, f"{what}: fp16 plane differs at {bad[:4].tolist()}: {got_h[tuple(bad[0])].item()} vs {h[tuple(bad[0])].item()}"
    if planes.lo is not None:
        got8 = planes.lo.reshape(p8.shape).cpu().view(torch.float8_e4m3fn).float()
        bad = (got8 != p8).nonzero()
        assert bad.numel() == 0, f"{what}: e4m3 plane differs at {bad[:4].tolist()}: {got8[tuple(bad[0])].item()} vs {p8[tuple(bad[0])].item()}"


def test_edge_set_reaches_the_edges():
    """The set covers what the producers are checked at: e4m3 saturation, fp16 overflow, fp16 subnormals, e4m3 subnormals in both
    slots, and ties of both formats."""
    h, p8 = _host(EDGES.view(-1, 64))
    s0 = p8.view(-1, 2, 2, 32)[:, :, 0].flatten()
    s1 = p8.view(-1, 2, 2, 32)[:, :, 1].flatten()
    sub16 = (h.float().abs() < 2.0 ** -14) & (h != 0)
    assert int(torch.isinf(h).sum()) >= 8 and int(sub16.sum()) >= 100
    assert int((s0.abs() == 448).sum()) >= 50 and int(((s0.abs() < 2.0 ** -6) & (s0 != 0)).sum()) >= 20
    assert int((s1.abs() == 448).sum()) >= 8 and int(((s1.abs() < 2.0 ** -6) & (s1 != 0)).sum()) >= 50
    assert bool(((EDGES == 65519.0) | (EDGES == 65520.0)).any()) and bool((EDGES == 464.0).any())


# ------------------------------------------------------------------------------------------ (a) producers
@pytest.mark.parametrize("weight", [False, True])
def test_split_f16_e4m3_at_the_edges(ops, cuda, weight):
    x = EDGES.view(-1, 640).to(cuda)
    p, names = _launched(lambda: ops.split_f16_e4m3(x, weight=weight))
    _assert_ran(names, "split_f16_e4m3_kernel")
    _assert_planes(p, x, weight, "split_f16_e4m3")


def _ln_kernel(rows, C):
    """norm.cu layernorm_launch: the bulk-copy kernel for plain rows with C % 128 == 0, C <= 1280 and >= 4096 rows, the register
    kernel for the other C % 128 == 0 up to 2048, the generic one-block-per-row kernel for every other C."""
    if C % 128:
        return ("layernorm_generic_kernel",)
    maxv = next(v for v in (2, 6, 10, 16) if C <= 128 * v)
    return ("layernorm_bulk_kernel" if C <= 1280 and rows >= 4096 else "layernorm_kernel", maxv)


@pytest.mark.parametrize("rows,C", [(4096, 1280), (300, 1280), (300, 224)])
@pytest.mark.parametrize("fmt", ["e4m3", "fp16"])
def test_layernorm_planes_at_the_edges(ops, cuda, rows, C, fmt):
    """gamma = 0: every row normalises to exactly beta, and beta carries C edge values per call."""
    kernel = _ln_kernel(rows, C)
    others = [k for k in (("layernorm_bulk_kernel", 10), ("layernorm_kernel", 10), ("layernorm_generic_kernel",)) if k != kernel]
    g = torch.Generator(device="cuda").manual_seed(rows + C)
    x = torch.randn(rows, C, device=cuda, generator=g) * 3 + 1
    gm = torch.zeros(C, device=cuda)
    n = EDGES.numel() // C * C
    for i, beta in enumerate(EDGES[:n].view(-1, C)):
        bt = beta.to(cuda)
        run = lambda: ops.layernorm(x, gm, bt, 1e-6, want_f32=True, out_e4m3=fmt == "e4m3", out_fp16=fmt == "fp16")[:2]
        (y, s), names = _launched(run) if i == 0 else (run(), ())
        if i == 0:
            _assert_ran(names, *kernel, alone_of=others)
        assert torch.equal(y, bt.expand(rows, C))
        assert (s.lo is None) == (fmt == "fp16")
        _assert_planes(s, bt.expand(rows, C), what=f"layernorm {kernel} chunk {i}")


@pytest.mark.parametrize("prec,N", [(3, 64), (3, 1280), (6, 64), (6, 1280)])
def test_gemm_e4m3_epilogue_at_the_edges(ops, cuda, prec, N):
    """out_e4m3 through the staged epilogue (BN 64 / 128) and the register epilogue of the 128 x 256 tiles (prec 6, N > 64).
    W = 0: the output is exactly the bias, which carries N edge values per call."""
    M, K = 256, 128
    BN = (64 if N <= 64 else 128) if prec == 3 else (64 if N <= 64 else 256)     # gemm_tc.cu hipie_gemm
    g = torch.Generator(device="cuda").manual_seed(N + prec)
    a = torch.randn(M, K, device=cuda, generator=g)
    A = ops.split(a) if prec == 3 else ops.split_f16_e4m3(a)
    W = ops.BF2.zeros((N, K), cuda, "bf16x2" if prec == 3 else "f16+e4m3")
    for i, bias in enumerate(EDGES.view(-1, N)):
        b = bias.to(cuda)
        run = lambda: ops.gemm(A, W, bias=b, want_f32=True, out_e4m3=True, prec=prec)
        (c, s, _), names = _launched(run) if i == 0 else (run(), ())
        if i == 0:
            _assert_ran(names, "gemm_tc_kernel", prec, BN)
        assert torch.equal(c, b.expand(M, N))
        _assert_planes(s, b.expand(M, N), what=f"gemm prec {prec} BN {BN} chunk {i}")


@pytest.mark.parametrize("prec", [3, 4])
@pytest.mark.parametrize("tma", [1, 0])
def test_gemm_fp16_epilogue_at_the_edges(ops, cuda, prec, tma):
    """out_fp16 (one IEEE fp16 plane) through the TMA-store and the register store path, on the staged epilogue (prec 3, BN 128)
    and the 128 x 256 register epilogue (prec 4)."""
    M, K, N = 256, 128, 1280
    g = torch.Generator(device="cuda").manual_seed(prec + 10 * tma)
    a = torch.randn(M, K, device=cuda, generator=g)
    A = ops.split(a) if prec == 3 else ops.BF2(a.half(), None)
    W = ops.BF2.zeros((N, K), cuda, "bf16x2" if prec == 3 else "f16x2")
    for i, bias in enumerate(EDGES.view(-1, N)):
        b = bias.to(cuda)
        with _option("gemm_tma_store", tma):
            run = lambda: ops.gemm(A, W, bias=b, want_f32=True, out_fp16=True, prec=prec)
            (c, s, _), names = _launched(run) if i == 0 else (run(), ())
        if i == 0:
            _assert_ran(names, "gemm_tc_kernel", prec, 128 if prec == 3 else 256)
        assert torch.equal(c, b.expand(M, N)) and s.lo is None
        _assert_planes(s, b.expand(M, N), what=f"gemm fp16 prec {prec} tma {tma} chunk {i}")


def test_gemm_transposed_fp16_epilogue_at_the_edges(ops, cuda):
    """The vectorised V^T epilogue (transposed fp16 plane, 8 rows per lane): gemm_tc.cu launch_gemm takes it for a transposed fp16
    plane alone (no fp32 output, residual, colscale, bits or activation) with M % 8 == 0 and ldc % 8 == 0."""
    M, K, N = 256, 64, 1280
    A = ops.split(torch.randn(M, K, device=cuda))
    W = ops.BF2.zeros((N, K), cuda, "bf16x2")
    assert M % 8 == 0
    for i, bias in enumerate(EDGES.view(-1, N)):
        b = bias.to(cuda)
        run = lambda: ops.gemm(A, W, bias=b, want_f32=False, transposed=True, out_fp16=True, prec=3)
        (_, s, _), names = _launched(run) if i == 0 else (run(), ())
        if i == 0:
            _assert_ran(names, "gemm_tc_kernel", 3, 128)
        assert s.hi.shape == (N, M)
        _assert_planes(s, b[:, None].expand(N, M), what=f"V^T chunk {i}")


def test_attention_tc_e4m3_output_at_the_edges(ops, cuda):
    """attention_tc(out_e4m3=True) on the bf16x3 path: every query meets one key whose score leads all others by > 170 (log2
    units > 250), so P is exactly one-hot (ex2 of the others flushes to 0), and the output row is V's row of that key, which
    carries B * H * 80 edge values per call."""
    B, H, hd, T = 4, 16, 80, 256
    E = H * hd
    assert T % 256 == 0                # attention_tc.cu attention_tc_impl: a global grid without rel-pos -> the 64-key-tile kernel
    qk = torch.zeros(B * T, 2 * E, device=cuda)
    qk[:, :E] = 1.0
    qk.view(B, T, 2 * E)[:, 0, E:] = 20.0                      # key 0 of every batch item: score 80 * 20 / sqrt(80) = 179
    vals = EDGES[:EDGES.numel() // (B * E) * (B * E)].view(-1, B, E)
    QK = ops.split(qk)
    q, k = QK[:, :E], QK[:, E:]
    for i, v0 in enumerate(vals):
        vt = torch.zeros(E, B, T, device=cuda)
        vt[:, :, 0] = v0.t().to(cuda)
        VT = ops.split(vt.view(E, B * T))
        run = lambda: ops.attention_tc(q, k, VT, B, H, T, hd, T * 2 * E, 2 * E, T * 2 * E, 2 * E, hd ** -0.5, want_f32=True,
                                       out_e4m3=True, prec=3)
        (o, s), names = _launched(run) if i == 0 else (run(), ())
        if i == 0:
            _assert_ran(names, "attn_tc_kernel", 3, False, False, 64)
        want = (VT.hi.float() + VT.lo.float()).view(E, B, T)[:, :, 0].t()[:, None, :].expand(B, T, E)
        assert torch.equal(o, want)
        _assert_planes(s, want, what=f"attention_tc chunk {i}")


def test_row_softmax_fp16_subnormal_probabilities(ops, cuda):
    """Logits spread over 40 nats: a fifth of the probabilities fall in fp16's subnormal range, some below it.  The fp16 plane is
    the IEEE rounding of the same call's fp32 probabilities (misc.cu hipie_row_softmax: aligned n <= 1024 -> the warp kernel, 8
    float4 chunks per lane above 512)."""
    rows, n = 24, 1024
    assert n % 4 == 0 and 512 < n <= 1024
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.linspace(0, -40, n, device=cuda).repeat(rows, 1) + torch.rand(rows, n, device=cuda, generator=g) * 0.1
    (pf, s), names = _launched(lambda: ops.row_softmax(x, want_f32=True, out_fp16=True))
    _assert_ran(names, "row_softmax_warp_kernel", 8, alone_of=[("row_softmax_warp_kernel", 4), ("row_softmax_smem_kernel",), ("row_softmax_kernel",)])
    sub = (pf < 2.0 ** -14) & (pf >= 2.0 ** -25)
    assert int(sub.sum()) > rows * 150 and int((pf < 2.0 ** -25).sum()) > 0
    assert s.lo is None and torch.equal(s.hi, pf.half())
    ref = torch.softmax(x.double(), -1)
    assert bool(((s.hi.double() - ref).abs() <= ref * (2.0 ** -11 + 1e-5) + 2.0 ** -25).all())


# ------------------------------------------------------------------------------------------ (b) consumers on edge planes
_E4M3_NAN = (0x7F, 0xFF)


def _edge_bytes(shape, g, dev):
    """e4m3 plane bytes: a third saturated (+-448), a third subnormal (exponent field 0), the rest anything but NaN."""
    b = torch.randint(0, 256, shape, generator=g, device=dev)
    kind = torch.randint(0, 3, shape, generator=g, device=dev)
    sign = torch.randint(0, 2, shape, generator=g, device=dev) * 0x80
    b = torch.where(kind == 0, 0x7E + sign, b)
    b = torch.where(kind == 1, (b & 0x07) + sign, b)
    b = torch.where((b == 0x7F) | (b == 0xFF), b - 1, b)
    return b.to(torch.uint8)


def _sub16(shape, g, dev):
    """fp16 subnormals k * 2^-24, |k| < 1024."""
    return (torch.randint(-1023, 1024, shape, generator=g, device=dev).float() * 2.0 ** -24).half()


def _f8(p):
    return p.view(torch.float8_e4m3fn).double()


@pytest.mark.parametrize("M,N,K", [(512, 512, 1280), (512, 256, 5120), (256, 64, 1280)])
def test_prec6_on_edge_planes(ops, cuda, M, N, K):
    """fc1 (K = 1280) and fc2 (K = 5120) shapes on the 128 x 256 tiles, and N = 64 on 128 x 64.  Row groups of A (and the same of
    W): normal fp16 with edge e4m3 slots; fp16 subnormals alone (e4m3 planes zero); e4m3 planes alone (fp16 plane zero), with
    saturated slots and subnormals; e4m3 subnormals alone.  Against fp64 on exactly these planes, relative to |planes|.|planes|^T:
    fp32 accumulation of the fp16 sweep (2^-16), and of the e4m3 sweep, whose wgmma accumulates in fewer bits (about 14, as public
    reports on Hopper's fp8 MMA state) -- 2^-11 of a term that is itself 2^-14 of the planes' scale.  A flushed subnormal or a
    misread saturated slot misses by the whole product."""
    g = torch.Generator(device="cuda").manual_seed(M + N + K)

    def planes(R):
        h = torch.randn(R, K, device=cuda, generator=g).half()
        p8 = _edge_bytes((R, 2 * K), g, cuda)
        q = R // 4
        h[q:2 * q] = _sub16((q, K), g, cuda)
        p8[q:2 * q] = 0
        h[2 * q:] = 0
        p8[3 * q:] = (p8[3 * q:] & 0x87)                                   # e4m3 subnormals (and zeros) only
        return ops.BF2(h, p8)

    A, W = planes(M), planes(N)
    (c, _, _), names = _launched(lambda: ops.gemm(A, W, prec=6))
    _assert_ran(names, "gemm_tc_kernel", 6, 64 if N <= 64 else 256)
    ref = A.hi.double() @ W.hi.double().t() + (_f8(A.lo) @ _f8(W.lo).t()) * 2.0 ** -14
    n16 = A.hi.double().abs() @ W.hi.double().abs().t()
    n8 = (_f8(A.lo).abs() @ _f8(W.lo).abs().t()) * 2.0 ** -14
    err = (c.double() - ref).abs()
    assert bool(torch.isfinite(c).all())
    tol = n16 * 2.0 ** -16 + n8 * 2.0 ** -11
    assert bool((err <= tol).all()), f"max err / tol {(err / tol.clamp_min(1e-300)).max().item()}"
    q, r = M // 4, N // 4
    assert 0 < n16[q:2 * q, r:2 * r].max() < 2.0 ** -12 and n8[q:2 * q, r:2 * r].max() == 0       # fp16 subnormal x fp16 subnormal
    assert 0 < n8[3 * q:, 3 * r:].max() < 2.0 ** -14 and n16[3 * q:, 3 * r:].max() == 0          # e4m3 subnormals only


@pytest.mark.parametrize("M,N,K", [(512, 512, 1280), (256, 64, 1280)])
def test_prec4_on_subnormal_planes(ops, cuda, M, N, K):
    """prec 4: A one fp16 plane with subnormal rows, W fp16 hi + lo where lo is subnormal (as for weights below ~2^-3) and a
    quarter of the rows carry their value in lo alone (hi = 0)."""
    g = torch.Generator(device="cuda").manual_seed(M + N + K + 4)
    a = torch.randn(M, K, device=cuda, generator=g).half()
    a[: M // 2] = _sub16((M // 2, K), g, cuda)
    wh = (torch.randn(N, K, device=cuda, generator=g) * 0.03).half()
    wl = _sub16((N, K), g, cuda)
    wh[: N // 4] = 0
    A, W = ops.BF2(a, None), ops.BF2(wh, wl)
    (c, _, _), names = _launched(lambda: ops.gemm(A, W, prec=4))
    _assert_ran(names, "gemm_tc_kernel", 4, 64 if N <= 64 else 256)
    ref = a.double() @ (wh.double() + wl.double()).t()
    norm = a.double().abs() @ (wh.double().abs() + wl.double().abs()).t()
    err = (c.double() - ref).abs()
    assert bool((err <= norm * 2.0 ** -16).all()), f"max rel {(err / norm.clamp_min(1e-300)).max().item()}"
    assert 0 < norm[: M // 2, : N // 4].max() < 2.0 ** -12                   # subnormal A x subnormal W-lo alone


def test_prec2_on_subnormal_planes(ops, cuda):
    """prec 2 (the VL-fusion contractions): fp16 x fp16 in one pass, with subnormal rows of A and subnormal columns of W."""
    M, N, K = 512, 384, 512
    g = torch.Generator(device="cuda").manual_seed(22)
    a = torch.randn(M, K, device=cuda, generator=g).half()
    w = torch.randn(N, K, device=cuda, generator=g).half()
    a[::2] = _sub16((M // 2, K), g, cuda)
    w[::3] = _sub16((N // 3, K), g, cuda)
    (c, _, _), names = _launched(lambda: ops.gemm(ops.BF2(a, None), ops.BF2(w, None), prec=2))
    _assert_ran(names, "gemm_tc_kernel", 1, 128)
    ref = a.double() @ w.double().t()
    norm = a.double().abs() @ w.double().abs().t()
    assert bool(((c.double() - ref).abs() <= norm * 2.0 ** -16).all())


def test_fp16_attention_on_subnormal_probabilities(ops, cuda):
    """Single-pass fp16 attention (the ViT's attn_fp16 path): per query one key at P = 1 and 255 keys 14 ... 20 binades below it,
    i.e. P in fp16's subnormal range, on positive V.  The PV pass and the denominator must use those probabilities as rounded to
    fp16: against fp64 with P rounded the same way, the keys below 2^-14 carry ~2^-8 of every output."""
    B, H, hd, T = 1, 2, 80, 256
    E = H * hd
    assert T % 256 == 0
    scale = hd ** -0.5
    g = torch.Generator().manual_seed(23)
    d = torch.rand(T, generator=g, dtype=torch.float64) * 6 + 14                # binades below the leading key
    d[0] = 0.0
    c = (150.0 - d / (scale * math.log2(math.e))).half()                        # key h-dim 0; query = e_0
    qk = torch.zeros(B * T, 2 * E, dtype=torch.float16)
    for h in range(H):
        qk[:, h * hd] = 1.0
        qk[:, E + h * hd] = c
    v = (1 + torch.rand(B * T, E, generator=g)).half()
    qk, vt = qk.to(cuda), v.t().contiguous().to(cuda)
    q, k, VT = ops.BF2(qk[:, :E], None), ops.BF2(qk[:, E:], None), ops.BF2(vt, None)
    run = lambda: ops.attention_tc(q, k, VT, B, H, T, hd, T * 2 * E, 2 * E, T * 2 * E, 2 * E, scale, want_f32=True, want_split=False,
                                   f16=True)
    (o, _), names = _launched(run)
    _assert_ran(names, "attn_tc_kernel", 1, False, True, 64)
    s = c.double() * scale * math.log2(math.e)
    p = torch.exp2(s - s.max()).half()
    assert int(((p.float() < 2.0 ** -14) & (p.float() > 0)).sum()) > 200
    ref = (p.double() @ v.double()) / p.double().sum()                          # the same for every query and head
    err = (o.cpu().double().view(B * T, E) - ref[None, :]).abs().max().item()
    assert err < 2.0 ** -14, err


# ------------------------------------------------------------------------------------------ (c) the accuracy class against range
def _device_errors(ops, cuda, a, w):
    A, W = ops.split_f16_e4m3(a.to(cuda)), ops.split_f16_e4m3(w.to(cuda), weight=True)
    c6, _, _ = ops.gemm(A, W, prec=6)
    c1, _, _ = ops.gemm(ops.BF2(A.hi, None), ops.BF2(W.hi, None), prec=2)
    exact = a.double() @ w.double().t()
    norm = a.double().abs() @ w.double().abs().t()
    rel = lambda c: ((c.cpu().double() - exact).abs() / norm).max().item()
    return bool(torch.isfinite(c6).all()), rel(c6), rel(c1)


@pytest.mark.parametrize("kind,value", IN_RANGE + IN_RANGE_OUTLIERS)
@pytest.mark.parametrize("K", [1280, 5120])
def test_prec6_accuracy_inside_the_range(ops, cuda, kind, value, K):
    """prec 6 on the 128 x 256 tiles (N = 320) against the exact product of the fp32 operands: the bound of
    tests/test_precision_planes.py holds on the device, well below one fp16 pass."""
    finite, err, err_one = _device_errors(ops, cuda, *range_case(kind, value, K, rows=128, cols=320))
    bound = OUTLIER_BOUND if "outliers" in kind else RANGE_BOUND
    assert finite and err < bound and err < err_one / 6, (math.log2(err), math.log2(err_one))


@pytest.mark.parametrize("kind,value", OUT_OF_RANGE)
def test_prec6_fallback_outside_the_range(ops, cuda, kind, value):
    """Outside the range the result stays finite and no worse than one fp16 pass over the same fp16 planes."""
    finite, err, err_one = _device_errors(ops, cuda, *range_case(kind, value, 1280, rows=128, cols=320))
    assert finite and err <= err_one, (math.log2(err), math.log2(err_one))
    assert err > OUTLIER_BOUND


# ------------------------------------------------------------------------------------------ (d) the operating range of the shipped map
class _Recorder:
    """Wraps ops.gemm / ops.layernorm / ops.attention_tc for one forward and keeps, per call site (engine file:line) and operand,
    the largest values seen: max |A| and |W| of every prec 2 / 4 / 6 GEMM, the fraction of their elements above 448 and of their
    nonzero rows whose max is below 2^-4, and max |x| of every fp16 plane produced or read."""

    def __init__(self, ops):
        self.ops, self.sites = ops, {}
        self.orig = {n: getattr(ops, n) for n in ("gemm", "layernorm", "attention_tc")}

    def __enter__(self):
        for n in self.orig:
            setattr(self.ops, n, getattr(self, "_" + n))
        return self

    def __exit__(self, *exc):
        for n, f in self.orig.items():
            setattr(self.ops, n, f)
        return False

    @staticmethod
    def _site():
        for fr in reversed(traceback.extract_stack()):
            if os.sep + "modeling" + os.sep in fr.filename:
                return f"{os.path.basename(fr.filename)}:{fr.lineno}"
        return "?"

    def _put(self, site, key, value, reduce=max):
        d = self.sites.setdefault(site, {})
        d[key] = value if key not in d else reduce(d[key], value)

    def _operand(self, site, name, t):
        x = t.detach().float().abs()
        rmax = x.reshape(-1, x.shape[-1]).amax(-1)
        nz = rmax > 0
        self._put(site, f"{name}_max", x.max().item())
        self._put(site, f"{name}_frac_above_448", (x > 448).float().mean().item())
        self._put(site, f"{name}_rows_below_2^-4", ((rmax < 2.0 ** -4) & nz).float().sum().item() / max(1, int(nz.sum())))
        if t.dtype == torch.float16:
            self._put(site, f"{name}_frac_fp16_subnormal", ((x < 2.0 ** -14) & (x > 0)).float().mean().item())

    def _plane(self, site, name, planes):
        if planes is not None and planes.hi.dtype == torch.float16:
            self._put(site, f"{name}_fp16_max", planes.hi.float().abs().max().item())

    def _gemm(self, a, w, *args, **kw):
        out = self.orig["gemm"](a, w, *args, **kw)
        prec = kw.get("prec") or self.ops.PREC
        if prec in (2, 4, 6):
            site = f"{self._site()} prec{prec}"
            self._put(site, "calls", 1, lambda x, y: x + y)
            self._operand(site, "A", a.hi)
            self._operand(site, "W", w.hi)
            self._plane(site, "out", out[1])
        return out

    def _layernorm(self, *args, **kw):
        out = self.orig["layernorm"](*args, **kw)
        if kw.get("out_fp16") or kw.get("out_e4m3"):
            site = f"{self._site()} layernorm" + ("+e4m3" if kw.get("out_e4m3") else "")
            self._put(site, "calls", 1, lambda x, y: x + y)
            self._plane(site, "out", out[1])
        return out

    def _attention_tc(self, q, k, vt, *args, **kw):
        out = self.orig["attention_tc"](q, k, vt, *args, **kw)
        if kw.get("f16") or kw.get("out_e4m3"):
            site = f"{self._site()} attention_tc"
            self._put(site, "calls", 1, lambda x, y: x + y)
            for name, p in (("q", q), ("k", k), ("vt", vt), ("out", out[1])):
                self._plane(site, name, p)
        return out


def _budget(need):
    if time.time() - _T0 + need > BUDGET_S:
        pytest.skip(f"time budget: {time.time() - _T0:.0f}s used, case needs ~{need:.0f}s")


def _report(name, sites, seconds):
    out_dir = os.environ.get("HIPIE_PARITY_DIR") or os.path.join(tempfile.gettempdir(), "hipie_parity")
    os.makedirs(out_dir, exist_ok=True)
    dev = torch.cuda.get_device_name(0)
    with open(os.path.join(out_dir, f"precision_range_{name}.json"), "w") as f:
        json.dump(dict(case=name, weights="synthetic (hipie_oracle.synth)", device=dev, seconds=seconds, sites=sites), f, indent=1)
    print(f"\n[{name}] operating range of the precision map, synthetic weights, {seconds:.1f} s on {dev}")
    for site, d in sorted(sites.items()):
        print(f"  {site:36s} " + "  ".join(f"{k} {v:.4g}" for k, v in d.items() if k != "calls") + f"  ({d['calls']} calls)")


def _check_range(sites):
    """The range DESIGN.md 3 states, with a margin of two: prec-6 activations below 224 with no row under 2^-4, prec-6 weights
    below 14; every fp16 plane finite and below 2^15."""
    seen6 = False
    for site, d in sites.items():
        if site.endswith("prec6"):
            seen6 = True
            assert d["A_max"] < 224 and d["A_frac_above_448"] == 0, (site, d)
            assert d["A_rows_below_2^-4"] == 0, (site, d)
            assert d["W_max"] < 14, (site, d)
        for k, v in d.items():
            if k.endswith("fp16_max"):
                assert math.isfinite(v) and v < 2.0 ** 15, (site, k, v)
    assert seen6


def test_operating_range_c1(cuda):
    """c1 (ViT-H, 1024 x 1024, 80 classes) as tests/test_fullsize_gpu.py builds it; only the oracle's weights are used."""
    _budget(200)
    from hipie_oracle import hparams, synth
    from hipie_oracle.model import HipieOracle
    from hipie_b200 import ops
    from hipie_b200.modeling.hipie_img import HIPIE_IMG
    torch.manual_seed(0)
    hp = hparams.get("vit_h")
    inputs, ids, am = synth.make_batch(1, 1024, 1024, 80, hp["max_query_len"])
    oracle = HipieOracle(hp).eval()
    synth.perturb_(oracle, seed=1)
    for x, i, a in zip(inputs, ids, am):
        x["input_ids"], x["attention_mask"] = i, a
    ops.set_precision(3)
    model = HIPIE_IMG(hp=hp, state_dict=oracle.state_dict(), device="cuda:0")
    del oracle
    t0 = time.time()
    with torch.no_grad(), _Recorder(ops) as rec:
        model(inputs)
    torch.cuda.synchronize()
    _report("c1_vith_1024_coco80", rec.sites, time.time() - t0)
    _check_range(rec.sites)


def test_operating_range_sam_vit_h(cuda):
    """The SAM vit_h image encoder (SamPredictor.set_image) on one 600 x 800 image."""
    _budget(120)
    import numpy as np
    import torch.nn.functional as F
    from hipie_oracle.sam import GEOMETRIES, build
    from hipie_b200 import ops
    from hipie_b200.modeling.sam import SamPredictor
    ops.set_precision(3)
    pred = SamPredictor(build(GEOMETRIES["vit_h"], seed=50).state_dict(), device=cuda)
    g = torch.Generator().manual_seed(51)
    base = torch.rand(1, 3, 600 // 16, 800 // 16, generator=g) * 255
    image = F.interpolate(base, (600, 800), mode="bilinear", align_corners=False)[0].clamp(0, 255).permute(1, 2, 0).numpy().astype(np.uint8)
    t0 = time.time()
    with _Recorder(ops) as rec:
        pred.set_image(image)
    torch.cuda.synchronize()
    _report("sam_vit_h_encoder", rec.sites, time.time() - t0)
    _check_range(rec.sites)
