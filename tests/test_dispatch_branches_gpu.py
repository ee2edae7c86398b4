"""GPU: the kernel variants and code paths that the launchers select only at production sizes, each reached on purpose and
compared with an fp64 restatement of the same operation (computed on the GPU from exactly the operands the kernel reads), plus
its counterpart just on the other side of the selecting threshold.

| Launcher | Branch | Taken when | Tests |
|---|---|---|---|
| `layernorm_launch` (norm.cu) | `layernorm_bulk_kernel<2/6/10>` | no `add`, C % 128 == 0, C <= 1280, rows >= 4096 | `test_layernorm_bulk_window_map_fp16`, `test_layernorm_bulk_e4m3_planes`, `test_layernorm_bulk_bf16_planes`, `test_layernorm_bulk_threshold` |
| same | grid-stride loop of `layernorm_kernel` | rows > 8 x resident CTAs (`ln_grid_cap`) | `test_layernorm_add_grid_stride` |
| same | `ln_bulk` / `ln_grid_cap` switched off | `hipie_set_option` | the four bulk tests and `test_layernorm_add_grid_stride` (bitwise A/B) |
| `hipie_groupnorm_nhwc` | grid-stride loop of the apply kernel (grid capped at 8 x SMs) | HW * C / 4 > 256 * 8 * SMs | `test_groupnorm_apply_grid` |
| same | `y_bstride` / `add_bstride` != HW * C | writes into the concatenated `src` | `test_groupnorm_apply_grid` |
| `hipie_row_softmax` | `row_softmax_smem_kernel` above 48 KB (opt-in shared memory) | 12288 < n <= 51200, n % 4 == 0 | `test_row_softmax_dispatch` |
| same | `out_fp16` on all three kernels | `attn_fp16` parity mode | `test_row_softmax_dispatch` |
| `hipie_gemm` | `m_fastest = 1` | tiles_m <= 8, tiles_n >= 4 * tiles_m | `test_gemm_m_fastest` |
| same | prec 2 (fp16 x fp16, single pass) | VL-fusion scores and P.V | `test_gemm_prec2_vl_fusion` |
| same | `relu_after_residual` | R50 bottleneck conv3 | `test_gemm_relu_after_residual` |
| misc.cu | `maxpool3x3s2_nhwc`, `im2col_nhwc` 7x7/2/3 on C = 8 and 1x1/2/0, `add_split` | R50 stem, strided shortcut, everywhere | `test_r50_stem_im2col_gemm`, `test_strided_1x1_shortcut`, `test_maxpool3x3s2`, `test_add_split` |

Where the variant is a kernel of its own, the test records the kernels launched (torch.profiler CUDA activity) and asserts the
expected one ran; where it is a runtime flag, a helper restates the launcher's predicate (citing its line) and the test asserts
its shape satisfies it.  The A/B switches (`ln_bulk`, `ln_grid_cap`, `gemm_tma_store`) pick code paths with the same arithmetic,
so their outputs must be bitwise equal to the defaults."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops(cuda):
    from hipie_b200 import ops as o
    o.set_precision(3)
    return o


def _split_ref(x):
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    return hi, lo


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _launched(fn):
    """Run fn under torch.profiler CUDA activity tracing -> (fn(), names of everything recorded, spaces removed)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, {e.key.replace(" ", "") for e in prof.key_averages()}


def _has(names, kernel, *targs):
    """Whether `kernel<targs...>` is among the recorded names, demangled or mangled."""
    dem = kernel + ("<" + ",".join(str(t) for t in targs) + ">" if targs else "(")
    man = kernel + ("I" + "".join(f"Li{t}E" for t in targs) + "E" if targs else "E")
    return any(dem in n or man in n for n in names)


def _assert_ran(names, kernel, *targs, alone_of=()):
    """`kernel<targs...>` was launched, and none of the (kernel, *targs) alternatives in `alone_of` was."""
    shown = sorted(n[:120] for n in names if "hipie" in n)
    assert _has(names, kernel, *targs), f"{kernel}{list(targs)} not launched; recorded: {shown}"
    for alt in alone_of:
        assert not _has(names, *alt), f"{alt} launched as well; recorded: {shown}"


class _option:
    """hipie_set_option(name, value) for the duration of a with block; the default (1) is restored in a finally."""

    def __init__(self, name, value):
        self.name, self.value = name, value

    def __enter__(self):
        from hipie_b200 import _lib
        _lib.set_option(self.name, self.value)

    def __exit__(self, *exc):
        from hipie_b200 import _lib
        _lib.set_option(self.name, 1)
        return False


# ------------------------------------------------------------------------------------------ LayerNorm
def _ln_kernel(rows, C, add):
    """norm.cu:335 (layernorm_launch): the bulk-copy kernel takes plain rows (no residual add) with C % 128 == 0, C <= 1280 and at
    least 4096 rows (x 16-byte aligned, ln_bulk on); the register kernel every other C % 128 == 0 up to 2048.  MAXV = C / 128
    rounded up to 2, 6, 10 (16)."""
    maxv = next(v for v in (2, 6, 10, 16) if C <= 128 * v)
    bulk = not add and C % 128 == 0 and C <= 1280 and rows >= 4096
    return ("layernorm_bulk_kernel" if bulk else "layernorm_kernel"), maxv


def _ln_inputs(rows, C, seed, dev):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(rows, C, device=dev, generator=g) * 2 + 0.5
    gm = torch.rand(C, device=dev, generator=g) + 0.5
    bt = torch.randn(C, device=dev, generator=g) * 0.5
    return x, gm, bt, g


def _ln_ref(x, gm, bt, eps):
    return F.layer_norm(x.double(), (x.shape[-1],), gm.double(), bt.double(), eps)


def _window_map(B, g, ws, dev):
    """ViT window partition as a row map: token (b, y, x) of a g x g grid -> row of its ws x ws window in the grid padded to a
    multiple of ws.  Returns (map, number of window rows, mask of the pad rows no token maps to)."""
    nw = (g + ws - 1) // ws
    b, y, x = torch.meshgrid(torch.arange(B, device=dev), torch.arange(g, device=dev), torch.arange(g, device=dev), indexing="ij")
    rmap = ((((b * nw + y // ws) * nw + x // ws) * ws + y % ws) * ws + x % ws).reshape(-1).int()
    out_rows = B * nw * nw * ws * ws
    pad = torch.ones(out_rows, dtype=torch.bool, device=dev)
    pad[rmap.long()] = False
    return rmap, out_rows, pad


def test_layernorm_bulk_window_map_fp16(ops, cuda):
    """ViT norm1: 8 images x 64 x 64 tokens = 32768 x 1280 scattered into 14 x 14 windows (70 x 70 padded grid) as one fp16
    plane.  The pad rows keep their sentinel, the plane is the rounding of the same call's fp32 rows."""
    B, g, ws, C = 8, 64, 14, 1280
    rmap, out_rows, pad = _window_map(B, g, ws, cuda)
    rows = B * g * g
    assert _ln_kernel(rows, C, add=False) == ("layernorm_bulk_kernel", 10)
    x, gm, bt, _ = _ln_inputs(rows, C, 1, cuda)
    sentinel = torch.full((out_rows, C), -7.25, dtype=torch.float16, device=cuda)

    def run():
        buf = ops.BF2(sentinel.clone(), None)
        y, _, _ = ops.layernorm(x, gm, bt, 1e-6, want_f32=True, row_map=rmap, out_rows=out_rows, out_split=buf, out_fp16=True)
        return y, buf.hi

    (y, h), names = _launched(run)
    _assert_ran(names, "layernorm_bulk_kernel", 10, alone_of=[("layernorm_kernel", 10)])
    m = rmap.long()
    assert (y[m].double() - _ln_ref(x, gm, bt, 1e-6)).abs().max().item() < 2e-5
    assert torch.equal(h[m], y[m].half())
    assert int(pad.sum()) == out_rows - rows and torch.equal(h[pad], sentinel[pad])
    with _option("ln_bulk", 0):
        (y0, h0), names0 = _launched(run)
    _assert_ran(names0, "layernorm_kernel", 10, alone_of=[("layernorm_bulk_kernel", 10)])
    assert torch.equal(y0[m], y[m]) and torch.equal(h0, h)


def test_layernorm_bulk_e4m3_planes(ops, cuda):
    """ViT norm2: 32768 x 1280 -> fp16 + e4m3 planes, bit for bit the split of the same call's fp32 rows."""
    rows, C = 32768, 1280
    assert _ln_kernel(rows, C, add=False) == ("layernorm_bulk_kernel", 10)
    x, gm, bt, _ = _ln_inputs(rows, C, 2, cuda)
    run = lambda: ops.layernorm(x, gm, bt, 1e-6, want_f32=True, out_e4m3=True)[:2]
    (y, s), names = _launched(run)
    _assert_ran(names, "layernorm_bulk_kernel", 10, alone_of=[("layernorm_kernel", 10)])
    assert (y.double() - _ln_ref(x, gm, bt, 1e-6)).abs().max().item() < 2e-5
    ref = ops.split_f16_e4m3(y)
    assert torch.equal(s.hi, ref.hi) and torch.equal(s.lo, ref.lo)
    with _option("ln_bulk", 0):
        (y0, s0), names0 = _launched(run)
    _assert_ran(names0, "layernorm_kernel", 10, alone_of=[("layernorm_bulk_kernel", 10)])
    assert torch.equal(y0, y) and torch.equal(s0.hi, s.hi) and torch.equal(s0.lo, s.lo)


@pytest.mark.parametrize("rows,C", [(21760, 256), (4096, 768)])
def test_layernorm_bulk_bf16_planes(ops, cuda, rows, C):
    """Encoder LN (B * S = 21760 rows at C = 256) and the 6-chunk instantiation: fp32 rows + bf16 hi / lo planes."""
    kernel, maxv = _ln_kernel(rows, C, add=False)
    assert kernel == "layernorm_bulk_kernel"
    x, gm, bt, _ = _ln_inputs(rows, C, rows + C, cuda)
    run = lambda: ops.layernorm(x, gm, bt, 1e-5, want_f32=True, want_split=True)[:2]
    (y, s), names = _launched(run)
    _assert_ran(names, "layernorm_bulk_kernel", maxv, alone_of=[("layernorm_kernel", maxv)])
    assert (y.double() - _ln_ref(x, gm, bt, 1e-5)).abs().max().item() < 2e-5
    hi, lo = _split_ref(y)
    assert torch.equal(s.hi, hi) and torch.equal(s.lo, lo)
    with _option("ln_bulk", 0):
        (y0, s0), names0 = _launched(run)
    _assert_ran(names0, "layernorm_kernel", maxv, alone_of=[("layernorm_bulk_kernel", maxv)])
    assert torch.equal(y0, y) and torch.equal(s0.hi, s.hi) and torch.equal(s0.lo, s.lo)


@pytest.mark.parametrize("C", [1280, 256])
@pytest.mark.parametrize("rows", [4095, 4096])
def test_layernorm_bulk_threshold(ops, cuda, rows, C):
    """Both sides of the 4096-row threshold: the register kernel below it, the bulk-copy kernel from it on."""
    kernel, maxv = _ln_kernel(rows, C, add=False)
    assert kernel == ("layernorm_bulk_kernel" if rows >= 4096 else "layernorm_kernel")
    x, gm, bt, _ = _ln_inputs(rows, C, 7 * rows + C, cuda)
    (y, s), names = _launched(lambda: ops.layernorm(x, gm, bt, 1e-6, want_f32=True, out_fp16=True)[:2])
    _assert_ran(names, kernel, maxv, alone_of=[("layernorm_kernel" if kernel == "layernorm_bulk_kernel" else "layernorm_bulk_kernel", maxv)])
    assert (y.double() - _ln_ref(x, gm, bt, 1e-6)).abs().max().item() < 2e-5
    assert torch.equal(s.hi, y.half())


def test_layernorm_add_grid_stride(ops, cuda):
    """32768 x 1280 with a residual add and the sum written back: the register kernel with its grid capped at the resident CTAs,
    so every warp loops over rows.  ln_grid_cap = 0 (one 8-row CTA per 8 rows, no loop) gives the same bits."""
    rows, C = 32768, 1280
    assert _ln_kernel(rows, C, add=True) == ("layernorm_kernel", 10)
    # norm.cu:315-324 caps the grid at the resident CTAs of layernorm_kernel<MAXV>: at most 8 CTAs of 256 threads per SM, so the
    # grid strides by at most 8 rows x 8 x SMs and 32768 rows need several passes; no cap between 1 and 8 CTAs per SM makes the
    # row count a multiple of the stride, so the last pass is partial
    sms = _sms()
    assert rows > 8 * 8 * sms
    assert all(rows % (8 * k * sms) != 0 for k in range(1, 9))
    x, gm, bt, g = _ln_inputs(rows, C, 3, cuda)
    add = torch.randn(rows, C, device=cuda, generator=g)
    run = lambda: ops.layernorm(x, gm, bt, 1e-6, add=add, want_f32=True, want_split=True, want_sum=True)
    (y, s, ssum), names = _launched(run)
    _assert_ran(names, "layernorm_kernel", 10, alone_of=[("layernorm_bulk_kernel", 10)])
    xs = x + add
    assert torch.equal(ssum, xs)
    assert (y.double() - _ln_ref(xs, gm, bt, 1e-6)).abs().max().item() < 2e-5
    hi, lo = _split_ref(y)
    assert torch.equal(s.hi, hi) and torch.equal(s.lo, lo)
    with _option("ln_grid_cap", 0):
        y0, s0, ssum0 = run()
    assert torch.equal(y0, y) and torch.equal(s0.hi, s.hi) and torch.equal(s0.lo, s.lo) and torch.equal(ssum0, ssum)


# ------------------------------------------------------------------------------------------ GroupNorm
@pytest.mark.parametrize("case", ["hw65536", "hw4100", "at_cap", "over_cap"])
def test_groupnorm_apply_grid(ops, cuda, case):
    """GroupNorm(32) + ReLU + post-add at C = 256: mask_features (HW = 65536, many passes of the capped apply grid), HW = 4100, and
    both sides of the cap.  Then the same call written into a view of a larger buffer (y_bstride) with the addend read from one
    (add_bstride), as the DETR input projections write the concatenated `src`: the gap rows keep their sentinel."""
    N, C = 2, 256
    sms = _sms()
    cap_hw = 256 * 8 * sms * 4 // C                      # norm.cu:406-408: apply grid = min(ceil(HW*C/4 / 256), 8 * SMs) blocks
    HW = {"hw65536": 65536, "hw4100": 4100, "at_cap": cap_hw, "over_cap": cap_hw + 4}[case]
    loops = HW * C // 4 > 256 * 8 * sms
    if case in ("hw65536", "over_cap"):
        assert loops
    if case == "at_cap":
        assert not loops
    g = torch.Generator(device="cuda").manual_seed(HW)
    x = torch.randn(N, HW, C, device=cuda, generator=g) * 3 + 1
    gm, bt = torch.randn(C, device=cuda, generator=g), torch.randn(C, device=cuda, generator=g)
    add = torch.randn(N, HW, C, device=cuda, generator=g)
    ref = F.relu(F.group_norm(x.double().transpose(1, 2), 32, gm.double(), bt.double(), 1e-5)).transpose(1, 2) + add.double()
    y, s = ops.groupnorm_nhwc(x, gm, bt, relu=True, post_add=add, want_split=True)
    assert (y.double() - ref).abs().max().item() < 2e-5
    hi, lo = _split_ref(y)
    assert torch.equal(s.hi, hi) and torch.equal(s.lo, lo)
    # strided output and addend: rows [3, 3 + HW) of a (HW + 7)-row slab per image, addend rows [2, 2 + HW) of (HW + 5)
    ybuf = torch.full((N, HW + 7, C), -5.5, device=cuda)
    abuf = torch.zeros(N, HW + 5, C, device=cuda)
    abuf[:, 2:2 + HW] = add
    yv = ybuf[:, 3:3 + HW]
    out, _ = ops.groupnorm_nhwc(x, gm, bt, relu=True, post_add=abuf[:, 2:2 + HW], out_f32=yv, y_bstride=(HW + 7) * C,
                                add_bstride=(HW + 5) * C)
    assert out.data_ptr() == yv.data_ptr()
    assert (yv.double() - ref).abs().max().item() < 2e-5
    assert bool((ybuf[:, :3] == -5.5).all()) and bool((ybuf[:, 3 + HW:] == -5.5).all())
    with pytest.raises(ValueError):                      # the bf16 planes are (N, HW, C): they cannot follow a larger y_bstride
        ops.groupnorm_nhwc(x, gm, bt, out_f32=yv, y_bstride=(HW + 7) * C, want_split=True)


# ------------------------------------------------------------------------------------------ row softmax
def _softmax_kernel(n, aligned=True):
    """misc.cu:691-711 (hipie_row_softmax): aligned rows (n % 4 == 0) of up to 1024 run the warp-per-row kernel (4 float4 chunks
    per lane up to 512, else 8), longer ones up to 51200 (200 KB) the shared-memory row kernel, everything else the generic one."""
    aligned = aligned and n % 4 == 0
    if aligned and n <= 1024:
        return "row_softmax_warp_kernel", (4 if n <= 512 else 8)
    if aligned and n * 4 <= 200 * 1024:
        return "row_softmax_smem_kernel", None
    return "row_softmax_kernel", None


def _softmax_ref(x, colbias, rows_per_batch, sub_rowmax, clampv=50000.0):
    v = x.double().clamp(-clampv, clampv)
    if sub_rowmax:
        v = (v - v.max(-1, keepdim=True)[0]).clamp(-clampv, clampv)
    if colbias is not None:
        n = x.shape[-1]
        v = (v.view(-1, rows_per_batch, n) + colbias.double()[:, None]).view(-1, n)
    return torch.softmax(v, -1)


# n: warp | smem across the 1024 bound; smem without / with the opt-in above 48 KB (12288 floats); the VL-fusion pixel counts
# S = 21760 / 34000; smem | generic across the 51200 bound; an unaligned n that falls back to the generic kernel
@pytest.mark.parametrize("n", [1024, 1028, 12288, 12292, 21760, 34000, 51200, 51204, 12290])
def test_row_softmax_dispatch(ops, cuda, n):
    """Masked softmax over text (colbias, fp32 + bf16 planes + fp16 plane) and softmax over pixels (row max subtracted, fp16 plane
    alone, as the fp16 VL-fusion path calls it) against fp64; every plane is the rounding of the same call's fp32 output."""
    kernel, nch = _softmax_kernel(n)
    if kernel == "row_softmax_smem_kernel":
        assert (n * 4 > 48 * 1024) == (n > 12288)       # dynamic shared memory above the 48 KB default needs the opt-in
    B, rpb = 2, 3
    g = torch.Generator(device="cuda").manual_seed(n)
    x = torch.randn(B * rpb, n, device=cuda, generator=g) * 4
    cb = torch.ones(B, n, device=cuda)
    cb[1, n // 3:] = -9e15
    targs = (nch,) if nch else ()

    def masked():
        pf, s = ops.row_softmax(x, colbias=cb, rows_per_batch=rpb, want_f32=True)
        pf16, h = ops.row_softmax(x, colbias=cb, rows_per_batch=rpb, want_f32=True, out_fp16=True)
        return pf, s, pf16, h

    (pf, s, pf16, h), names = _launched(masked)
    variants = [("row_softmax_warp_kernel", 4), ("row_softmax_warp_kernel", 8), ("row_softmax_smem_kernel",), ("row_softmax_kernel",)]
    _assert_ran(names, kernel, *targs, alone_of=[v for v in variants if v != (kernel, *targs)])
    ref = _softmax_ref(x, cb, rpb, False)
    assert (pf.double() - ref).abs().max().item() < 1e-6
    hi, lo = _split_ref(pf)
    assert torch.equal(s.hi, hi) and torch.equal(s.lo, lo)
    assert torch.equal(pf16, pf) and h.lo is None and torch.equal(h.hi, pf.half())
    # over pixels: fp16 plane only, against fp64 within the fp16 rounding (half an ulp, 2^-11 relative; 2^-25 absolute in the
    # subnormal range) plus the fp32 arithmetic; and equal to the plane of the same call with the fp32 output requested
    _, h2 = ops.row_softmax(x, sub_rowmax=True, want_split=True, out_fp16=True)
    ref2 = _softmax_ref(x, None, rpb, True)
    assert bool(((h2.hi.double() - ref2).abs() <= ref2 * (2.0 ** -11 + 1e-5) + 2.0 ** -25).all())
    p2, h2f = ops.row_softmax(x, sub_rowmax=True, want_f32=True, out_fp16=True)
    assert (p2.double() - ref2).abs().max().item() < 1e-6
    assert torch.equal(h2f.hi, h2.hi) and torch.equal(h2.hi, p2.half())


# ------------------------------------------------------------------------------------------ GEMM
def _tiles(M, N):
    """gemm_tc.cu:1122-1130, 1077-1078: prec 1 / 2 / 3 run 128 x 64 tiles for N <= 64, 128 x 128 otherwise."""
    BN = 64 if N <= 64 else 128
    return (M + 127) // 128, (N + BN - 1) // BN


def _m_fastest(M, N):
    """gemm_tc.cu:1079 (launch_gemm): p.m_fastest = tiles_m <= 8 && tiles_n >= 4 * tiles_m."""
    tm, tn = _tiles(M, N)
    return tm <= 8 and tn >= 4 * tm


def _pack_bits(c):
    """(.., rows, N) -> (.., rows, N / 32) int32 words, bit j of word w = c[.., 32 w + j] > 0."""
    pred = (c > 0.0).view(*c.shape[:-1], c.shape[-1] // 32, 32).long()
    want = (pred << torch.arange(32, device=c.device)).sum(-1)
    return torch.where(want >= 2 ** 31, want - 2 ** 32, want).int()


# (M, N): the mask-embed shape (300 queries x 4096 pixels, 3 x 32 tiles); 300 rows on both sides of tiles_n = 4 tiles_m (11 / 12
# N tiles); tiles_m = 8 (M = 1000) at and below 32 N tiles; tiles_m = 9, where the flag is off whatever N
@pytest.mark.parametrize("M,N,flag", [(300, 4096, True), (300, 1408, False), (300, 1536, True), (1000, 4096, True), (1000, 3968, False),
                                      (1032, 4096, False)])
@pytest.mark.parametrize("prec", [3, 1])
def test_gemm_m_fastest(ops, cuda, M, N, flag, prec):
    """Batched (B = 2) short-wide GEMM, fp32 rows + the fused (x > 0) bit-packed mask along N, against fp64; the TMA-store and the
    register epilogue give the same bits."""
    assert _m_fastest(M, N) == flag
    B, K = 2, 256
    g = torch.Generator(device="cuda").manual_seed(M + N + prec)
    a = torch.randn(B * M, K, device=cuda, generator=g)
    w = torch.randn(B * N, K, device=cuda, generator=g) * 0.1
    A, W = ops.split(a), ops.split(w)
    run = lambda: ops.gemm(A, W, M=M, N=N, K=K, batch=B, lda=K, ldw=K, a_bstride=M * K, w_bstride=N * K, bits_threshold=0.0, prec=prec)
    c, _, bits = run()
    if prec == 3:
        ref = torch.einsum("bmk,bnk->bmn", a.view(B, M, K).double(), w.view(B, N, K).double())
        tol = 3e-5 * math.sqrt(K) * 0.1 * 4 + 1e-5
    else:
        ref = torch.einsum("bmk,bnk->bmn", A.hi.view(B, M, K).double(), W.hi.view(B, N, K).double())
        tol = 1e-4 * math.sqrt(K) * 0.1 + 1e-5
    assert c.shape == (B, M, N)
    err = (c.double() - ref).abs().max().item()
    assert err < tol, f"max err {err} (tol {tol})"
    assert torch.equal(bits.view(B, M, N // 32), _pack_bits(c))
    with _option("gemm_tma_store", 0):
        c0, _, bits0 = run()
    assert torch.equal(c0, c) and torch.equal(bits0, bits)


def test_gemm_prec2_vl_fusion(ops, cuda):
    """The fp16 VL-fusion contractions of one head (E = 2048, hd = 256, Lt = 256 tokens, S = 1020 pixels padded to an Sp = 1024
    pitch, B = 2): scores (B, S, Lt) and their transpose from strided fp16 column slices, and both P.V products written as bf16
    hi / lo into column slices of preallocated (B * S, E) / (B * Lt, E) buffers whose other columns keep their sentinel."""
    B, E, hd, Lt, S = 2, 2048, 256, 256, 1020
    Sp = (S + 7) // 8 * 8
    g = torch.Generator(device="cuda").manual_seed(17)
    q16 = torch.randn(B * S, E, device=cuda, generator=g).half()
    k16 = (torch.randn(B * Lt, E, device=cuda, generator=g) * 0.1).half()
    vlT = (torch.randn(E, B * Lt, device=cuda, generator=g) * 0.1).half()                      # values of the text side, K-major
    vvT = torch.zeros(E, B, Sp, device=cuda, dtype=torch.float16)                              # values of the image side, Sp pitch
    vvT[:, :, :S] = (torch.randn(E, B, S, device=cuda, generator=g) * 0.1).half()
    vvT = vvT.view(E, B * Sp)
    pv = torch.rand(B * S, Lt, device=cuda, generator=g).half()                                 # softmax over text (fp16 plane)
    pl = torch.zeros(B * Lt, Sp, device=cuda, dtype=torch.float16)                              # softmax over pixels, zero pad columns
    pl[:, :S] = torch.rand(B * Lt, S, device=cuda, generator=g).half()
    sub = lambda t, c0, c1: ops.BF2(t[:, c0:c1], None)
    tol = lambda K, sa, sw: 1e-4 * math.sqrt(K) * sa * sw + 1e-5
    out_v = ops.BF2(torch.full((B * S, E), 3.0, dtype=torch.bfloat16, device=cuda), torch.full((B * S, E), -3.0, dtype=torch.bfloat16, device=cuda))
    out_l = ops.BF2(torch.full((B * Lt, E), 3.0, dtype=torch.bfloat16, device=cuda), torch.full((B * Lt, E), -3.0, dtype=torch.bfloat16, device=cuda))
    heads = (1, 6)
    for h in heads:
        c0, c1 = h * hd, (h + 1) * hd
        qh, kh = sub(q16, c0, c1), sub(k16, c0, c1)

        def scores():
            sc, _, _ = ops.gemm(qh, kh, M=S, N=Lt, K=hd, batch=B, lda=E, ldw=E, a_bstride=S * E, w_bstride=Lt * E, prec=2)
            scT, _, _ = ops.gemm(kh, qh, M=Lt, N=S, K=hd, batch=B, lda=E, ldw=E, a_bstride=Lt * E, w_bstride=S * E, prec=2)
            return sc, scT

        (sc, scT), names = _launched(scores)
        _assert_ran(names, "gemm_tc_kernel", 1, 128)                          # prec 2 shares the single-plane kernel (fp16 wgmma)
        ref = torch.einsum("bsc,btc->bst", q16[:, c0:c1].reshape(B, S, hd).double(), k16[:, c0:c1].reshape(B, Lt, hd).double())
        assert (sc.double() - ref).abs().max().item() < tol(hd, 1.0, 0.1)
        assert (scT.double() - ref.transpose(1, 2)).abs().max().item() < tol(hd, 1.0, 0.1)
        # out_v[b, s, c0:c1] = pv[b] (S x Lt) . vlT[c0:c1, b Lt:(b+1) Lt]^T ; out_l[b, t, c0:c1] = pl[b] (Lt x Sp) . vvT[c0:c1, b Sp:(b+1) Sp]^T
        pv_args = dict(M=S, N=hd, K=Lt, batch=B, lda=Lt, ldw=B * Lt, a_bstride=S * Lt, w_bstride=Lt, prec=2)
        pl_args = dict(M=Lt, N=hd, K=Sp, batch=B, lda=Sp, ldw=B * Sp, a_bstride=Lt * Sp, w_bstride=Sp, prec=2)
        ops.gemm(ops.BF2(pv, None), ops.BF2(vlT[c0:c1], None), want_f32=False, ldc=E, c_bstride=S * E,
                 out_split=ops.BF2(out_v.hi[:, c0:c1], out_v.lo[:, c0:c1]), **pv_args)
        ops.gemm(ops.BF2(pl, None), ops.BF2(vvT[c0:c1], None), want_f32=False, ldc=E, c_bstride=Lt * E,
                 out_split=ops.BF2(out_l.hi[:, c0:c1], out_l.lo[:, c0:c1]), **pl_args)
        # the same products as fp32: against fp64, and the planes are exactly their bf16 split
        fv, _, _ = ops.gemm(ops.BF2(pv, None), ops.BF2(vlT[c0:c1], None), **pv_args)
        fl, _, _ = ops.gemm(ops.BF2(pl, None), ops.BF2(vvT[c0:c1], None), **pl_args)
        ref_v = torch.einsum("bst,bct->bsc", pv.view(B, S, Lt).double(), vlT[c0:c1].view(hd, B, Lt).permute(1, 0, 2).double())
        ref_l = torch.einsum("btk,bck->btc", pl.view(B, Lt, Sp).double(), vvT[c0:c1].view(hd, B, Sp).permute(1, 0, 2).double())
        assert (fv.double() - ref_v).abs().max().item() < tol(Lt, 1.0, 0.1)
        assert (fl.double() - ref_l).abs().max().item() < tol(Sp, 1.0, 0.1)
        for buf, f in ((out_v, fv), (out_l, fl)):
            hi, lo = _split_ref(f.reshape(-1, hd))
            assert torch.equal(buf.hi[:, c0:c1], hi) and torch.equal(buf.lo[:, c0:c1], lo)
        with _option("gemm_tma_store", 0):
            fv0, _, _ = ops.gemm(ops.BF2(pv, None), ops.BF2(vlT[c0:c1], None), **pv_args)
            o0 = ops.BF2(torch.empty(B * S, hd, dtype=torch.bfloat16, device=cuda), torch.empty(B * S, hd, dtype=torch.bfloat16, device=cuda))
            ops.gemm(ops.BF2(pv, None), ops.BF2(vlT[c0:c1], None), want_f32=False, ldc=hd, c_bstride=S * hd, out_split=o0, **pv_args)
        assert torch.equal(fv0, fv) and torch.equal(o0.hi, out_v.hi[:, c0:c1]) and torch.equal(o0.lo, out_v.lo[:, c0:c1])
    untouched = torch.ones(E, dtype=torch.bool, device=cuda)
    for h in heads:
        untouched[h * hd:(h + 1) * hd] = False
    for buf in (out_v, out_l):
        assert bool((buf.hi[:, untouched] == 3.0).all()) and bool((buf.lo[:, untouched] == -3.0).all())


def _fast_epilogue_slices(M, N, ldc, ldr):
    """gemm_tc.cu:229-231 (epilogue_rows): a warp's 32-row x 64-column slice of a 128 x 128 tile takes epilogue_rows_fast when the
    rows are float4-aligned (ldc, ldr % 4 == 0), all 32 rows exist, the slice ends inside N and nothing is remapped.
    Returns (slices on the fast path, slices on the generic path)."""
    vec_ok = ldc % 4 == 0 and ldr % 4 == 0
    tm, tn = _tiles(M, N)
    fast = slow = 0
    for m0 in range(0, tm * 128, 32):
        if m0 >= M:
            continue
        for n0 in range(0, tn * 128, 128):
            for col_end in (64, 128):
                if vec_ok and M - m0 >= 32 and n0 + col_end <= N:
                    fast += 1
                else:
                    slow += 1
    return fast, slow


# N = 200: interior slices on epilogue_rows_fast, the ragged last row tile and column tile on the vectorised generic path;
# N = 198: rows not float4-aligned, every element on the scalar path
@pytest.mark.parametrize("N", [200, 198])
@pytest.mark.parametrize("prec", [3, 1])
def test_gemm_relu_after_residual(ops, cuda, N, prec):
    """R50 bottleneck conv3: relu(A.W^T + b + r) with bias, on the interior and the ragged epilogue, against fp64; the bf16
    planes are exactly the split of the fp32 output."""
    M, K = 1000, 256
    fast, slow = _fast_epilogue_slices(M, N, N, N)
    if N % 4 == 0:
        assert fast > 0 and slow > 0
    else:
        assert fast == 0
    g = torch.Generator(device="cuda").manual_seed(N + prec)
    a = torch.randn(M, K, device=cuda, generator=g)
    w = torch.randn(N, K, device=cuda, generator=g) * 0.1
    b = torch.randn(N, device=cuda, generator=g)
    r = torch.randn(M, N, device=cuda, generator=g)
    A, W = ops.split(a), ops.split_weight(w)
    c, s, _ = ops.gemm(A, W, bias=b, residual=r, relu_after_residual=True, want_split=True, prec=prec)
    if prec == 3:
        pre = a.double() @ w.double().t()
        tol = 3e-5 * math.sqrt(K) * 0.1 * 4 + 1e-5
    else:
        pre = A.hi.double() @ W.hi.double().t()
        tol = 1e-4 * math.sqrt(K) * 0.1 + 1e-5
    pre = pre + b.double() + r.double()
    assert 0.2 < float((pre < 0).double().mean()) < 0.8
    err = (c.double() - torch.relu(pre)).abs().max().item()
    assert err < tol, f"max err {err} (tol {tol})"
    assert bool((c >= 0).all())
    hi, lo = _split_ref(c)
    assert torch.equal(s.hi, hi) and torch.equal(s.lo, lo)


# ------------------------------------------------------------------------------------------ R50 helpers (misc.cu)
def _unfold_nhwc(x, k, stride, pad):
    """(B, H, W, C) -> (B * Ho * Wo, k * k * C) patch rows in (ky, kx, c) column order, by F.unfold (an exact copy)."""
    B, H, W, C = x.shape
    u = F.unfold(x.permute(0, 3, 1, 2), k, padding=pad, stride=stride)          # (B, C * k * k, L), rows (c, ky, kx)
    L = u.shape[-1]
    return u.view(B, C, k, k, L).permute(0, 4, 2, 3, 1).reshape(B * L, k * k * C)


@pytest.mark.parametrize("H,W", [(64, 80), (37, 50)])
def test_r50_stem_im2col_gemm(ops, cuda, H, W):
    """The stem: NHWC image with 3 real and 5 zero channels -> im2col 7 x 7 / 2 / pad 3 (bit for bit the unfolded patches) -> GEMM
    with bias + ReLU, against F.conv2d in fp64."""
    B = 2
    g = torch.Generator(device="cuda").manual_seed(H * W)
    x3 = torch.randn(B, 3, H, W, device=cuda, generator=g)
    x = F.pad(x3.permute(0, 2, 3, 1), (0, 5)).contiguous()
    cols, Ho, Wo = ops.im2col_nhwc(x, 7, 2, 3)
    assert (Ho, Wo) == ((H + 6 - 7) // 2 + 1, (W + 6 - 7) // 2 + 1)
    hi, lo = _split_ref(_unfold_nhwc(x, 7, 2, 3))
    assert torch.equal(cols.hi, hi) and torch.equal(cols.lo, lo)
    w3 = torch.randn(64, 3, 7, 7, device=cuda, generator=g) * 0.1
    b = torch.randn(64, device=cuda, generator=g)
    wk = F.pad(w3, (0, 0, 0, 0, 0, 5)).permute(0, 2, 3, 1).reshape(64, -1).contiguous()
    y, _, _ = ops.gemm(cols, ops.split_weight(wk), bias=b, act=ops.ACT_RELU)
    ref = F.relu(F.conv2d(x3.double(), w3.double(), b.double(), stride=2, padding=3)).permute(0, 2, 3, 1).reshape(-1, 64)
    assert (y.double() - ref).abs().max().item() < 1e-4


@pytest.mark.parametrize("H,W", [(28, 38), (27, 37)])
def test_strided_1x1_shortcut(ops, cuda, H, W):
    """Strided 1 x 1 shortcut: im2col with k = 1, stride 2, pad 0 is row subsampling, x[:, ::2, ::2], bit for bit."""
    B, C = 2, 256
    x = torch.randn(B, H, W, C, device=cuda)
    sub, Ho, Wo = ops.im2col_nhwc(x, 1, 2, 0)
    assert (Ho, Wo) == ((H - 1) // 2 + 1, (W - 1) // 2 + 1)
    hi, lo = _split_ref(x[:, ::2, ::2].reshape(-1, C))
    assert torch.equal(sub.hi, hi) and torch.equal(sub.lo, lo)


@pytest.mark.parametrize("H,W", [(16, 24), (17, 25), (16, 25), (1, 2)])
def test_maxpool3x3s2(ops, cuda, H, W):
    """The stem max-pool against F.max_pool2d(3, 2, 1) on odd and even sizes, bit for bit (fp32 and bf16 planes)."""
    B, C = 2, 64
    x = torch.randn(B, H, W, C, device=cuda)
    y, s = ops.maxpool3x3s2_nhwc(x, want_f32=True, want_split=True)
    ref = F.max_pool2d(x.permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
    assert y.shape == ref.shape and torch.equal(y, ref)
    hi, lo = _split_ref(ref.contiguous())
    assert torch.equal(s.hi, hi) and torch.equal(s.lo, lo)


@pytest.mark.parametrize("with_b", [True, False])
def test_add_split(ops, cuda, with_b):
    """add_split at the encoder size (B * S * 256): the fp32 sum and its bf16 planes, bit for bit."""
    n = 2 * 21760 * 256
    g = torch.Generator(device="cuda").manual_seed(5)
    a = torch.randn(n, device=cuda, generator=g) * 3
    b = torch.randn(n, device=cuda, generator=g) if with_b else None
    s, o = ops.add_split(a, b, want_f32=True)
    want = a + b if with_b else a
    assert torch.equal(s, want)
    hi, lo = _split_ref(want)
    assert torch.equal(o.hi, hi) and torch.equal(o.lo, lo)
    _, o2 = ops.add_split(a, b)
    assert torch.equal(o2.hi, hi) and torch.equal(o2.lo, lo)
