"""GPU: the 128 x 256 GEMM tiles of prec 6 (fp16 + e4m3 split) and prec 4 (two-pass fp16), whose epilogue runs straight from the
wgmma register fragment, against fp64 on exactly the planes the kernel reads.  Covers ragged M with an odd number of 128-row
tiles, N that is not a multiple of 256, K = 5120, the proj call (residual plus a per-window row map with -1 pad rows, written in
place), the fc1 call (GELU -> fp16 + e4m3 planes, bit for bit the split of the fp32 result) and the qk call (prec 4 -> one fp16
plane at N = 2560).  Tolerances are those of the 128 x 128 tiles' tests."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops(cuda):
    from hipie_b200 import ops as o
    o.set_precision(3)
    return o


def _e4m3(t):
    return t.view(torch.float8_e4m3fn).double()


def _p6_inputs(ops, M, N, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, K, device="cuda", generator=g) * 1.5
    w = torch.randn(N, K, device="cuda", generator=g) * 0.05
    b = torch.randn(N, device="cuda", generator=g)
    A, W = ops.split_f16_e4m3(a), ops.split_f16_e4m3(w, weight=True)
    planes = A.hi.double() @ W.hi.double().t() + (_e4m3(A.lo) @ _e4m3(W.lo).t()) * 2.0 ** -14 + b.double()
    return A, W, b, planes, 3e-5 * math.sqrt(K) * 1.5 * 0.05 * 4 + 1e-5


# (M, N, K): 3 row tiles with a ragged last one; N = 2.5 wide tiles; one wide tile minus a 32-column chunk; N = 96 (one ragged
# tile); K = 5120 (fc2)
@pytest.mark.parametrize("M,N,K", [(300, 640, 256), (421, 480, 128), (130, 96, 64), (256, 1280, 5120)])
def test_gemm_wide_p6_f32(ops, cuda, M, N, K):
    A, W, b, planes, tol = _p6_inputs(ops, M, N, K, M + 3 * N + K)
    c, _, _ = ops.gemm(A, W, bias=b, prec=6)
    err = (c.double() - planes).abs().max().item()
    assert err < tol, f"vs the planes: {err} (tol {tol})"


def test_gemm_wide_p6_residual_row_map_in_place(ops, cuda):
    """Windowed proj: 2 images x 25 windows x 196 rows (64 x 64 tokens padded to 70 x 70), -1 for the pad tokens, scattered into
    the 2 x 4096 token rows of the residual stream, which is also the output."""
    B, g, ws = 2, 64, 14
    gp = 70
    nw = gp // ws
    y = torch.arange(gp).view(nw, 1, ws, 1).expand(nw, nw, ws, ws)
    x = torch.arange(gp).view(1, nw, 1, ws).expand(nw, nw, ws, ws)
    ok = (y < g) & (x < g)
    rm = torch.full((B, nw, nw, ws, ws), -1, dtype=torch.int32)
    for i in range(B):
        rm[i][ok] = (i * g * g + y * g + x)[ok].int()
    rm = rm.reshape(-1).to(cuda)
    M, N, K = rm.numel(), 1280, 256
    A, W, b, planes, tol = _p6_inputs(ops, M, N, K, 11)
    res = torch.randn(B * g * g, N, device=cuda)
    xs = res.clone()
    ops.gemm(A, W, bias=b, residual=xs, out_f32=xs, row_map=rm, out_rows=B * g * g, prec=6)
    ref = res.double().clone()
    keep = rm >= 0
    ref[rm[keep].long()] += planes[keep]
    assert int(keep.sum()) == B * g * g
    err = (xs.double() - ref).abs().max().item()
    assert err < tol, f"{err} (tol {tol})"


def test_gemm_wide_p6_gelu_planes(ops, cuda):
    """fc1: the GELU epilogue's fp16 + e4m3 planes are exactly the split of its fp32 result (ragged M, N = 1.25 wide tiles)."""
    M, N, K = 1000, 1280 + 320, 256
    A, W, b, planes, tol = _p6_inputs(ops, M, N, K, 5)
    c32, _, _ = ops.gemm(A, W, bias=b, act=ops.ACT_GELU, prec=6)
    gelu = 0.5 * planes * (1.0 + torch.special.erf(planes / math.sqrt(2.0)))
    assert (c32.double() - gelu).abs().max().item() < tol
    _, s, _ = ops.gemm(A, W, bias=b, act=ops.ACT_GELU, want_f32=False, out_e4m3=True, prec=6)
    ref = ops.split_f16_e4m3(c32)
    assert torch.equal(s.hi, ref.hi) and torch.equal(s.lo, ref.lo)


def test_gemm_wide_p4_qk(ops, cuda):
    """qk: A one fp16 plane, W fp16 hi + lo, N = 2560 -> one fp16 plane, equal to the rounded fp32 output of the same call."""
    g = torch.Generator(device="cuda").manual_seed(7)
    M, N, K = 1100, 2560, 1280
    a = torch.randn(M, K, device=cuda, generator=g)
    w = torch.randn(N, K, device=cuda, generator=g) * 0.05
    b = torch.randn(N, device=cuda, generator=g)
    A, W = ops.BF2(a.half(), None), ops.split_weight_f16(w)
    c, s16, _ = ops.gemm(A, W, bias=b, prec=4, want_split=True, out_fp16=True)
    ref = A.hi.double() @ w.double().t() + b.double()
    tol = 3e-5 * math.sqrt(K) * 0.05 * 4 + 1e-5
    err = (c.double() - ref).abs().max().item()
    assert err < tol, f"max err {err} (tol {tol})"
    assert torch.equal(s16.hi, c.half())
    _, only16, _ = ops.gemm(A, W, bias=b, prec=4, want_f32=False, want_split=True, out_fp16=True)
    assert torch.equal(only16.hi, s16.hi)


def test_gemm_p6_rejects_transposed_and_bits(ops, cuda):
    A, W, _, _, _ = _p6_inputs(ops, 128, 256, 64, 3)
    with pytest.raises(RuntimeError):
        ops.gemm(A, W, transposed=True, prec=6)
    with pytest.raises(RuntimeError):
        ops.gemm(A, W, bits_threshold=0.0, prec=6)
