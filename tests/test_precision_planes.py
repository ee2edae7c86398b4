"""CPU: the operand-plane formats of the precision map (DESIGN.md 3), restated in plain torch.

The device kernels (csrc/common.cuh: split4_f16_e4m3, e4m3_slot0; csrc/gemm_tc.cu prec 6) are checked against these formulas in
tests/test_kernels_gpu.py; here the formulas themselves are pinned: the layout of the e4m3 planes, the reconstruction the host
helper BF2.float() performs, and the accuracy class of the fp16 + e4m3 split product against an fp64 product."""
import math

import pytest
import torch

from hipie_b200.ops import BF2


def f8(t):
    return t.clamp(-448.0, 448.0).to(torch.float8_e4m3fn).float()


def split_planes(x, weight=False):
    """(h16 (rows, K) fp16, p8 (rows, 2K) uint8): slot 0 / slot 1 interleaved in 32-column groups, byte (k // 32) * 64 + k % 32 (+ 32)."""
    h = x.half()
    lo = x - h.float()
    s0, s1 = (f8(lo * 2.0 ** 14), f8(h.float() * 2.0 ** 4)) if weight else (f8(h.float()), f8(lo * 2.0 ** 10))
    rows, K = x.shape
    p8 = torch.stack([s0.view(rows, K // 32, 32), s1.view(rows, K // 32, 32)], 2).reshape(rows, 2 * K)
    return h, p8.to(torch.float8_e4m3fn).view(torch.uint8)


def test_plane_layout_and_reconstruction():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(7, 96, generator=g) * torch.logspace(-2, 1.5, 96)
    h, p8 = split_planes(x)
    assert p8.shape == (7, 192) and p8.dtype == torch.uint8
    k = 40                                                   # column 40 lives in group 1: bytes 64 + 8 (slot 0) and 64 + 32 + 8 (slot 1)
    v = p8.view(torch.float8_e4m3fn).float()
    assert torch.equal(v[:, 64 + 8], f8(h.float())[:, k]) and torch.equal(v[:, 64 + 32 + 8], f8((x - h.float()) * 1024.0)[:, k])
    rec = BF2(h, p8).float()                                 # hi + slot 1 / 2^10
    assert (rec - x).abs().max() <= (x.abs() * 2.0 ** -15).max()
    assert (h.float() - x).abs().max() > (rec - x).abs().max() * 8      # the second slot carries ~4 more bits


@pytest.mark.parametrize("K", [256, 1280])
def test_split_product_accuracy_class(K):
    """Ah.Wh + 2^-14 (A8 . W8^T) against the fp64 product: the error class of the three-pass bf16 split (2^-16 per product),
    an order of magnitude below one fp16 pass."""
    g = torch.Generator().manual_seed(K)
    a = torch.randn(64, K, generator=g, dtype=torch.float64).float() * 1.5
    w = torch.randn(48, K, generator=g, dtype=torch.float64).float() * 0.05
    ah, a8 = split_planes(a)
    wh, w8 = split_planes(w, weight=True)
    e = lambda p: p.view(torch.float8_e4m3fn).double()
    split = ah.double() @ wh.double().t() + (e(a8) @ e(w8).t()) * 2.0 ** -14
    exact = a.double() @ w.double().t()
    one_pass = ah.double() @ wh.double().t()
    bf = lambda t: (t.bfloat16().double(), (t - t.bfloat16().float()).bfloat16().double())
    (a1, a2), (w1, w2) = bf(a), bf(w)
    bf16x3 = a1 @ w1.t() + a1 @ w2.t() + a2 @ w1.t()
    err_split, err_one, err_x3 = (split - exact).abs().max().item(), (one_pass - exact).abs().max().item(), (bf16x3 - exact).abs().max().item()
    assert err_split < 6e-5 * math.sqrt(K) * 1.5 * 0.05 * 4
    assert err_split < err_one / 8 and err_split < 4 * err_x3 + 1e-7, (err_split, err_one, err_x3)


FORMATS = {"bf16": (torch.bfloat16, None), "bf16x2": (torch.bfloat16, torch.bfloat16), "f16": (torch.float16, None),
           "f16x2": (torch.float16, torch.float16), "f16+e4m3": (torch.float16, torch.uint8)}


@pytest.mark.parametrize("fmt", sorted(FORMATS))
def test_fmt_is_derived_from_the_plane_dtypes(fmt):
    dhi, dlo = FORMATS[fmt]
    hi = torch.zeros(4, 64, dtype=dhi)
    lo = None if dlo is None else torch.zeros(4, 128 if dlo == torch.uint8 else 64, dtype=dlo)
    assert BF2(hi, lo).fmt == fmt


@pytest.mark.parametrize("dhi,dlo", [(torch.bfloat16, torch.uint8), (torch.bfloat16, torch.float16), (torch.float16, torch.bfloat16),
                                     (torch.float32, None)])
def test_fmt_rejects_an_impossible_pair(dhi, dlo):
    p = BF2(torch.zeros(2, 32, dtype=dhi), None if dlo is None else torch.zeros(2, 32, dtype=dlo))
    with pytest.raises(TypeError):
        p.fmt


@pytest.mark.parametrize("fmt", sorted(FORMATS))
def test_allocators_shape_both_planes(fmt):
    dhi, dlo = FORMATS[fmt]
    for make, zero in ((BF2.empty, False), (BF2.zeros, True)):
        p = make((3, 5, 64), "cpu", fmt)
        assert p.fmt == fmt and p.shape == (3, 5, 64) and p.hi.dtype == dhi
        if dlo is None:
            assert p.lo is None
        else:
            assert p.lo.dtype == dlo and p.lo.shape == ((3, 5, 128) if fmt == "f16+e4m3" else (3, 5, 64))
        if zero:
            assert not p.hi.any() and (p.lo is None or not p.lo.any())


def test_default_allocation_follows_the_precision_mode():
    from hipie_b200 import ops
    prec = ops.PREC
    try:
        ops.set_precision(3)
        assert BF2.empty((2, 8), "cpu").fmt == "bf16x2"
        ops.set_precision(1)
        assert BF2.zeros((2, 8), "cpu").fmt == "bf16"
    finally:
        ops.set_precision(prec)


def test_view_and_row_cut_of_e4m3_planes():
    """view and a cut of leading dimensions commute with the split: the result reconstructs to the numbers of the source cut first."""
    g = torch.Generator().manual_seed(1)
    x = torch.randn(6, 4, 64, generator=g)
    h, p8 = split_planes(x.view(24, 64))
    flat = BF2(h, p8)
    cube = flat.view(6, 4, 64)
    assert cube.hi.shape == (6, 4, 64) and cube.lo.shape == (6, 4, 128) and cube.fmt == "f16+e4m3"
    assert torch.equal(cube.float(), flat.float().view(6, 4, 64))
    assert torch.equal(cube.view(-1, 64).lo, p8)
    for cut in (slice(1, 5), 2, (slice(0, 3), slice(1, 3)), (4, 1)):
        part = cube[cut]
        assert part.lo.shape[-1] == 128
        assert torch.equal(part.float(), BF2(*split_planes(x[cut].reshape(-1, 64))).float().view(x[cut].shape))
    rows = flat[3:11]
    assert torch.equal(rows.hi, h[3:11]) and torch.equal(rows.lo, p8[3:11])


@pytest.mark.parametrize("dims,cut", [((8, 64), (slice(None), slice(0, 32))), ((2, 4, 64), (slice(None), slice(None), slice(0, 32))),
                                      ((2, 4, 64), (Ellipsis, slice(0, 32))), ((2, 4, 64), (0, 0, 0))])
def test_column_cut_of_e4m3_planes_raises(dims, cut):
    planes = BF2(*split_planes(torch.randn(8, 64))).view(*dims)
    with pytest.raises(IndexError):
        planes[cut]


def test_cuts_of_plain_planes_apply_to_each_present_plane():
    x = torch.randn(8, 64)
    both = BF2(x.bfloat16(), (x - x.bfloat16().float()).bfloat16())
    one = BF2(x.half())
    assert torch.equal(both[2:6, 32:].lo, both.lo[2:6, 32:]) and torch.equal(both.view(2, 4, 64).lo, both.lo.view(2, 4, 64))
    assert one[:, :16].lo is None and one.view(-1).lo is None and one.map(lambda t: t.t()).hi.shape == (64, 8)
    assert torch.equal(both[:, 8:24].float(), both.float()[:, 8:24])
