"""CPU: the operand-plane formats of the precision map (DESIGN.md 3), restated in plain torch.

The device kernels (csrc/common.cuh: split4_f16_e4m3, e4m3_slot0; csrc/gemm_tc.cu prec 6) are checked against these formulas in
tests/test_kernels_gpu.py; here the formulas themselves are pinned: the layout of the e4m3 planes, the reconstruction the host
helper BF2.float() performs, the accuracy class of the fp16 + e4m3 split product against an fp64 product, and the operand range that
class holds in (tests/test_precision_range_gpu.py asserts the same range on the device, on the same operands)."""
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


# ---------------------------------------------------------------------------------------------------- the range of the split
# Per product a.w the split drops nothing but Al.Wl (2^-22 |a w|) and rounds the four factors of the two cross terms (each
# <= 2^-11 |a w|) to e4m3, 2^-4 relative at most while they are normal: <= 2^-13 |a w| in the worst case, ~2^-15.5 rms.  Over K
# products with independent errors the sum then carries ~2^-15.5 sqrt(sum p^2) / sum |p| of sum |p|, i.e. 2^-20 at K = 1280 for
# unit-spread operands; max |C - A.W| / (|A|.|W|^T) over a 64 x 48 output comes out at 2^-19 (one fp16 pass: 2^-14.3).  The
# lower end of the range is gradual: RANGE_BOUND is met down to activation rows of max 2^-4 (2^-17.4 there).  Rows dominated by a
# few in-range outlier channels average over fewer products (2^-16.8 with 8 channels at 300) and are held at OUTLIER_BOUND.
#
# The range ends where a factor leaves e4m3's normal range:
#   slot 0 of an activation, e4m3(Ah), saturates at 448 (464 rounds down to it): past that the Ah.Wl term is lost in proportion;
#   slot 1 of an activation, e4m3(2^10 Al) <= 2^-1 |a|, turns subnormal for rows below ~2^-5 and vanishes below ~2^-9;
#   slot 1 of a weight, e4m3(2^4 Wh), saturates at |W| = 28; slot 0, e4m3(2^14 Wl) <= 2^3 |w|, turns subnormal for rows below ~2^-9.
# Outside it the split is still a correction of the fp16 pass: finite and no worse than the fp16 pass alone.
RANGE_BOUND, OUTLIER_BOUND = 2.0 ** -17, 2.0 ** -16


def range_case(kind, value, K=1280, rows=64, cols=48, seed=0):
    """(A, W) fp32 operands of one point of the range: kind "rowmax" (every activation row scaled to max |a| = value), "outliers"
    (8 activation channels at +-value, the rest unit normal), "wrowmax" / "woutliers" (the same on the weight rows / 8 weight
    channels).  Weights are N(0, 0.03^2) where not set otherwise.  Generated on the CPU: the GPU tests feed the same numbers."""
    g = torch.Generator().manual_seed(seed + K)
    a = torch.randn(rows, K, generator=g, dtype=torch.float64).float()
    w = torch.randn(cols, K, generator=g, dtype=torch.float64).float() * 0.03
    idx = torch.randperm(K, generator=g)[:8]
    sign = lambda n: torch.randint(0, 2, (n, 8), generator=g).float() * 2 - 1
    if kind == "rowmax":
        a = a / a.abs().amax(1, keepdim=True) * value
    elif kind == "outliers":
        a[:, idx] = sign(rows) * value
    elif kind == "wrowmax":
        w = w / w.abs().amax(1, keepdim=True) * value
    elif kind == "woutliers":
        w[:, idx] = sign(cols) * value
    else:
        raise ValueError(kind)
    return a, w


def split_errors(a, w):
    """max |C - A.W| / (|A|.|W|^T) of the split product (exact products, fp64 sums) and of the fp16 pass Ah.Wh alone."""
    ah, a8 = split_planes(a)
    wh, w8 = split_planes(w, weight=True)
    e = lambda p: p.view(torch.float8_e4m3fn).double()
    one = ah.double() @ wh.double().t()
    split = one + (e(a8) @ e(w8).t()) * 2.0 ** -14
    exact = a.double() @ w.double().t()
    norm = a.double().abs() @ w.double().abs().t()
    return ((split - exact).abs() / norm).max().item(), ((one - exact).abs() / norm).max().item()


# (kind, value): inside the range
IN_RANGE = [("rowmax", 448.0), ("rowmax", 4.0), ("rowmax", 1.0), ("rowmax", 2.0 ** -2), ("rowmax", 2.0 ** -4), ("wrowmax", 1.0),
            ("wrowmax", 2.0 ** -6)]
IN_RANGE_OUTLIERS = [("outliers", 300.0), ("outliers", 448.0), ("woutliers", 28.0)]
# ... and outside it: activation outliers past 464, activation rows below 2^-6, weight channels past 28, weight rows below 2^-9
OUT_OF_RANGE = [("outliers", 1000.0), ("outliers", 4000.0), ("rowmax", 2.0 ** -7), ("rowmax", 2.0 ** -8), ("woutliers", 40.0),
                ("wrowmax", 2.0 ** -11)]


@pytest.mark.parametrize("kind,value", IN_RANGE + IN_RANGE_OUTLIERS)
@pytest.mark.parametrize("K", [1280, 5120])
def test_split_accuracy_inside_the_range(kind, value, K):
    err, err_one = split_errors(*range_case(kind, value, K))
    bound = OUTLIER_BOUND if "outliers" in kind else RANGE_BOUND
    assert err < bound and err < err_one / 6, (math.log2(err), math.log2(err_one))


@pytest.mark.parametrize("kind,value", OUT_OF_RANGE)
def test_split_accuracy_outside_the_range(kind, value):
    """Past the range the class is lost (the error leaves OUTLIER_BOUND), but the result stays a correction of the fp16 pass."""
    err, err_one = split_errors(*range_case(kind, value))
    assert math.isfinite(err) and err <= err_one, (math.log2(err), math.log2(err_one))
    assert err > OUTLIER_BOUND, math.log2(err)


def test_slot_limits_of_the_split():
    """Where the slots leave e4m3's normal range: slot 0 of an activation holds 416 exactly and saturates at 448 from there on
    (464, the tie between 448 and the unrepresentable 480, rounds down to it); 2^10 Al of a row at 2^-7 is subnormal; slot 1 of a
    weight saturates at |W| = 28."""
    x = torch.tensor([[416.0, 448.0, 464.0, 465.0, 896.0, -1000.0] + [0.0] * 26])
    _, p8 = split_planes(x)
    assert p8.view(torch.float8_e4m3fn).float()[0, :6].tolist() == [416.0, 448.0, 448.0, 448.0, 448.0, -448.0]
    g = torch.Generator().manual_seed(3)
    row = 2.0 ** -7 * (1 + torch.rand(1, 32, generator=g))
    _, p8 = split_planes(row)
    slot1 = p8.view(torch.float8_e4m3fn).float()[0, 32:]
    assert 0 < slot1.abs().max() < 2.0 ** -6                                               # e4m3's smallest normal
    w = torch.tensor([[26.0, 28.0, 28.5, 40.0] + [0.0] * 28])
    _, w8 = split_planes(w, weight=True)
    assert w8.view(torch.float8_e4m3fn).float()[0, 32:36].tolist() == [416.0, 448.0, 448.0, 448.0]


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
