"""GPU: every CUDA kernel of libhipie_b200.so, called through the C-ABI (hipie_b200.ops -> ctypes), against
fp64 / fp32 PyTorch restatements of the same op and the CPU oracle.  Tolerances are written per test."""
import math
import os

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


def test_split(ops, cuda):
    x = torch.randn(4, 1000, device=cuda) * 3
    s = ops.split(x)
    hi, lo = _split_ref(x)
    assert torch.equal(s.hi, hi) and torch.equal(s.lo, lo)
    assert (s.float() - x).abs().max() <= x.abs().max() * 2 ** -16


# ------------------------------------------------------------------------------------------ MSDA
def _msda_inputs(N, Lq, shapes, M, D, P, dev, dtype=torch.float32, seed=0):
    g = torch.Generator().manual_seed(seed)
    shapes_t = torch.as_tensor(shapes, dtype=torch.long)
    S = int(shapes_t.prod(1).sum())
    L = len(shapes)
    value = torch.randn(N, S, M, D, generator=g, dtype=dtype)
    loc = (torch.rand(N, Lq, M, L, P, 2, generator=g, dtype=dtype) * 1.2 - 0.1)
    w = torch.softmax(torch.randn(N, Lq, M, L * P, generator=g, dtype=dtype), -1).view(N, Lq, M, L, P)
    lsi = torch.cat((shapes_t.new_zeros((1,)), shapes_t.prod(1).cumsum(0)[:-1]))
    return value, shapes_t, lsi, loc, w


def test_msda_reference_test_py_fixtures(ops, cuda, golden_dir):
    """The reference's own ops/test.py cases (seed 3; fp64 allclose default, fp32 rtol 1e-2 atol 1e-3)."""
    cases = torch.load(os.path.join(golden_dir, "msda_core.pt"))
    for name, c in cases.items():
        shapes = c["shapes"]
        lsi = torch.cat((shapes.new_zeros((1,)), shapes.prod(1).cumsum(0)[:-1]))
        out = ops.msda_forward(c["value"].to(cuda), shapes.to(cuda), lsi.to(cuda), c["loc"].to(cuda), c["w"].to(cuda)).cpu()
        if c["value"].dtype == torch.float64:
            assert torch.allclose(out, c["out"]), name
        else:
            assert torch.allclose(out, c["out"], rtol=1e-2, atol=1e-3), name
            assert (out - c["out"]).abs().max() < 2e-5, name


@pytest.mark.parametrize("Lq", [1, 33, 910])
def test_msda_fast_vs_oracle(ops, cuda, Lq):
    from hipie_oracle.msda import ms_deform_attn_core
    shapes = [(32, 32), (16, 16), (8, 8), (4, 4)]
    value, shapes_t, lsi, loc, w = _msda_inputs(2, Lq, shapes, 8, 32, 4, cuda, seed=Lq)
    ref = ms_deform_attn_core(value.double(), shapes_t, loc.double(), w.double()).float()
    out = ops.msda_forward(value.to(cuda), shapes_t.to(cuda), lsi.to(cuda), loc.to(cuda), w.to(cuda)).cpu()
    assert (out - ref).abs().max() < 1e-5
    # bf16 value map (fast mode): error bounded by bf16 rounding of value
    outb = ops.msda_forward(value.to(cuda).bfloat16(), shapes_t.to(cuda), lsi.to(cuda), loc.to(cuda), w.to(cuda)).cpu()
    assert (outb - ref).abs().max() < 2e-2


def test_msda_empty_queries(ops, cuda):
    value, shapes_t, lsi, loc, w = _msda_inputs(1, 0, [(4, 4), (2, 2), (2, 2), (1, 1)], 8, 32, 4, cuda)
    out = ops.msda_forward(value.to(cuda), shapes_t.to(cuda), lsi.to(cuda), loc.to(cuda), w.to(cuda))
    assert out.shape == (1, 0, 256)


@pytest.mark.parametrize("ref_dim", [2, 4])
def test_msda_fused_front_half(ops, cuda, ref_dim):
    """softmax + location arithmetic of MSDeformAttn.forward (ms_deform_attn.py:97-109) fused with the core."""
    from hipie_oracle.msda import ms_deform_attn_core
    shapes = [(24, 20), (12, 10), (6, 5), (3, 3)]
    g = torch.Generator().manual_seed(3)
    shapes_t = torch.as_tensor(shapes)
    S = int(shapes_t.prod(1).sum())
    N, Lq, M, L, P = 2, 77, 8, 4, 4
    value = torch.randn(N, S, M * 32, generator=g)
    offs = torch.randn(N, Lq, M, L, P, 2, generator=g) * 2
    logits = torch.randn(N, Lq, M, L * P, generator=g)
    if ref_dim == 2:
        refp = torch.rand(N, Lq, L, 2, generator=g)
        norm = torch.stack([shapes_t[:, 1], shapes_t[:, 0]], -1).float()
        loc = refp[:, :, None, :, None, :] + offs / norm[None, None, None, :, None, :]
    else:
        refp = torch.rand(N, Lq, L, 4, generator=g)
        loc = refp[:, :, None, :, None, :2] + offs / P * refp[:, :, None, :, None, 2:] * 0.5
    w = torch.softmax(logits, -1).view(N, Lq, M, L, P)
    ref = ms_deform_attn_core(value.view(N, S, M, 32).double(), shapes_t, loc.double(), w.double()).float()
    lsi = torch.cat((shapes_t.new_zeros((1,)), shapes_t.prod(1).cumsum(0)[:-1]))
    packed = torch.cat([offs.reshape(N, Lq, -1), logits.reshape(N, Lq, -1)], -1).to(cuda)
    out = ops.msda_fused(value.to(cuda), shapes_t.to(cuda), lsi.to(cuda), packed, refp.to(cuda), want_split=False).cpu()
    assert (out - ref).abs().max() < 2e-5
    s = ops.msda_fused(value.to(cuda), shapes_t.to(cuda), lsi.to(cuda), packed, refp.to(cuda), want_split=True)
    assert (s.float().cpu() - ref).abs().max() < 2e-4
    # IEEE fp16 value map (the encoders' storage format, DESIGN.md 3): exact against the same op on the fp16-rounded values,
    # and within the 2^-12 operand rounding of the fp32 result
    v16 = value.half()
    ref16 = ms_deform_attn_core(v16.float().view(N, S, M, 32).double(), shapes_t, loc.double(), w.double()).float()
    out16 = ops.msda_fused(v16.to(cuda), shapes_t.to(cuda), lsi.to(cuda), packed, refp.to(cuda), want_split=False).cpu()
    assert (out16 - ref16).abs().max() < 2e-5
    assert (out16 - ref).abs().max() < 2.0 ** -11 * value.abs().max()


# ------------------------------------------------------------------------------------------ GEMM
def _gemm_ref(a, w, bias=None, act=0, colscale=None, residual=None, alpha=1.0):
    c = (a.double() @ w.double().transpose(-1, -2)) * alpha
    if bias is not None:
        c = c + bias.double()
    if act == 1:
        c = torch.relu(c)
    elif act == 2:
        c = F.gelu(c)
    elif act == 3:
        c = torch.sigmoid(c)
    if colscale is not None:
        c = c * colscale.double()
    if residual is not None:
        c = c + residual.double()
    return c


@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (256, 512, 128), (300, 256, 256), (4096, 1280, 768), (910, 384, 256),
                                   (77, 4, 256), (130, 100, 40), (1000, 3840, 1280)])
@pytest.mark.parametrize("prec", [3, 1])
def test_gemm_plain(ops, cuda, M, N, K, prec):
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N)
    a = torch.randn(M, K, device=cuda, generator=g)
    w = torch.randn(N, K, device=cuda, generator=g) * 0.05
    A, W = ops.split(a), ops.split_weight(w)
    c, _, _ = ops.gemm(A, W, prec=prec)
    if prec == 3:
        ref = _gemm_ref(a, w)
        tol = 3e-5 * math.sqrt(K) * 0.05 * 4 + 1e-5
    else:
        ref = _gemm_ref(A.hi.float(), W.hi.float())   # exact-input reference: only accumulation order differs
        tol = 1e-4 * math.sqrt(K) * 0.05 + 1e-5
    err = (c.double() - ref).abs().max().item()
    assert err < tol, f"max err {err} (tol {tol})"


def test_gemm_epilogues(ops, cuda):
    g = torch.Generator(device="cuda").manual_seed(1)
    M, N, K = 517, 640, 256
    a = torch.randn(M, K, device=cuda, generator=g)
    w = torch.randn(N, K, device=cuda, generator=g) * 0.06
    bias = torch.randn(N, device=cuda, generator=g)
    cs = torch.rand(N, device=cuda, generator=g)
    res = torch.randn(M, N, device=cuda, generator=g)
    A, W = ops.split(a), ops.split_weight(w)
    for act in (0, 1, 2, 3):
        c, s, _ = ops.gemm(A, W, bias=bias, act=act, colscale=cs, residual=res, alpha=0.5, want_split=True)
        ref = _gemm_ref(a, w, bias, act, cs, res, 0.5)
        assert (c.double() - ref).abs().max() < 2e-4, act
        assert (s.float().double() - ref).abs().max() < 2e-3
        hi, lo = _split_ref(c)
        assert torch.equal(s.hi, hi) and torch.equal(s.lo, lo)
    # in-place residual update (x = x + f(x) pattern)
    x = res.clone()
    ops.gemm(A, W, bias=bias, residual=x, out_f32=x)
    assert (x.double() - _gemm_ref(a, w, bias, residual=res)).abs().max() < 2e-4


def test_gemm_row_map(ops, cuda):
    g = torch.Generator(device="cuda").manual_seed(2)
    M, N, K = 300, 128, 64
    a = torch.randn(M, K, device=cuda, generator=g)
    w = torch.randn(N, K, device=cuda, generator=g) * 0.1
    perm = torch.randperm(M, device=cuda, generator=g).int()
    perm[::7] = -1
    out = torch.full((M, N), 7.0, device=cuda)
    resid = out.clone()
    ops.gemm(ops.split(a), ops.split_weight(w), row_map=perm, residual=resid, out_f32=out)
    ref = _gemm_ref(a, w)
    for r in range(0, M, 13):
        d = int(perm[r])
        if d >= 0:
            assert (out[d].double() - (ref[r] + 7.0)).abs().max() < 1e-4
    untouched = torch.ones(M, dtype=torch.bool, device=cuda)
    untouched[perm[perm >= 0].long()] = False
    assert torch.all(out[untouched] == 7.0)


def test_gemm_batched_transposed_bits(ops, cuda):
    """The mask-embed contraction layout: out[b, q, hw] = sum_c F[b, hw, c] E[b, q, c], + bit-packed threshold."""
    g = torch.Generator(device="cuda").manual_seed(4)
    B, HW, Q, C = 3, 1000, 300, 256
    Fm = torch.randn(B, HW, C, device=cuda, generator=g)
    E = torch.randn(B, Q, C, device=cuda, generator=g) * 0.1
    A, W = ops.split(Fm), ops.split(E)
    c, _, bits = ops.gemm(A, W, M=HW, N=Q, K=C, batch=B, lda=C, ldw=C, a_bstride=HW * C, w_bstride=Q * C,
                          transposed=True, bits_threshold=0.0)
    ref = torch.einsum("bqc,bhc->bqh", E.double(), Fm.double())
    assert c.shape == (B, Q, HW)
    assert (c.double() - ref).abs().max() < 2e-4
    words = (HW + 31) // 32
    got = bits.view(B, Q, words)
    pad = words * 32 - HW
    pred = F.pad((c > 0.0), (0, pad)).view(B, Q, words, 32).long()
    want = (pred << torch.arange(32, device=cuda)).sum(-1)
    want = torch.where(want >= 2 ** 31, want - 2 ** 32, want).int()
    assert torch.equal(got, want)


# ------------------------------------------------------------------------------------------ norms
@pytest.mark.parametrize("C", [256, 768, 1280, 2048, 100])
def test_layernorm(ops, cuda, C):
    x = torch.randn(333, C, device=cuda) * 2 + 0.5
    add = torch.randn(333, C, device=cuda)
    gm = torch.randn(C, device=cuda)
    bt = torch.randn(C, device=cuda)
    y, s, ssum = ops.layernorm(x, gm, bt, 1e-6, add=add, want_f32=True, want_split=True, want_sum=True)
    ref = F.layer_norm((x + add).double(), (C,), gm.double(), bt.double(), 1e-6)
    assert (y.double() - ref).abs().max() < 2e-5
    assert torch.equal(ssum, x + add)
    assert (s.float().double() - ref).abs().max() < 1e-3
    y2, _, _ = ops.layernorm(x, gm, bt, 1e-5, want_f32=True, want_split=False)
    assert (y2.double() - F.layer_norm(x.double(), (C,), gm.double(), bt.double(), 1e-5)).abs().max() < 2e-5


def test_layernorm_row_map(ops, cuda):
    x = torch.randn(50, 256, device=cuda)
    gm, bt = torch.ones(256, device=cuda), torch.zeros(256, device=cuda)
    rmap = (torch.arange(50, device=cuda) * 2 + 1).int()
    out = ops.BF2(torch.zeros(120, 256, dtype=torch.bfloat16, device=cuda), torch.zeros(120, 256, dtype=torch.bfloat16, device=cuda))
    ops.layernorm(x, gm, bt, 1e-6, row_map=rmap, out_split=out)
    ref = F.layer_norm(x, (256,))
    assert (out.float()[1:100:2] - ref).abs().max() < 1e-3
    assert out.float()[0::2].abs().max() == 0


@pytest.mark.parametrize("HW", [64, 1000])
def test_groupnorm_nhwc(ops, cuda, HW):
    x = torch.randn(3, HW, 256, device=cuda) * 3 + 1
    gm, bt = torch.randn(256, device=cuda), torch.randn(256, device=cuda)
    add = torch.randn(3, HW, 256, device=cuda)
    y, s = ops.groupnorm_nhwc(x, gm, bt, relu=True, post_add=add, want_split=True)
    ref = F.relu(F.group_norm(x.double().transpose(1, 2), 32, gm.double(), bt.double(), 1e-5)).transpose(1, 2) + add.double()
    assert (y.double() - ref).abs().max() < 5e-5
    assert (s.float().double() - ref).abs().max() < 1e-3


# ------------------------------------------------------------------------------------------ data movement
def test_patchify_matches_conv(ops, cuda):
    img = torch.rand(2, 3, 64, 96, device=cuda) * 255
    mean, std = [123.675, 116.28, 103.53], [58.395, 57.12, 57.375]
    w = torch.randn(40, 3, 16, 16, device=cuda) * 0.05
    rows = ops.patchify(img, mean, std)
    c, _, _ = ops.gemm(rows, ops.split_weight(w.view(40, -1)))
    xn = (img - torch.tensor(mean, device=cuda).view(1, 3, 1, 1)) / torch.tensor(std, device=cuda).view(1, 3, 1, 1)
    ref = F.conv2d(xn.double(), w.double(), stride=16).permute(0, 2, 3, 1).reshape(-1, 40)
    assert (c.double() - ref).abs().max() < 1e-4


@pytest.mark.parametrize("stride", [1, 2])
def test_im2col_conv3x3(ops, cuda, stride):
    x = torch.randn(2, 10, 12, 16, device=cuda)
    w = torch.randn(24, 16, 3, 3, device=cuda) * 0.1
    cols, Ho, Wo = ops.im2col_nhwc(x, 3, stride, 1)
    wk = w.permute(0, 2, 3, 1).reshape(24, -1).contiguous()       # (ky, kx, c) column order
    c, _, _ = ops.gemm(cols, ops.split_weight(wk))
    ref = F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), stride=stride, padding=1).permute(0, 2, 3, 1).reshape(-1, 24)
    assert (Ho, Wo) == (ref.shape[0] // 2 // ((12 + 2 - 3) // stride + 1), (12 + 2 - 3) // stride + 1)
    assert (c.double() - ref).abs().max() < 1e-4


def test_convtranspose2x2_as_gemm(ops, cuda):
    B, H, W, Ci, Co = 2, 6, 5, 32, 16
    x = torch.randn(B, H, W, Ci, device=cuda)
    wt = torch.randn(Ci, Co, 2, 2, device=cuda) * 0.1
    bias = torch.randn(Co, device=cuda)
    wk = wt.permute(2, 3, 1, 0).reshape(4 * Co, Ci).contiguous()   # rows (dy, dx, co)
    g, _, _ = ops.gemm(ops.split(x.view(-1, Ci)), ops.split_weight(wk), bias=bias.repeat(4))
    y, _ = ops.pixel_shuffle2(g, B, H, W, Co)
    ref = F.conv_transpose2d(x.permute(0, 3, 1, 2).double(), wt.double(), bias.double(), stride=2).permute(0, 2, 3, 1)
    assert (y.double() - ref).abs().max() < 1e-4


def test_maxpool(ops, cuda):
    x = torch.randn(2, 8, 6, 16, device=cuda)
    y, _ = ops.maxpool2_nhwc(x)
    ref = F.max_pool2d(x.permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)
    assert torch.equal(y, ref)


def test_row_softmax(ops, cuda):
    x = torch.randn(2 * 5, 77, device=cuda) * 4
    cb = torch.zeros(2, 77, device=cuda)
    cb[1, 50:] = -9e15
    cb[cb == 0] = 1.0
    p, s = ops.row_softmax(x, colbias=cb, rows_per_batch=5, want_f32=True)
    ref = torch.softmax(x.double().clamp(-5e4, 5e4).view(2, 5, 77) + cb.double()[:, None], -1).view(10, 77)
    assert (p.double() - ref).abs().max() < 1e-6
    p2, _ = ops.row_softmax(x, sub_rowmax=True, want_f32=True, want_split=False)
    xr = x.double()
    ref2 = torch.softmax((xr - xr.max(-1, keepdim=True)[0]).clamp(-5e4, 5e4), -1)
    assert (p2.double() - ref2).abs().max() < 1e-6


@pytest.mark.parametrize("n", [512, 640, 2176, 132])
def test_row_softmax_vectorised(ops, cuda, n):
    """warp-per-row (n <= 1024) and smem-cached block-per-row variants against fp64"""
    g = torch.Generator(device="cuda").manual_seed(n)
    x = torch.randn(3 * 7, n, device=cuda, generator=g) * 4
    cb = torch.ones(3, n, device=cuda)
    cb[1, n // 2:] = -9e15
    p, s = ops.row_softmax(x, colbias=cb, rows_per_batch=7, want_f32=True)
    ref = torch.softmax(x.double().clamp(-5e4, 5e4).view(3, 7, n) + cb.double()[:, None], -1).view(21, n)
    assert (p.double() - ref).abs().max() < 1e-6
    assert ((s.hi.float() + s.lo.float()).double() - ref).abs().max() < 1e-5
    p2, _ = ops.row_softmax(x, sub_rowmax=True, want_f32=True, want_split=False)
    xr = x.double()
    ref2 = torch.softmax((xr - xr.max(-1, keepdim=True)[0]).clamp(-5e4, 5e4), -1)
    assert (p2.double() - ref2).abs().max() < 1e-6


# ------------------------------------------------------------------------------------------ attention
def _attn_ref(q, k, v, scale, rel_h=None, rel_w=None, kh=0, kw=0, key_bias=None):
    # q,k,v: (B,H,T,hd) double
    s = (q * scale) @ k.transpose(-1, -2)
    if rel_h is not None:
        B, H, Tq, _ = q.shape
        s = (s.view(B, H, Tq, kh, kw) + rel_h.double()[..., :, None] + rel_w.double()[..., None, :]).view(B, H, Tq, kh * kw)
    if key_bias is not None:
        s = s + key_bias.double()[:, None, None, :]
    return torch.softmax(s, -1) @ v


@pytest.mark.parametrize("hd,H", [(80, 4), (64, 3), (32, 8)])
@pytest.mark.parametrize("Tq,Tk", [(196, 196), (64, 64), (100, 300), (910, 910)])
@pytest.mark.parametrize("prec", [3, 1])
def test_attention(ops, cuda, hd, H, Tq, Tk, prec):
    g = torch.Generator(device="cuda").manual_seed(hd + Tq)
    B = 2
    qkv = torch.randn(B, max(Tq, Tk), 3, H, hd, device=cuda, generator=g)
    S = ops.split(qkv)
    q, k, v = S[:, :Tq, 0], S[:, :Tk, 1], S[:, :Tk, 2]
    ts, bs = 3 * H * hd, max(Tq, Tk) * 3 * H * hd
    kb = None
    if Tk == 300:
        kb = torch.zeros(B, Tk, device=cuda)
        kb[1, 250:] = -1e9
    o, _ = ops.attention(ops.BF2(q.hi, q.lo), ops.BF2(k.hi, k.lo), ops.BF2(v.hi, v.lo), B, H, Tq, Tk, hd,
                         (bs, ts, hd), (bs, ts, hd), (bs, ts, hd), hd ** -0.5, key_bias=kb, want_f32=True,
                         want_split=False, prec=prec)
    if prec == 3:
        qq, kk, vv = (qkv[:, :Tq, 0], qkv[:, :Tk, 1], qkv[:, :Tk, 2])
    else:
        qq, kk, vv = (S.hi[:, :Tq, 0].float(), S.hi[:, :Tk, 1].float(), S.hi[:, :Tk, 2].float())
    ref = _attn_ref(qq.permute(0, 2, 1, 3).double(), kk.permute(0, 2, 1, 3).double(), vv.permute(0, 2, 1, 3).double(),
                    hd ** -0.5, key_bias=kb).permute(0, 2, 1, 3).reshape(B, Tq, H * hd)
    err = (o.double() - ref).abs().max().item()
    assert err < (2e-5 if prec == 3 else 2e-2), err


def test_attention_decomposed_relpos(ops, cuda):
    """rel-pos tables built by relpos_bias + fused attention == Attention.forward with add_decomposed_rel_pos."""
    g = torch.Generator(device="cuda").manual_seed(9)
    B, H, hd, gh, gw = 2, 4, 80, 14, 14
    T = gh * gw
    qkv = torch.randn(B, T, 3, H, hd, device=cuda, generator=g)
    Rh = torch.randn(gh, gh, hd, device=cuda, generator=g) * 0.2     # get_rel_pos output (q, k, c)
    Rw = torch.randn(gw, gw, hd, device=cuda, generator=g) * 0.2
    S = ops.split(qkv)
    ts, bs = 3 * H * hd, T * 3 * H * hd
    qs = ops.BF2(S.hi[:, :, 0], S.lo[:, :, 0])
    rel_h = ops.relpos_bias(qs, (bs, ts, hd), Rh.permute(0, 2, 1).contiguous(), 0, gh, gw, B, H, hd)
    rel_w = ops.relpos_bias(qs, (bs, ts, hd), Rw.permute(0, 2, 1).contiguous(), 1, gh, gw, B, H, hd)
    q = qkv[:, :, 0].permute(0, 2, 1, 3).double()
    rq = q.reshape(B, H, gh, gw, hd)
    ref_h = torch.einsum("bnhwc,hkc->bnhwk", rq, Rh.double()).reshape(B, H, T, gh)
    ref_w = torch.einsum("bnhwc,wkc->bnhwk", rq, Rw.double()).reshape(B, H, T, gw)
    assert (rel_h.double() - ref_h).abs().max() < 1e-4
    assert (rel_w.double() - ref_w).abs().max() < 1e-4
    # tensor-core variant (the one the engine uses)
    th = ops.relpos_bias_tc(qs, (bs, ts, hd), ops.split_weight(Rh), 0, gh, gw, B, H, hd)
    tw = ops.relpos_bias_tc(qs, (bs, ts, hd), ops.split_weight(Rw), 1, gh, gw, B, H, hd)
    assert (th.double() - ref_h).abs().max() < 1e-4
    assert (tw.double() - ref_w).abs().max() < 1e-4
    o, _ = ops.attention(qs, ops.BF2(S.hi[:, :, 1], S.lo[:, :, 1]), ops.BF2(S.hi[:, :, 2], S.lo[:, :, 2]), B, H, T, T, hd,
                         (bs, ts, hd), (bs, ts, hd), (bs, ts, hd), hd ** -0.5, rel_h=rel_h, rel_w=rel_w, kh=gh, kw=gw,
                         want_f32=True, want_split=False)
    ref = _attn_ref(q, qkv[:, :, 1].permute(0, 2, 1, 3).double(), qkv[:, :, 2].permute(0, 2, 1, 3).double(), hd ** -0.5,
                    ref_h, ref_w, gh, gw).permute(0, 2, 1, 3).reshape(B, T, H * hd)
    assert (o.double() - ref).abs().max() < 3e-5


@pytest.mark.parametrize("prec", [3, 1])
@pytest.mark.parametrize("with_rel", [True, False])
def test_attention_tcgen05(ops, cuda, prec, with_rel):
    """wgmma flash attention (global ViT-H blocks) vs fp64 softmax attention; V supplied transposed."""
    g = torch.Generator(device="cuda").manual_seed(21 + prec)
    B, H, hd, gh, gw = 2, 3, 80, 4, 64          # T = 256 tokens: 2 query tiles x 4 key tiles
    T, E = gh * gw, H * hd
    qk = torch.randn(B * T, 2 * E, device=cuda, generator=g)
    v = torch.randn(B * T, E, device=cuda, generator=g)
    S, Vs = ops.split(qk), ops.split(v.t().contiguous())          # vt: (E, B*T)
    q = ops.BF2(S.hi[:, :E], S.lo[:, :E])
    k = ops.BF2(S.hi[:, E:], S.lo[:, E:])
    rel_h = rel_w = None
    if with_rel:
        rel_h = torch.randn(B, H, T, gh, device=cuda, generator=g)
        rel_w = torch.randn(B, H, T, gw, device=cuda, generator=g)
    o, _ = ops.attention_tc(q, k, Vs, B, H, T, hd, T * 2 * E, 2 * E, T * 2 * E, 2 * E, hd ** -0.5, rel_h=rel_h, rel_w=rel_w,
                            kh=gh, kw=gw, want_f32=True, want_split=False, prec=prec)
    if prec == 3:
        qq, kk, vv = qk[:, :E], qk[:, E:], v
    else:
        qq, kk, vv = S.hi[:, :E].float(), S.hi[:, E:].float(), Vs.hi.float().t()
    sh = lambda x: x.reshape(B, T, H, hd).permute(0, 2, 1, 3).double()
    ref = _attn_ref(sh(qq), sh(kk), sh(vv), hd ** -0.5, rel_h, rel_w, gh, gw).permute(0, 2, 1, 3).reshape(B, T, E)
    err = (o.double() - ref).abs().max().item()
    assert err < (3e-5 if prec == 3 else 3e-2), err


@pytest.mark.parametrize("prec", [3, 2])
def test_attention_tcgen05_80_wide_grid(ops, cuda, prec):
    """1280-pixel inputs give an 80-wide token grid: the kernel keeps its 64-key tiles, so a tile starts at grid column (64 j) mod 80
    and straddles two key rows in 3 of the 5 phases (rel_w index rotation + two rel_h scalars per tile); vs fp64 attention."""
    g = torch.Generator(device="cuda").manual_seed(51 + prec)
    B, H, hd, gh, gw = 2, 2, 80, 16, 80          # T = 1280 tokens: 5 query tile pairs x 20 key tiles (4 periods of 5 phases)
    T, E = gh * gw, H * hd
    qk = torch.randn(B * T, 2 * E, device=cuda, generator=g)
    v = torch.randn(B * T, E, device=cuda, generator=g)
    rel_h = torch.randn(B, H, T, gh, device=cuda, generator=g)
    rel_w = torch.randn(B, H, T, gw, device=cuda, generator=g)
    if prec == 3:
        S, Vs = ops.split(qk), ops.split(v.t().contiguous())
        q, k = ops.BF2(S.hi[:, :E], S.lo[:, :E]), ops.BF2(S.hi[:, E:], S.lo[:, E:])
        qq, kk, vv, tol = qk[:, :E], qk[:, E:], v, 3e-5
    else:
        qk16, vt16 = qk.half(), v.t().contiguous().half()
        q, k, Vs = ops.BF2(qk16[:, :E], None), ops.BF2(qk16[:, E:], None), ops.BF2(vt16, None)
        qq, kk, vv, tol = qk16[:, :E].float(), qk16[:, E:].float(), vt16.float().t(), 2e-3     # P is rounded to fp16 (2^-11)
    o, _ = ops.attention_tc(q, k, Vs, B, H, T, hd, T * 2 * E, 2 * E, T * 2 * E, 2 * E, hd ** -0.5, rel_h=rel_h, rel_w=rel_w,
                            kh=gh, kw=gw, want_f32=True, want_split=False, prec=prec if prec == 3 else None, f16=prec == 2)
    sh = lambda x: x.reshape(B, T, H, hd).permute(0, 2, 1, 3).double()
    ref = _attn_ref(sh(qq), sh(kk), sh(vv), hd ** -0.5, rel_h, rel_w, gh, gw).permute(0, 2, 1, 3).reshape(B, T, E)
    err = (o.double() - ref).abs().max().item()
    assert err < tol, err
    with pytest.raises(RuntimeError):          # 80-wide but T % 320 != 0: refused, the caller falls back to the mma.sync kernel
        ops.attention_tc(q, k, Vs, B, H, 1024, hd, T * 2 * E, 2 * E, T * 2 * E, 2 * E, hd ** -0.5, rel_h=rel_h, rel_w=rel_w,
                         kh=1024 // 80, kw=80, want_f32=True, want_split=False, prec=prec if prec == 3 else None, f16=prec == 2)


def test_relpos_tc_global_grid(ops, cuda):
    g = torch.Generator(device="cuda").manual_seed(11)
    B, H, hd, gh, gw = 1, 2, 80, 64, 64
    T = gh * gw
    qkv = torch.randn(B, T, 3, H, hd, device=cuda, generator=g)
    Rh = torch.randn(gh, gh, hd, device=cuda, generator=g) * 0.2
    Rw = torch.randn(gw, gw, hd, device=cuda, generator=g) * 0.2
    S = ops.split(qkv)
    ts, bs = 3 * H * hd, T * 3 * H * hd
    qs = ops.BF2(S.hi[:, :, 0], S.lo[:, :, 0])
    th = ops.relpos_bias_tc(qs, (bs, ts, hd), ops.split_weight(Rh), 0, gh, gw, B, H, hd)
    tw = ops.relpos_bias_tc(qs, (bs, ts, hd), ops.split_weight(Rw), 1, gh, gw, B, H, hd)
    rq = qkv[:, :, 0].permute(0, 2, 1, 3).double().reshape(B, H, gh, gw, hd)
    ref_h = torch.einsum("bnhwc,hkc->bnhwk", rq, Rh.double()).reshape(B, H, T, gh)
    ref_w = torch.einsum("bnhwc,wkc->bnhwk", rq, Rw.double()).reshape(B, H, T, gw)
    assert (th.double() - ref_h).abs().max() < 2e-4
    assert (tw.double() - ref_w).abs().max() < 2e-4


@pytest.mark.parametrize("prec", [3, 1])
def test_attention_tcgen05_window_mode(ops, cuda, prec):
    """14x14-window mode of the wgmma attention kernel: 196 tokens per (window, head), keys padded to 4x64 and masked,
    decomposed rel-pos bias rel_h[q, k // 14] + rel_w[q, k % 14]; vs fp64 softmax attention."""
    g = torch.Generator(device="cuda").manual_seed(31 + prec)
    B, H, hd, gh, gw = 5, 3, 80, 14, 14          # 5 windows
    T, E = gh * gw, H * hd
    qk = torch.randn(B * T, 2 * E, device=cuda, generator=g)
    v = torch.randn(B * T, E, device=cuda, generator=g)
    S = ops.split(qk)
    vpad = torch.zeros(E, B, 200, device=cuda)                    # vt: every window at a 200-column pitch, pad columns zero
    vpad[:, :, :T] = v.t().reshape(E, B, T)
    Vs = ops.split(vpad.view(E, B * 200))
    q = ops.BF2(S.hi[:, :E], S.lo[:, :E])
    k = ops.BF2(S.hi[:, E:], S.lo[:, E:])
    rel_h = torch.randn(B, H, T, gh, device=cuda, generator=g)
    rel_w = torch.randn(B, H, T, gw, device=cuda, generator=g)
    o, _ = ops.attention_tc(q, k, Vs, B, H, T, hd, T * 2 * E, 2 * E, T * 2 * E, 2 * E, hd ** -0.5, rel_h=rel_h, rel_w=rel_w,
                            kh=gh, kw=gw, want_f32=True, want_split=False, prec=prec)
    if prec == 3:
        qq, kk, vv = qk[:, :E], qk[:, E:], v
    else:
        qq, kk, vv = S.hi[:, :E].float(), S.hi[:, E:].float(), Vs.hi.float().view(E, B, 200)[:, :, :T].reshape(E, B * T).t()
    sh = lambda x: x.reshape(B, T, H, hd).permute(0, 2, 1, 3).double()
    ref = _attn_ref(sh(qq), sh(kk), sh(vv), hd ** -0.5, rel_h, rel_w, gh, gw).permute(0, 2, 1, 3).reshape(B, T, E)
    err = (o.double() - ref).abs().max().item()
    assert err < (3e-5 if prec == 3 else 3e-2), err


# ------------------------------------------------------------------------------------------ CondInst
def test_condinst_fused(ops, cuda):
    from hipie_oracle.condinst import dynamic_mask_with_coords
    g = torch.Generator().manual_seed(2)
    B, Q, Hf, Wf = 2, 9, 12, 10
    feats = torch.randn(B, 8, Hf, Wf, generator=g)
    params = torch.randn(B, Q, 169, generator=g) * 0.3
    ref_px = torch.rand(B, Q, 2, generator=g) * 80
    ref = dynamic_mask_with_coords(feats, ref_px, params, stride=8)       # (B, Q, 2Hf, 2Wf)
    out = ops.condinst_masks(feats.permute(0, 2, 3, 1).contiguous().to(cuda), params.to(cuda), ref_px.to(cuda), Hf, Wf).cpu()
    assert (out - ref).abs().max() < 2e-3 * ref.abs().max()


# ------------------------------------------------------------------------------------------ fused semantic / panoptic
@pytest.mark.parametrize("Q,C,h,w,Hc,Wc", [(70, 13, 24, 20, 90, 77), (200, 100, 16, 16, 64, 64), (64, 80, 12, 40, 48, 160)])
def test_seg_postprocess_fused(ops, cuda, Q, C, h, w, Hc, Wc):
    """hipie_seg_postprocess vs the reference op chain (upsample x4 -> crop -> sigmoid -> einsum / argmax / areas,
    H/models/hipie_img.py:880-1023) evaluated on the CPU in fp64."""
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(Q + C)
    masks = torch.randn(Q, h, w, generator=g) * 4
    cls = F.softmax(torch.randn(Q, C, generator=g) * 3, dim=-1)
    thr = 0.25
    sem, ids, areas, scores, labels = ops.seg_postprocess(masks.to(cuda), cls.to(cuda), thr, Hc, Wc)
    up = F.interpolate(masks[:, None], size=(4 * h, 4 * w), mode="bilinear", align_corners=False)[:, 0, :Hc, :Wc]
    sg = up.double().sigmoid()
    sem_ref = torch.einsum("qc,qhw->chw", cls.double(), sg)
    assert (sem.cpu().double() - sem_ref).abs().max() < 2e-4 * max(1.0, float(sem_ref.abs().max()))
    sc, lb = cls.max(-1)
    assert torch.equal(lb, labels.cpu())
    keep = sc > thr
    kidx = keep.nonzero()[:, 0]
    ids_c = ids.cpu().long()
    if kidx.numel() == 0:
        assert (ids_c == -1).all()
        return
    prob = sc[keep].double().view(-1, 1, 1) * sg[keep]
    win = kidx[prob.argmax(0)]
    got = ids_c >> 1
    mism = got != win
    # near-ties may resolve differently in fp32; wherever the winner differs the two products must be equal to 1e-5
    if mism.any():
        pg = (sc[got[mism]].double() * sg[got[mism], mism.nonzero()[:, 0], mism.nonzero()[:, 1]])
        pw = prob.max(0)[0][mism]
        assert (pg - pw).abs().max() < 1e-5 and mism.float().mean() < 1e-3
    inter_flag = (ids_c & 1).bool()
    sg_w = sg.gather(0, got.unsqueeze(0))[0]
    assert ((sg_w >= 0.5) != inter_flag).float().mean() < 1e-3
    own = got.unsqueeze(0) == torch.arange(Q).view(Q, 1, 1)
    ref_area = torch.stack([own.flatten(1).sum(1), (sg >= 0.5).flatten(1).sum(1), (own & (sg >= 0.5)).flatten(1).sum(1)])
    a = areas.cpu().long()
    assert (a[:, keep] - ref_area[:, keep]).abs().max() <= 2
    assert (a[1] - ref_area[1]).abs().max() <= 2


@pytest.mark.parametrize("N,h,w,Hc,Wc", [(7, 24, 20, 90, 77), (3, 16, 16, 64, 64), (0, 8, 8, 32, 32)])
def test_upsample_threshold(ops, cuda, N, h, w, Hc, Wc):
    """instance-mask kernel vs F.interpolate(bilinear, x4) -> sigmoid -> > thr -> crop (hipie_img.py:1003-1007)"""
    import torch.nn.functional as F
    g = torch.Generator(device="cuda").manual_seed(N + h)
    m = torch.randn(N, h, w, device=cuda, generator=g) * 3
    for thr in (0.5, 0.3):
        out = ops.upsample_threshold(m, thr, Hc, Wc)
        assert out.dtype == torch.bool and tuple(out.shape) == (N, Hc, Wc)
        if N == 0:
            continue
        up = F.interpolate(m[:, None], size=(4 * h, 4 * w), mode="bilinear", align_corners=False)[:, 0, :Hc, :Wc]
        ref = up.sigmoid() > thr
        # pixels whose logit is within rounding of the threshold may flip; everything else must agree
        margin = (up.double().sigmoid() - thr).abs() > 1e-6
        assert torch.equal(out[margin], ref[margin])
        assert (out != ref).float().mean() < 1e-4


def test_sine_embed(ops, cuda):
    """fused reference-point sine embedding vs the reference op chain (deformable_transformer_dino.py:636-670)"""
    import math
    g = torch.Generator(device="cuda").manual_seed(5)
    pos_full = torch.rand(2, 37, 4, 4, device=cuda, generator=g)
    pos = pos_full[:, :, 0, :]                                   # strided rows, like ref_in[:, :, 0, :]
    out, s = ops.sine_embed(pos, want_f32=True, want_split=True)
    dim_t = torch.arange(128, dtype=torch.float32, device=cuda)
    dim_t = 10000 ** (2 * torch.div(dim_t, 2, rounding_mode="floor") / 128)
    def emb(v):
        p = (v * (2 * math.pi))[..., None] / dim_t
        return torch.stack((p[..., 0::2].sin(), p[..., 1::2].cos()), dim=-1).flatten(-2)
    ref = torch.cat([emb(pos[..., 1]), emb(pos[..., 0]), emb(pos[..., 2]), emb(pos[..., 3])], dim=-1).view(-1, 512)
    assert (out - ref).abs().max() < 2e-6
    assert ((s.hi.float() + s.lo.float()) - ref).abs().max() < 1e-4


def test_gemm_row_major_bits_short_wide(ops, cuda):
    """short-and-wide batched GEMM (the mask-embed shape class: M = 300 queries = 3 M tiles with a ragged last one, N = pixels):
    N = 1536 is 12 = 4 x 3 N tiles, the smallest width that runs the M-fastest tile order (launch_gemm: tiles_m <= 8 and
    tiles_n >= 4 tiles_m); fp32 rows + fused (x > 0) bit-packed along N"""
    g = torch.Generator(device="cuda").manual_seed(77)
    B, M, N, K = 2, 300, 1536, 256
    a = torch.randn(B * M, K, device=cuda, generator=g)
    w = torch.randn(B * N, K, device=cuda, generator=g) * 0.1
    A, W = ops.split(a), ops.split(w)
    c, _, bits = ops.gemm(A, W, M=M, N=N, K=K, batch=B, lda=K, ldw=K, a_bstride=M * K, w_bstride=N * K, bits_threshold=0.0)
    ref = torch.einsum("bmk,bnk->bmn", a.view(B, M, K).double(), w.view(B, N, K).double())
    assert (c.double() - ref).abs().max() < 2e-4
    want = (c > 0).view(B, M, N // 32, 32).long().cpu()
    want = (want << torch.arange(32)).sum(-1)
    want = torch.where(want >= 2 ** 31, want - 2 ** 32, want).int()
    assert torch.equal(bits.cpu().view(B, M, N // 32), want)


# ------------------------------------------------------------------------------------------------ selection kernels (a20)
@pytest.mark.parametrize("max_pool", [False, True])
def test_class_scores_matches_reference_loop(cuda, max_pool):
    """hipie_class_scores against the reference's per-class host loop (hipie_img.py:1025-1052, restated in the oracle)."""
    from hipie_oracle.model import HipieOracle
    from hipie_b200 import ops
    g = torch.Generator().manual_seed(0)
    R, Lt, C = 37, 64, 11
    pos_map, cur = {}, 1
    for c in range(1, C + 1):
        if c == 4:
            continue                                   # a class missing from the positive map keeps score 0
        n = 1 + (c % 3)
        pos_map[c] = list(range(cur, cur + n))
        cur += n + 1
    is_thing = {c: c % 2 == 1 for c in range(1, C + 1)}
    logits = torch.randn(2, R, Lt, generator=g) * 3
    iou = torch.randn(2, R, 1, generator=g)
    maxlen = max(len(v) for v in pos_map.values())
    tok = torch.zeros(C, maxlen, dtype=torch.int32)
    cnt = torch.zeros(C, dtype=torch.int32)
    fg = torch.zeros(C, dtype=torch.int8)
    for c, t in pos_map.items():
        tok[c - 1, :len(t)] = torch.tensor(t, dtype=torch.int32)
        cnt[c - 1] = len(t)
        fg[c - 1] = 0 if is_thing[c] else 1
    ref = HipieOracle.convert_grounding_to_od_logits(logits, C, pos_map, is_thing, mode="FG", max_pool=max_pool)
    ref_prob = torch.sqrt(ref.sigmoid() * iou.sigmoid())
    sc, prob, rmax, rarg = ops.class_scores(logits.view(-1, Lt).cuda(), tok.cuda(), cnt.cuda(), masked=fg.cuda(), iou=iou.view(-1).cuda(),
                                            max_pool=max_pool)
    assert torch.allclose(sc.cpu().view(2, R, C), ref, atol=1e-6)
    assert torch.allclose(prob.cpu().view(2, R, C), ref_prob, atol=1e-6)
    m, a = ref_prob.view(-1, C).max(1)
    assert torch.allclose(rmax.cpu(), m, atol=1e-6) and torch.equal(rarg.cpu().long(), a)
    sc2, _, _, _ = ops.class_scores(logits.view(-1, Lt).cuda(), tok.cuda(), cnt.cuda(), masked=None, iou=None, max_pool=max_pool, want_prob=False)
    assert torch.allclose(sc2.cpu().view(2, R, C), HipieOracle.convert_grounding_to_od_logits(logits, C, pos_map, is_thing, mode=None, max_pool=max_pool), atol=1e-6)


@pytest.mark.parametrize("N", [1, 37, 900])
def test_batched_nms_matches_torchvision(cuda, N):
    """hipie_batched_nms against torchvision.ops.batched_nms (what the reference calls, hipie_img.py:629) incl. near-duplicate
    boxes, several classes and equal scores."""
    import torchvision.ops as tvops
    from hipie_b200 import ops
    g = torch.Generator().manual_seed(N)
    B = 3
    boxes = torch.cat([torch.rand(B, N, 2, generator=g) * 0.6 + 0.2, torch.rand(B, N, 2, generator=g) * 0.3 + 0.05], -1)
    if N > 10:
        boxes[:, N // 2:N // 2 + N // 4] = boxes[:, :N // 4] + torch.randn(B, N // 4, 4, generator=g) * 0.01     # heavy overlaps
    scores = torch.rand(B, N, generator=g)
    if N > 10:
        scores[:, 5] = scores[:, 3]                                                                              # an exact tie
    cls = torch.randint(0, 4, (B, N), generator=g, dtype=torch.int32)
    keep, nkeep = ops.batched_nms(boxes.cuda(), scores.cuda(), cls.cuda(), 0.7)
    for b in range(B):
        cx, cy, w, h = boxes[b].unbind(-1)
        xyxy = torch.stack([cx - 0.5 * w, cy - 0.5 * h, cx + 0.5 * w, cy + 0.5 * h], -1)
        ref = tvops.batched_nms(xyxy, scores[b], cls[b].long(), 0.7)
        n = int(nkeep[b])
        assert n == len(ref), (n, len(ref))
        assert torch.equal(keep[b, :n].cpu().long(), ref)
        assert bool((keep[b, n:] == -1).all())


@pytest.mark.parametrize("n,k", [(50, 100), (2400, 100), (21760, 900), (700000, 100)])
def test_topk_matches_torch(cuda, n, k):
    from hipie_b200 import ops
    g = torch.Generator().manual_seed(n)
    v = torch.randn(3, n, generator=g)
    v[1, : n // 2] = v[1, n // 2: n // 2 * 2]            # many exact ties
    v[2, ::3] = -9999.0
    ov, oi = ops.topk(v.cuda(), k)
    kk = min(k, n)
    rv, ri = torch.topk(v, kk, dim=1)
    assert torch.equal(ov[:, :kk].cpu(), rv)
    # indices: same values, and among equal values the lowest index first
    assert torch.equal(torch.gather(v, 1, oi[:, :kk].cpu().long()), rv)
    for r in range(3):
        idx = oi[r, :kk].cpu().long()
        assert len(set(idx.tolist())) == kk
        same = rv[r, 1:] == rv[r, :-1]
        assert bool((idx[1:][same] > idx[:-1][same]).all())
    if k > n:
        assert bool((oi[:, n:] == -1).all()) and bool(torch.isinf(ov[:, n:]).all())
    # device-side row count: only the first 7 rows x 10 columns of a compacted matrix are valid
    if n >= 100:
        nr = torch.tensor([7, 0, 3], dtype=torch.int32)
        ov2, oi2 = ops.topk(v.cuda(), 20, n_rows=nr.cuda(), n_cols_per_row=10)
        assert torch.equal(ov2[0].cpu(), torch.topk(v[0, :70], 20)[0]) and bool((oi2[1] == -1).all())
        assert torch.equal(ov2[2].cpu(), torch.topk(v[2, :30], 20)[0])


def test_seg_postprocess_wide_vocabulary(cuda):
    """C = 150 and 847 classes (ADE-150 / ADE-847): class chunks of the fused kernel against the op chain."""
    from hipie_b200 import ops
    g = torch.Generator().manual_seed(5)
    for C, Q in ((150, 70), (847, 40)):
        masks = torch.randn(Q, 24, 32, generator=g) * 4
        cls = torch.softmax(torch.randn(Q, C, generator=g) * 3, -1)
        sem, ids, areas, scores, labels = ops.seg_postprocess(masks.cuda(), cls.cuda(), 0.25, 96, 120)
        up = torch.nn.functional.interpolate(masks[None], size=(96, 128), mode="bilinear", align_corners=False)[0][:, :, :120].sigmoid()
        ref = torch.einsum("qc,qhw->chw", cls, up)
        assert (sem.cpu() - ref).abs().max() < 1e-3 * max(1.0, ref.abs().max().item())
        sc, lb = cls.max(-1)
        keep = sc > 0.25
        prob = torch.where(keep[:, None, None], sc[:, None, None] * up, torch.full_like(up, -1.0))
        win = prob.argmax(0)
        got = ids.cpu()
        assert ((got >> 1) == win).float().mean() > 0.999 or not keep.any()


# ------------------------------------------------------------------------------------------ single-pass fp16 attention path
def test_gemm_fp16_plane_output(ops, cuda):
    """hipie_gemm with c_fp16: the epilogue rounds the fp32 result to ONE IEEE fp16 plane (row-major through both store paths and
    transposed with the window row padding)."""
    g = torch.Generator(device="cuda").manual_seed(3)
    M, N, K = 1024, 320, 256
    a, w, b = torch.randn(M, K, device=cuda, generator=g), torch.randn(N, K, device=cuda, generator=g) * 0.1, torch.randn(N, device=cuda, generator=g)
    A, W = ops.split(a), ops.split_weight(w)
    ref32, _, _ = ops.gemm(A, W, bias=b)
    for tma in (1, 0):
        _lib_set("gemm_tma_store", tma)
        _, s, _ = ops.gemm(A, W, bias=b, want_f32=False, want_split=True, out_fp16=True)
        assert s.hi.dtype == torch.float16 and s.lo is None
        assert torch.equal(s.hi, ref32.half())
    _lib_set("gemm_tma_store", 1)
    _, st, _ = ops.gemm(A, W, bias=b, want_f32=False, want_split=True, transposed=True, out_fp16=True)
    assert torch.equal(st.hi, ref32.t().half())


def _lib_set(name, v):
    from hipie_b200 import _lib
    _lib.set_option(name, v)


@pytest.mark.parametrize("M,N,K", [(256, 256, 64), (4096, 2560, 1280), (2048, 1280, 1280), (1000, 100, 512), (3000, 384, 256), (130, 40, 64)])
def test_gemm_two_pass_fp16(ops, cuda, M, N, K):
    """prec 4 (the qkv linears, DESIGN.md 3): A is ONE fp16 plane, W is fp16 hi + lo, two MMA passes.  Against fp64 on the SAME
    fp16-rounded activation the result is fp32-class (the weight is exact to ~2^-22); all tile variants (CTA pairs / single, BN 256 / 128)."""
    g = torch.Generator(device="cuda").manual_seed(M + 3 * N + K)
    a = torch.randn(M, K, device=cuda, generator=g)
    w = torch.randn(N, K, device=cuda, generator=g) * 0.05
    b = torch.randn(N, device=cuda, generator=g)
    A = ops.BF2(a.half(), None)
    W = ops.split_weight_f16(w)
    c, s16, _ = ops.gemm(A, W, bias=b, prec=4, want_split=True, out_fp16=True)
    ref = _gemm_ref(A.hi.float(), w, bias=b)
    tol = 3e-5 * math.sqrt(K) * 0.05 * 4 + 1e-5
    err = (c.double() - ref).abs().max().item()
    assert err < tol, f"max err {err} (tol {tol})"
    assert torch.equal(s16.hi, c.half())
    ct, _, _ = ops.gemm(A, W, bias=b, prec=4, transposed=True)
    assert (ct.t().double() - ref).abs().max().item() < tol
    with pytest.raises(RuntimeError):
        ops.gemm(A, ops.BF2(W.hi, None), prec=4)


def test_gemm_transposed_fp16_vectorised_epilogue(ops, cuda):
    """The V^T epilogue (transposed fp16 plane) stores 8 (plain) or 4 (per-window row padding) rows per lane through shared memory: it
    must write exactly what the scalar epilogue writes, including the untouched pad columns, ragged N and prec 3 / 4 operands."""
    g = torch.Generator(device="cuda").manual_seed(77)
    for (M, N, K, grp, pad) in ((2048, 320, 256, 0, 0), (8 * 196, 200, 128, 196, 4), (4096, 1280, 1280, 0, 0), (25 * 196, 1280, 256, 196, 4)):
        a, w, b = torch.randn(M, K, device=cuda, generator=g), torch.randn(N, K, device=cuda, generator=g) * 0.1, torch.randn(N, device=cuda, generator=g)
        ld = M if grp == 0 else (M // grp) * (grp + pad)
        for prec, A, W in ((3, ops.split(a), ops.split_weight(w)), (4, ops.BF2(a.half(), None), ops.split_weight_f16(w))):
            outs = []
            for fast in (0, 1):
                _lib_set("gemm_fast_transposed", fast)
                buf = ops.BF2(torch.full((N, ld), 7.0, dtype=torch.float16, device=cuda), None)
                ops.gemm(A, W, bias=b, want_f32=False, transposed=True, ldc=ld, out_split=buf, t_row_group=grp, t_row_pad=pad if grp else 0,
                         out_fp16=True, prec=prec)
                outs.append(buf.hi.clone())
            _lib_set("gemm_fast_transposed", 1)
            assert torch.equal(outs[0], outs[1])
            ref = (A.float() if prec == 3 else A.hi.float()) @ w.t() + b
            got = outs[1].float().view(N, -1, grp + pad)[:, :, :grp].reshape(N, M) if grp else outs[1].float()
            assert (got.t() - ref).abs().max() < 2e-2
            if grp:
                assert (outs[1].view(N, -1, grp + pad)[:, :, grp:] == 7.0).all()


def _e4m3(t):
    return t.view(torch.float8_e4m3fn).float()


def _slots(p8):
    """(rows, 2K) e4m3 plane -> (slot 0, slot 1), each (rows, K): the slots are interleaved in 32-column groups (csrc/common.cuh)."""
    v = p8.view(p8.shape[0], -1, 2, 32)
    return _e4m3(v[:, :, 0, :].reshape(p8.shape[0], -1)), _e4m3(v[:, :, 1, :].reshape(p8.shape[0], -1))


def test_split_f16_e4m3_planes(ops, cuda):
    """hipie_split_f16_e4m3 against torch's own fp16 / float8_e4m3fn conversions (round-to-nearest-even, saturating at 448)."""
    g = torch.Generator(device="cuda").manual_seed(21)
    x = torch.randn(300, 256, device=cuda, generator=g) * torch.logspace(-3, 1.5, 256, device=cuda)
    f8 = lambda t: t.clamp(-448, 448).to(torch.float8_e4m3fn).float()
    h = x.half()
    a = ops.split_f16_e4m3(x)
    assert a.hi.dtype == torch.float16 and a.lo.dtype == torch.uint8 and a.lo.shape == (300, 512)
    assert torch.equal(a.hi, h)
    s0, s1 = _slots(a.lo)
    assert torch.equal(s0, f8(h.float())) and torch.equal(s1, f8((x - h.float()) * 1024.0))
    assert (a.float() - x).abs().max() <= (x.abs() * 2.0 ** -15).max()      # hi + lo / 2^10 restores x to ~2^-16
    w = ops.split_f16_e4m3(x * 0.01, weight=True)
    hw = (x * 0.01).half()
    assert torch.equal(w.hi, hw)
    s0, s1 = _slots(w.lo)
    assert torch.equal(s0, f8((x * 0.01 - hw.float()) * 16384.0)) and torch.equal(s1, f8(hw.float() * 16.0))


@pytest.mark.parametrize("M,N,K", [(256, 256, 128), (4096, 5120, 1280), (2048, 1280, 5120), (1000, 96, 320), (3000, 384, 224), (130, 40, 64)])
def test_gemm_f16_e4m3_split(ops, cuda, M, N, K):
    """prec 6: C = Ah.Wh (fp16 pass) + 2^-14 (A8 . W8^T) (ONE e4m3 pass over 2K, folded in by the scale-input-d of the first fp16 MMA).
    (i) against fp64 on exactly the planes the kernel reads: only fp32 accumulation differs; (ii) against the unrounded fp32 product:
    the split restores A.W to the accuracy class of the three-pass bf16 mode."""
    g = torch.Generator(device="cuda").manual_seed(M + 3 * N + K)
    a = torch.randn(M, K, device=cuda, generator=g) * 1.5
    w = torch.randn(N, K, device=cuda, generator=g) * 0.05
    b = torch.randn(N, device=cuda, generator=g)
    A, W = ops.split_f16_e4m3(a), ops.split_f16_e4m3(w, weight=True)
    c, _, _ = ops.gemm(A, W, bias=b, prec=6)
    planes = A.hi.double() @ W.hi.double().t() + (_e4m3(A.lo).double() @ _e4m3(W.lo).double().t()) * 2.0 ** -14 + b.double()
    tol = 3e-5 * math.sqrt(K) * 1.5 * 0.05 * 4 + 1e-5
    err = (c.double() - planes).abs().max().item()
    assert err < tol, f"vs the planes: {err} (tol {tol})"
    exact = a.double() @ w.double().t() + b.double()
    c3, _, _ = ops.gemm(ops.split(a), ops.split_weight(w), bias=b, prec=3)
    e6, e3 = (c.double() - exact).abs().max().item(), (c3.double() - exact).abs().max().item()
    assert e6 < 4e-5 * math.sqrt(K) * 1.5 * 0.05 * 4 + 1e-5, f"vs exact: {e6} (three-pass bf16: {e3})"


def test_gemm_f16_e4m3_output_planes(ops, cuda):
    """fc1 -> fc2 hand-off: the GELU epilogue emits the fp16 plane and the e4m3 planes of its result (TMA-store path); they must be
    exactly the split of the fp32 result."""
    g = torch.Generator(device="cuda").manual_seed(5)
    M, N, K = 1024, 640, 256
    a, w, b = torch.randn(M, K, device=cuda, generator=g), torch.randn(N, K, device=cuda, generator=g) * 0.1, torch.randn(N, device=cuda, generator=g)
    A, W = ops.split_f16_e4m3(a), ops.split_f16_e4m3(w, weight=True)
    c32, _, _ = ops.gemm(A, W, bias=b, act=ops.ACT_GELU, prec=6)
    _, s, _ = ops.gemm(A, W, bias=b, act=ops.ACT_GELU, want_f32=False, out_e4m3=True, prec=6)
    ref = ops.split_f16_e4m3(c32)
    assert torch.equal(s.hi, ref.hi) and torch.equal(s.lo, ref.lo)
    # and through the bf16x3 mainloop as well (the epilogue does not depend on the operand format)
    _, s3, _ = ops.gemm(ops.split(a), ops.split_weight(w), bias=b, want_f32=False, out_e4m3=True, prec=3)
    c3, _, _ = ops.gemm(ops.split(a), ops.split_weight(w), bias=b, prec=3)
    r3 = ops.split_f16_e4m3(c3)
    assert torch.equal(s3.hi, r3.hi) and torch.equal(s3.lo, r3.lo)


def test_layernorm_e4m3_planes(ops, cuda):
    g = torch.Generator(device="cuda").manual_seed(9)
    for C in (1280, 224):
        x = torch.randn(300, C, device=cuda, generator=g) * 2 + 0.3
        gm, bt = torch.randn(C, device=cuda, generator=g), torch.randn(C, device=cuda, generator=g)
        y32, s, _ = ops.layernorm(x, gm, bt, 1e-6, want_f32=True, out_e4m3=True)
        ref = ops.split_f16_e4m3(y32)
        assert torch.equal(s.hi, ref.hi) and torch.equal(s.lo, ref.lo)


def test_layernorm_fp16_plane(ops, cuda):
    """hipie_layernorm_f16: the same statistics, the normalised rows rounded once to IEEE fp16 (with and without a row map)."""
    g = torch.Generator(device="cuda").manual_seed(8)
    for C in (1280, 256, 200):
        x = torch.randn(300, C, device=cuda, generator=g) * 2 + 0.3
        gm, bt = torch.randn(C, device=cuda, generator=g), torch.randn(C, device=cuda, generator=g)
        y32, s, _ = ops.layernorm(x, gm, bt, 1e-6, want_f32=True, out_fp16=True)
        assert s.hi.dtype == torch.float16 and s.lo is None
        assert torch.equal(s.hi, y32.half())
        assert (y32 - F.layer_norm(x, (C,), gm, bt, 1e-6)).abs().max() < 2e-5
    rmap = torch.randperm(300, device=cuda).int()
    out = ops.BF2(torch.zeros(320, 1280, dtype=torch.float16, device=cuda), None)
    x = torch.randn(300, 1280, device=cuda, generator=g)
    gm, bt = torch.randn(1280, device=cuda, generator=g), torch.randn(1280, device=cuda, generator=g)
    ops.layernorm(x, gm, bt, 1e-6, row_map=rmap, out_split=out, out_fp16=True)
    assert torch.equal(out.hi[rmap.long()], F.layer_norm(x, (1280,), gm, bt, 1e-6).half()) or \
        (out.hi[rmap.long()].float() - F.layer_norm(x, (1280,), gm, bt, 1e-6)).abs().max() < 4e-3
    assert (out.hi[300:] == 0).all()


@pytest.mark.parametrize("win", [False, True])
def test_attention_tcgen05_fp16_single_pass(ops, cuda, win):
    """prec 2: q / k / v^T as single fp16 planes, P as fp16, one MMA pass -- against fp64 attention on the SAME fp16-rounded
    operands (tight) and on the unrounded fp32 operands (the 2^-12 operand-rounding budget of DESIGN.md 3)."""
    g = torch.Generator(device="cuda").manual_seed(41)
    if win:
        B, H, hd, gh, gw = 5, 3, 80, 14, 14
    else:
        B, H, hd, gh, gw = 2, 3, 80, 4, 64
    T, E = gh * gw, H * hd
    qk = torch.randn(B * T, 2 * E, device=cuda, generator=g)
    v = torch.randn(B * T, E, device=cuda, generator=g)
    qk16 = qk.half()
    if win:
        vpad = torch.zeros(E, B, 200, device=cuda)
        vpad[:, :, :T] = v.t().reshape(E, B, T)
        vt16 = vpad.view(E, B * 200).half()
        v16 = vt16.float().view(E, B, 200)[:, :, :T].reshape(E, B * T).t()
    else:
        vt16 = v.t().contiguous().half()
        v16 = vt16.float().t()
    q, k, vt = ops.BF2(qk16[:, :E], None), ops.BF2(qk16[:, E:], None), ops.BF2(vt16, None)
    rel_h = torch.randn(B, H, T, gh, device=cuda, generator=g)
    rel_w = torch.randn(B, H, T, gw, device=cuda, generator=g)
    o, _ = ops.attention_tc(q, k, vt, B, H, T, hd, T * 2 * E, 2 * E, T * 2 * E, 2 * E, hd ** -0.5, rel_h=rel_h, rel_w=rel_w, kh=gh, kw=gw,
                            want_f32=True, want_split=False, f16=True)
    sh = lambda x: x.reshape(B, T, H, hd).permute(0, 2, 1, 3).double()
    ref16 = _attn_ref(sh(qk16[:, :E].float()), sh(qk16[:, E:].float()), sh(v16), hd ** -0.5, rel_h, rel_w, gh, gw).permute(0, 2, 1, 3).reshape(B, T, E)
    ref32 = _attn_ref(sh(qk[:, :E]), sh(qk[:, E:]), sh(v), hd ** -0.5, rel_h, rel_w, gh, gw).permute(0, 2, 1, 3).reshape(B, T, E)
    assert (o.double() - ref16).abs().max().item() < 2e-3        # P is rounded to fp16 (2^-12 relative) before the PV pass
    assert (o.double() - ref32).abs().max().item() < 8e-3        # + fp16 rounding of q / k / v: ~8x tighter than the bf16 pass (3e-2)


def test_attention_tcgen05_output_planes(ops, cuda):
    """hipie_attention_tc_planes: the same attention, output as fp16 + e4m3 planes == the split of the fp32 output (global and window mode)."""
    g = torch.Generator(device="cuda").manual_seed(43)
    for win in (False, True):
        B, H, hd, gh, gw = (5, 2, 80, 14, 14) if win else (2, 2, 80, 4, 64)
        T, E = gh * gw, H * hd
        qk16 = torch.randn(B * T, 2 * E, device=cuda, generator=g).half()
        v = torch.randn(B * T, E, device=cuda, generator=g)
        if win:
            vpad = torch.zeros(E, B, 200, device=cuda)
            vpad[:, :, :T] = v.t().reshape(E, B, T)
            vt16 = vpad.view(E, B * 200).half()
        else:
            vt16 = v.t().contiguous().half()
        q, k, vt = ops.BF2(qk16[:, :E], None), ops.BF2(qk16[:, E:], None), ops.BF2(vt16, None)
        rel_h = torch.randn(B, H, T, gh, device=cuda, generator=g)
        rel_w = torch.randn(B, H, T, gw, device=cuda, generator=g)
        kw = dict(rel_h=rel_h, rel_w=rel_w, kh=gh, kw=gw, f16=True)
        o32, _ = ops.attention_tc(q, k, vt, B, H, T, hd, T * 2 * E, 2 * E, T * 2 * E, 2 * E, hd ** -0.5, want_f32=True, want_split=False, **kw)
        _, s = ops.attention_tc(q, k, vt, B, H, T, hd, T * 2 * E, 2 * E, T * 2 * E, 2 * E, hd ** -0.5, out_e4m3=True, **kw)
        ref = ops.split_f16_e4m3(o32.view(B * T, E))
        assert torch.equal(s.hi.view(B * T, E), ref.hi) and torch.equal(s.lo.view(B * T, 2 * E), ref.lo)


def test_relpos_tc_fp16(ops, cuda):
    g = torch.Generator(device="cuda").manual_seed(12)
    B, H, hd, gh, gw = 1, 2, 80, 64, 64
    T = gh * gw
    qk = torch.randn(B * T, 2 * H * hd, device=cuda, generator=g)
    q16 = qk.half()
    Rh = torch.randn(gh, gh, hd, device=cuda, generator=g) * 0.2
    Rw = torch.randn(gw, gw, hd, device=cuda, generator=g) * 0.2
    st = (T * 2 * H * hd, 2 * H * hd, hd)
    th = ops.relpos_bias_tc_f16(q16[:, :H * hd], st, ops.split_weight_f16(Rh), 0, gh, gw, B, H, hd)
    tw = ops.relpos_bias_tc_f16(q16[:, :H * hd], st, ops.split_weight_f16(Rw), 1, gh, gw, B, H, hd)
    rq = q16[:, :H * hd].float().reshape(B, T, H, hd).permute(0, 2, 1, 3).double().reshape(B, H, gh, gw, hd)
    ref_h = torch.einsum("bnhwc,hkc->bnhwk", rq, Rh.double()).reshape(B, H, T, gh)
    ref_w = torch.einsum("bnhwc,wkc->bnhwk", rq, Rw.double()).reshape(B, H, T, gw)
    assert (th.double() - ref_h).abs().max() < 2e-4 and (tw.double() - ref_w).abs().max() < 2e-4


# ------------------------------------------------------------------------------------------ MSDeformAttn encoder: window kernel
@pytest.mark.parametrize("shapes,offs_scale", [([(32, 32), (16, 16), (8, 8), (4, 4)], 1.5), ([(40, 56), (20, 28), (10, 14), (5, 7)], 1.5),
                                               ([(24, 20), (12, 10), (6, 5), (3, 3)], 12.0), ([(64, 64), (32, 32), (16, 16), (8, 8)], 3.0)])
def test_msda_encoder_window_kernel(ops, cuda, shapes, offs_scale):
    """hipie_msda_encoder_forward (TMA-staged shared-memory windows, Lq == S, encoder reference points) against the flat fused
    kernel -- bit for bit -- and against the oracle core; ragged level sizes, borders, and offsets far larger than the halo (the
    global fallback path) included."""
    from hipie_oracle.msda import ms_deform_attn_core
    from hipie_b200 import ops as O
    g = torch.Generator().manual_seed(7)
    shapes_t = torch.as_tensor(shapes)
    S = int(shapes_t.prod(1).sum())
    N, M, L, P = 2, 8, 4, 4
    value = torch.randn(N, S, M * 32, generator=g)
    offs = torch.randn(N, S, M, L, P, 2, generator=g) * offs_scale
    logits = torch.randn(N, S, M, L * P, generator=g)
    # encoder reference points: the query's own pixel centre, the same normalised point on every level (valid ratios 1)
    refs = []
    for (H_, W_) in shapes:
        ry, rx = torch.meshgrid(torch.linspace(0.5, H_ - 0.5, H_) / H_, torch.linspace(0.5, W_ - 0.5, W_) / W_, indexing="ij")
        refs.append(torch.stack((rx.reshape(-1), ry.reshape(-1)), -1))
    refp = torch.cat(refs, 0)[None, :, None, :].repeat(N, 1, L, 1).contiguous()
    norm = torch.stack([shapes_t[:, 1], shapes_t[:, 0]], -1).float()
    loc = refp[:, :, None, :, None, :] + offs / norm[None, None, None, :, None, :]
    w = torch.softmax(logits, -1).view(N, S, M, L, P)
    ref = ms_deform_attn_core(value.view(N, S, M, 32).double(), shapes_t, loc.double(), w.double()).float()
    lsi = torch.cat((shapes_t.new_zeros((1,)), shapes_t.prod(1).cumsum(0)[:-1]))
    packed = torch.cat([offs.reshape(N, S, -1), logits.reshape(N, S, -1)], -1).to(cuda)
    args = (value.to(cuda), shapes_t.to(cuda), lsi.to(cuda), packed, refp.to(cuda))
    O.MSDA_WINDOWS = False
    flat = ops.msda_fused(*args, want_split=False)
    flat_s = ops.msda_fused(*args, want_split=True)
    O.MSDA_WINDOWS = True
    try:
        win = ops.msda_fused(*args, want_split=False, shapes_host=shapes)
        win_s = ops.msda_fused(*args, want_split=True, shapes_host=shapes)
    finally:
        O.MSDA_WINDOWS = False
    assert (win.cpu() - ref).abs().max() < 2e-5
    assert torch.equal(win, flat)
    assert torch.equal(win_s.hi, flat_s.hi) and torch.equal(win_s.lo, flat_s.lo)
