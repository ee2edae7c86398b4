"""Python wrappers of the C-ABI hot-path operators (include/hipie_b200.h).

torch is used for device memory and streams only: every function takes CUDA tensors, passes raw
pointers to libhipie_b200.so on the current stream and returns freshly allocated outputs.  Nothing in
here computes on the CPU or through ATen; a missing library or a CPU tensor raises.
"""
import ctypes
from typing import Optional

import torch

from . import _lib

# operand precision of the tensor-core paths: 3 = bf16x3 split (fp32-class results, parity mode),
# 1 = plain bf16 (fast mode).
PREC = 3

ACT_NONE, ACT_RELU, ACT_GELU, ACT_SIGMOID, ACT_QUICK_GELU = 0, 1, 2, 3, 4


def set_precision(prec: int):
    global PREC
    assert prec in (1, 3)
    PREC = prec


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


class _Profiler:
    """Optional CUDA-event timing of individual kernel launches on the launching stream (used by bench.py for the
    live roofline numbers).  Disabled by default: no events, no overhead."""

    def __init__(self):
        self.enabled = False
        self.shapes = False    # include GEMM shapes in the tags
        self.records = []      # (tag, work, start_event, end_event)

    def start(self):
        self.records = []
        self.enabled = True

    def stop(self):
        self.enabled = False
        torch.cuda.synchronize()
        out = {}
        for tag, work, s, e in self.records:
            d = out.setdefault(tag, {"ms": 0.0, "launches": 0, "work": 0.0})
            d["ms"] += s.elapsed_time(e)
            d["launches"] += 1
            d["work"] += work
        self.records = []
        return out


profiler = _Profiler()


class _timed:
    def __init__(self, tag, work=0.0):
        self.tag, self.work = tag, work

    def __enter__(self):
        if profiler.enabled:
            self.s = torch.cuda.Event(enable_timing=True)
            self.s.record()
        return self

    def __exit__(self, *a):
        if profiler.enabled:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            profiler.records.append((self.tag, self.work, self.s, e))
        return False


def _p(t: Optional[torch.Tensor]):
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError("hipie_b200 ops take CUDA tensors only (no CPU fallback)")
    return ctypes.c_void_p(t.data_ptr())


class BF2:
    """bf16 hi/lo planes of an fp32 tensor (lo is None in plain-bf16 mode)."""

    __slots__ = ("hi", "lo")

    def __init__(self, hi, lo=None):
        self.hi, self.lo = hi, lo

    @property
    def shape(self):
        return self.hi.shape

    def view(self, *s):
        return BF2(self.hi.view(*s), None if self.lo is None else self.lo.view(*s))

    def __getitem__(self, idx):
        return BF2(self.hi[idx], None if self.lo is None else self.lo[idx])

    def float(self):
        f = self.hi.float()
        if self.lo is not None and self.lo.dtype == torch.uint8:      # fp16 + e4m3 planes of an ACTIVATION (split_f16_e4m3): [e4m3(h) | e4m3(2^10 l)]
            K = self.hi.shape[-1]
            slot1 = self.lo.view(*self.lo.shape[:-1], K // 32, 2, 32)[..., 1, :].reshape(self.hi.shape)      # slots interleaved in 32-column groups
            return f + slot1.view(torch.float8_e4m3fn).float() / 1024.0
        return f if self.lo is None else f + self.lo.float()


def _empty_bf2(shape, device, need_lo=None):
    need_lo = (PREC == 3) if need_lo is None else need_lo
    hi = torch.empty(shape, dtype=torch.bfloat16, device=device)
    lo = torch.empty(shape, dtype=torch.bfloat16, device=device) if need_lo else None
    return BF2(hi, lo)


def split(x: torch.Tensor) -> BF2:
    x = x.contiguous()
    assert x.dtype == torch.float32
    out = _empty_bf2(x.shape, x.device)
    _lib.check(_lib.load().hipie_split_bf16(_p(x), _p(out.hi), _p(out.lo), x.numel(), _stream()), "split_bf16")
    return out


def split_weight(w: torch.Tensor) -> BF2:
    """Weights always carry both planes so the precision mode can be switched at run time."""
    w = w.contiguous().float()
    out = _empty_bf2(w.shape, w.device, need_lo=True)
    _lib.check(_lib.load().hipie_split_bf16(_p(w), _p(out.hi), _p(out.lo), w.numel(), _stream()), "split_bf16")
    return out


def split_f16_e4m3(x: torch.Tensor, weight=False) -> BF2:
    """Operand planes of a prec-6 GEMM (fp16 hi x hi pass + ONE e4m3 pass for both cross terms, DESIGN.md 3): hi = fp16(x) (rows, K),
    lo = uint8 storage of the e4m3 planes (rows, 2K): activations [e4m3(h) | e4m3(2^10 (x - h))], weights [e4m3(2^14 (w - h)) | e4m3(2^4 h)]."""
    x = x.contiguous().float()
    K = x.shape[-1]
    rows = x.numel() // K
    h = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    p8 = torch.empty(x.shape[:-1] + (2 * K,), dtype=torch.uint8, device=x.device)
    _lib.check(_lib.load().hipie_split_f16_e4m3(_p(x), _p(h), _p(p8), rows, K, 1 if weight else 0, _stream()), "split_f16_e4m3")
    return BF2(h, p8)


def add_split(a, b=None, want_f32=False, want_split=True):
    a = a.contiguous()
    if b is not None:
        b = b.contiguous()
        assert a.shape == b.shape
    s = torch.empty_like(a) if want_f32 else None
    o = _empty_bf2(a.shape, a.device) if want_split else None
    _lib.check(_lib.load().hipie_add_split(_p(a), _p(b), _p(s), _p(o.hi) if o else None, _p(o.lo) if o else None,
                                           a.numel(), _stream()), "add_split")
    return s, o


def gemm(a: BF2, w: BF2, bias=None, act=ACT_NONE, colscale=None, residual=None, alpha=1.0, want_f32=True,
         want_split=False, out_f32=None, transposed=False, row_map=None, out_rows=None, bits_threshold=None,
         M=None, N=None, K=None, batch=1, lda=None, ldw=None, a_bstride=0, w_bstride=0, ldc=None, c_bstride=0,
         ldr=None, r_bstride=0, prec=None, out_split=None, t_row_group=0, t_row_pad=0, out_fp16=False, relu_after_residual=False,
         out_e4m3=False):
    """C = act(alpha * A.W^T + bias) * colscale + residual.

    A: (.., M, K) planes, W: (N, K) planes.  Default: 2-D row-major operands.  Strided / batched views
    are described with the explicit M/N/K/ld*/bstride arguments (elements).
    Returns (c_f32 or None, c_split or None, c_bits or None).
    """
    lib = _lib.load()
    prec = PREC if prec is None else prec
    if prec == 3 and (a.lo is None or w.lo is None):
        raise RuntimeError("gemm: prec=3 needs lo planes")
    if prec == 6 and not (a.lo is not None and w.lo is not None and a.lo.dtype == torch.uint8 and w.lo.dtype == torch.uint8):
        raise RuntimeError("gemm: prec=6 takes fp16 + e4m3 planes (split_f16_e4m3 / layernorm(out_e4m3=True) / gemm(out_e4m3=True))")
    if prec in (2, 4, 6) and not (a.hi.dtype == torch.float16 and w.hi.dtype == torch.float16):
        raise RuntimeError("gemm: prec=2 / 4 take fp16 planes (gemm(out_fp16=True) / layernorm(out_fp16=True) / row_softmax(out_fp16=True) / split_weight_f16)")
    if prec == 4 and (w.lo is None or w.lo.dtype != torch.float16):
        raise RuntimeError("gemm: prec=4 (A one fp16 plane, W fp16 hi + lo) needs the weight's fp16 lo plane (split_weight_f16)")
    dev = a.hi.device
    if M is None:
        assert a.hi.dim() == 2 and w.hi.dim() == 2
        M, K = a.hi.shape
        N = w.hi.shape[0]
        assert w.hi.shape[1] == K
        lda = a.hi.stride(0)
        ldw = w.hi.stride(0)
    rows_out = out_rows if out_rows is not None else M
    if transposed:
        shape = (batch, N, rows_out) if batch > 1 else (N, rows_out)
        ldc_ = rows_out if ldc is None else ldc
        cb = N * rows_out if (batch > 1 and c_bstride == 0) else c_bstride
    else:
        shape = (batch, rows_out, N) if batch > 1 else (rows_out, N)
        ldc_ = N if ldc is None else ldc
        cb = rows_out * N if (batch > 1 and c_bstride == 0) else c_bstride
    # transposed output with a padded leading dimension (e.g. a TMA consumer needs 16-byte row strides): allocate (N, ldc)
    # and hand back the logical (N, rows_out) view
    padded = transposed and batch == 1 and ldc is not None and ldc > rows_out
    ashape = (N, ldc) if padded else shape
    c_f32 = out_f32 if out_f32 is not None else (torch.empty(ashape, dtype=torch.float32, device=dev) if want_f32 else None)
    c8 = None
    if out_e4m3:       # fp16 plane + e4m3 planes (rows, 2N): the A operand of a following prec-6 GEMM
        assert not transposed and batch == 1 and out_split is None
        c8 = torch.empty((rows_out, 2 * N), dtype=torch.uint8, device=dev)
        c_split = BF2(torch.empty(ashape, dtype=torch.float16, device=dev), None)
        out_fp16 = True
    elif out_fp16:     # one IEEE fp16 plane (operand of the single-pass fp16 contractions); returned as BF2(hi=fp16 tensor, lo=None)
        c_split = out_split if out_split is not None else BF2(torch.empty(ashape, dtype=torch.float16, device=dev), None)
        assert c_split.lo is None
    else:
        c_split = out_split if out_split is not None else (_empty_bf2(ashape, dev) if want_split else None)
    c_bits = None
    if bits_threshold is not None:       # x > threshold, bit-packed along the contiguous output dimension
        c_bits = torch.zeros((batch, N, (M + 31) // 32) if transposed else (batch, rows_out, (N + 31) // 32), dtype=torch.int32, device=dev)
    if residual is not None and ldr is None:
        ldr = residual.stride(-2) if not transposed else residual.stride(-2)
    args = _lib.GemmArgs(
        a_hi=a.hi.data_ptr(), a_lo=a.lo.data_ptr() if (a.lo is not None and prec == 3) else None, lda=lda, a_bstride=a_bstride,
        w_hi=w.hi.data_ptr(), w_lo=w.lo.data_ptr() if (w.lo is not None and prec in (3, 4)) else None, ldw=ldw, w_bstride=w_bstride,
        bias=bias.data_ptr() if bias is not None else None,
        colscale=colscale.data_ptr() if colscale is not None else None,
        residual=residual.data_ptr() if residual is not None else None,
        ldr=ldr or 0, r_bstride=r_bstride,
        c_f32=c_f32.data_ptr() if c_f32 is not None else None,
        c_hi=c_split.hi.data_ptr() if c_split is not None else None,
        c_lo=c_split.lo.data_ptr() if (c_split is not None and c_split.lo is not None) else None,
        ldc=ldc_, c_bstride=cb,
        c_bits=c_bits.data_ptr() if c_bits is not None else None,
        bits_threshold=float(bits_threshold) if bits_threshold is not None else 0.0,
        M=M, N=N, K=K, batch=batch, act=act, prec=prec, alpha=float(alpha), transposed=1 if transposed else 0,
        c_row_map=row_map.data_ptr() if row_map is not None else None, t_row_group=t_row_group, t_row_pad=t_row_pad,
        relu_after_residual=1 if relu_after_residual else 0, c_fp16=1 if out_fp16 else 0,
        a8=a.lo.data_ptr() if prec == 6 else None, lda8=a.lo.stride(-2) if prec == 6 else 0,
        w8=w.lo.data_ptr() if prec == 6 else None, ldw8=w.lo.stride(-2) if prec == 6 else 0,
        c8=c8.data_ptr() if c8 is not None else None, ldc8=2 * N if c8 is not None else 0)
    tag = {2: "gemm_tc[f16x1]", 4: "gemm_tc[f16x2]", 6: "gemm_tc[f16+e4m3]"}.get(prec, f"gemm_tc[p{prec}]") + (":mask_embed" if c_bits is not None else "")
    if profiler.enabled and profiler.shapes:
        tag += f" {M}x{N}x{K}" + (f"x{batch}" if batch > 1 else "") + ("T" if transposed else "")
    work = 2.0 * M * N * K * batch
    if c_bits is not None:   # the mask-embed contraction is HBM-bound (SURVEY 8d): report algorithmic bytes instead of flops
        work = float(batch) * ((M * K + N * K) * 2.0 * (2 if prec == 3 else 1) + M * N * 4.0 + M * N / 8.0)
    with _timed(tag, work):
        _lib.check(lib.hipie_gemm(ctypes.byref(args), _stream()), "gemm")
    if c8 is not None:
        c_split = BF2(c_split.hi, c8)
    if padded:
        if c_f32 is not None and out_f32 is None:
            c_f32 = c_f32[:, :rows_out]
        if c_split is not None and out_split is None:
            c_split = BF2(c_split.hi[:, :rows_out], None if c_split.lo is None else c_split.lo[:, :rows_out])
    return c_f32, c_split, c_bits


def linear(x: BF2, w: BF2, bias=None, **kw):
    """x: (..., K) planes -> (..., N); convenience over gemm for contiguous inputs."""
    lead = x.hi.shape[:-1]
    x2 = x.view(-1, x.hi.shape[-1])
    f, s, _ = gemm(x2, w, bias=bias, **kw)
    N = w.hi.shape[0]
    if f is not None:
        f = f.view(*lead, N)
    if s is not None:
        s = s.view(*lead, N)
    return f, s


def layernorm(x, gamma, beta, eps, add=None, want_f32=False, want_split=True, want_sum=False, row_map=None,
              out_rows=None, out_split: Optional[BF2] = None, out_fp16=False, out_e4m3=False):
    """out_fp16: the normalised rows leave as ONE IEEE fp16 plane (BF2(hi=fp16, lo=None)), the A operand of a prec-4 GEMM;
    out_e4m3: fp16 plane + e4m3 planes (rows, 2C) (BF2(hi=fp16, lo=uint8)), the A operand of a prec-6 GEMM."""
    out_fp16 = out_fp16 or out_e4m3
    x = x.contiguous()
    C = x.shape[-1]
    rows = x.numel() // C
    if add is not None:
        add = add.contiguous()
    oshape = x.shape if out_rows is None else (out_rows, C)
    y = torch.empty(oshape, dtype=torch.float32, device=x.device) if want_f32 else None
    if out_e4m3:
        assert out_split is None and row_map is None
        s = BF2(torch.empty(oshape, dtype=torch.float16, device=x.device), torch.empty(tuple(oshape[:-1]) + (2 * C,), dtype=torch.uint8, device=x.device))
    elif out_fp16:
        s = out_split if out_split is not None else BF2(torch.empty(oshape, dtype=torch.float16, device=x.device), None)
        assert s.hi.dtype == torch.float16 and s.lo is None
    else:
        s = out_split if out_split is not None else (_empty_bf2(oshape, x.device) if want_split else None)
    ssum = torch.empty_like(x) if (want_sum and add is not None) else None
    planes = 2 if (out_e4m3 or (PREC == 3 and not out_fp16)) else 1
    nbytes = x.numel() * 4.0 * (1 + (add is not None) + (ssum is not None) + (y is not None)) + (x.numel() * 2.0 * planes if s else 0.0)
    with _timed("layernorm", nbytes):
        if out_fp16:
            _lib.check(_lib.load().hipie_layernorm_f16(_p(x), _p(add), _p(gamma), _p(beta), float(eps), _p(ssum), _p(y), _p(s.hi),
                                                       _p(s.lo) if out_e4m3 else None, rows, C, _p(row_map), _stream()), "layernorm_f16")
        else:
            _lib.check(_lib.load().hipie_layernorm(_p(x), _p(add), _p(gamma), _p(beta), float(eps), _p(ssum), _p(y),
                                                   _p(s.hi) if s else None, _p(s.lo) if (s and s.lo is not None) else None,
                                                   rows, C, _p(row_map), _stream()), "layernorm")
    return y, s, ssum


_gn_ws = {}


def groupnorm_nhwc(x, gamma, beta, eps=1e-5, groups=32, relu=False, post_add=None, want_f32=True, want_split=False,
                   out_f32=None, y_bstride=None, add_bstride=None):
    """x: (N, HW, C) fp32 contiguous."""
    N, HW, C = x.shape
    dev = x.device
    key = (dev, N * groups, torch.cuda.current_stream(dev).cuda_stream)       # one workspace per stream: branches of the forward overlap
    ws = _gn_ws.get(key)
    if ws is None:
        ws = torch.empty(2 * N * groups, dtype=torch.float64, device=dev)
        _gn_ws[key] = ws
    y = out_f32 if out_f32 is not None else (torch.empty_like(x) if want_f32 else None)
    s = _empty_bf2(x.shape, dev) if want_split else None
    yb = HW * C if y_bstride is None else y_bstride
    ab = HW * C if add_bstride is None else add_bstride
    _lib.check(_lib.load().hipie_groupnorm_nhwc(_p(x), _p(gamma), _p(beta), float(eps), _p(post_add), _p(y),
                                                _p(s.hi) if s else None, _p(s.lo) if (s and s.lo is not None) else None,
                                                _p(ws), N, HW, C, groups, 1 if relu else 0, HW * C, yb, ab, _stream()),
               "groupnorm_nhwc")
    return y, s


def patchify(img, mean, std, P=16) -> BF2:
    B, _, H, W = img.shape
    img = img.contiguous()
    rows = B * (H // P) * (W // P)
    out = _empty_bf2((rows, 3 * P * P), img.device)
    m = (ctypes.c_float * 3)(*[float(v) for v in mean])
    s = (ctypes.c_float * 3)(*[float(v) for v in std])
    _lib.check(_lib.load().hipie_patchify(_p(img), _p(out.hi), _p(out.lo), B, H, W, P,
                                          ctypes.cast(m, ctypes.c_void_p), ctypes.cast(s, ctypes.c_void_p), _stream()),
               "patchify")
    return out


def im2col_nhwc(x, ksz=3, stride=1, pad=1) -> BF2:
    B, H, W, C = x.shape
    x = x.contiguous()
    Ho = (H + 2 * pad - ksz) // stride + 1
    Wo = (W + 2 * pad - ksz) // stride + 1
    out = _empty_bf2((B * Ho * Wo, ksz * ksz * C), x.device)
    _lib.check(_lib.load().hipie_im2col_nhwc(_p(x), _p(out.hi), _p(out.lo), B, H, W, C, ksz, stride, pad, _stream()),
               "im2col_nhwc")
    return out, Ho, Wo


def pixel_shuffle2(g, B, H, W, C, want_f32=True, want_split=False):
    g = g.contiguous()
    y = torch.empty((B, 2 * H, 2 * W, C), dtype=torch.float32, device=g.device) if want_f32 else None
    s = _empty_bf2((B, 2 * H, 2 * W, C), g.device) if want_split else None
    _lib.check(_lib.load().hipie_pixel_shuffle2(_p(g), _p(y), _p(s.hi) if s else None,
                                                _p(s.lo) if (s and s.lo is not None) else None, B, H, W, C, _stream()),
               "pixel_shuffle2")
    return y, s


def maxpool2_nhwc(x, want_f32=True, want_split=False):
    B, H, W, C = x.shape
    x = x.contiguous()
    y = torch.empty((B, H // 2, W // 2, C), dtype=torch.float32, device=x.device) if want_f32 else None
    s = _empty_bf2((B, H // 2, W // 2, C), x.device) if want_split else None
    _lib.check(_lib.load().hipie_maxpool2_nhwc(_p(x), _p(y), _p(s.hi) if s else None,
                                               _p(s.lo) if (s and s.lo is not None) else None, B, H, W, C, _stream()),
               "maxpool2_nhwc")
    return y, s


def maxpool3x3s2_nhwc(x, want_f32=True, want_split=False):
    B, H, W, C = x.shape
    x = x.contiguous()
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    y = torch.empty((B, Ho, Wo, C), dtype=torch.float32, device=x.device) if want_f32 else None
    s = _empty_bf2((B, Ho, Wo, C), x.device) if want_split else None
    _lib.check(_lib.load().hipie_maxpool3x3s2_nhwc(_p(x), _p(y), _p(s.hi) if s else None, _p(s.lo) if (s and s.lo is not None) else None,
                                                   B, H, W, C, _stream()), "maxpool3x3s2_nhwc")
    return y, s


def row_softmax(x, colbias=None, rows_per_batch=None, clampv=50000.0, sub_rowmax=False, want_split=True, want_f32=False, out_fp16=False):
    n = x.shape[-1]
    rows = x.numel() // n
    x = x.contiguous()
    if out_fp16:
        s = BF2(torch.empty(x.shape, dtype=torch.float16, device=x.device), None)
    else:
        s = _empty_bf2(x.shape, x.device) if want_split else None
    pf = torch.empty_like(x) if want_f32 else None
    nbytes = x.numel() * 4.0 * (1 + (pf is not None)) + (x.numel() * 2.0 * (2 if (s.lo is not None) else 1) if s else 0.0)
    with _timed("row_softmax", nbytes):
        _lib.check(_lib.load().hipie_row_softmax(_p(x), _p(colbias), rows, rows_per_batch or rows, n, float(clampv),
                                                 1 if sub_rowmax else 0, _p(s.hi) if s else None,
                                                 _p(s.lo) if (s and s.lo is not None) else None, _p(pf), 1 if out_fp16 else 0, _stream()),
                   "row_softmax")
    return pf, s


def attention(q: BF2, k: BF2, v: BF2, B, H, Tq, Tk, hd, q_strides, k_strides, v_strides, scale, rel_h=None, rel_w=None,
              kh=0, kw=0, key_bias=None, want_f32=False, want_split=True, prec=None, key_mask=None):
    """q/k/v: planes with explicit (batch, token, head) element strides; output (B, Tq, H*hd).
    key_mask: (B, Tq, ceil(Tk/32)) int32 bit words, bit set = key masked out for that query (boolean attn_mask, all heads)."""
    prec = PREC if prec is None else prec
    dev = q.hi.device
    o = torch.empty((B, Tq, H * hd), dtype=torch.float32, device=dev) if want_f32 else None
    s = _empty_bf2((B, Tq, H * hd), dev) if want_split else None
    lo = lambda t: t.lo.data_ptr() if (t.lo is not None and prec == 3) else None
    args = _lib.AttnArgs(
        q_hi=q.hi.data_ptr(), q_lo=lo(q), k_hi=k.hi.data_ptr(), k_lo=lo(k), v_hi=v.hi.data_ptr(), v_lo=lo(v),
        q_bs=q_strides[0], q_ts=q_strides[1], q_hs=q_strides[2],
        k_bs=k_strides[0], k_ts=k_strides[1], k_hs=k_strides[2],
        v_bs=v_strides[0], v_ts=v_strides[1], v_hs=v_strides[2],
        rel_h=rel_h.data_ptr() if rel_h is not None else None, rel_w=rel_w.data_ptr() if rel_w is not None else None,
        kh=kh, kw=kw, key_bias=key_bias.data_ptr() if key_bias is not None else None,
        out_f32=o.data_ptr() if o is not None else None, out_hi=s.hi.data_ptr() if s else None,
        out_lo=s.lo.data_ptr() if (s and s.lo is not None) else None, o_bs=Tq * H * hd, o_ts=H * hd,
        B=B, H=H, Tq=Tq, Tk=Tk, hd=hd, scale=float(scale), prec=prec, key_mask=key_mask.data_ptr() if key_mask is not None else None)
    with _timed(f"attention[p{prec}]" + (":global" if Tq >= 1024 else ":small"), 4.0 * B * H * Tq * Tk * hd):
        _lib.check(_lib.load().hipie_attention(ctypes.byref(args), _stream()), "attention")
    return o, s


def attention_tc(q: BF2, k: BF2, vt: BF2, B, H, T, hd, q_bs, q_ts, k_bs, k_ts, scale, rel_h=None, rel_w=None, kh=0, kw=0,
                 want_f32=False, want_split=True, prec=None, f16=False, out_e4m3=False):
    """wgmma flash attention.  q, k: plane views whose row (token) holds all heads contiguously (head h at columns
    [80h, 80h+80) of the view); vt: BF2 (H*hd, B*T) = V transposed.  Output (B, T, H*hd)."""
    prec = PREC if prec is None else prec
    if f16:            # q / k / vt are single fp16 planes (gemm(out_fp16=True)); the output stays bf16 hi/lo for the 3-pass proj GEMM
        assert q.hi.dtype == torch.float16 and k.hi.dtype == torch.float16 and vt.hi.dtype == torch.float16
        prec = 2
    dev = q.hi.device
    o = torch.empty((B, T, H * hd), dtype=torch.float32, device=dev) if want_f32 else None
    if out_e4m3:       # output as fp16 + e4m3 planes (the A operand of a prec-6 proj GEMM)
        s = BF2(torch.empty((B, T, H * hd), dtype=torch.float16, device=dev), torch.empty((B, T, 2 * H * hd), dtype=torch.uint8, device=dev))
    else:
        s = _empty_bf2((B, T, H * hd), dev) if want_split else None
    lo = lambda t: _p(t.lo) if (t.lo is not None and prec == 3) else None
    fn = _lib.load().hipie_attention_tc_planes if out_e4m3 else _lib.load().hipie_attention_tc
    with _timed("attention_tc[f16x1]" if f16 else f"attention_tc[p{prec}]", 4.0 * B * H * T * T * hd):
        _lib.check(fn(
            _p(q.hi), lo(q), q_bs, q_ts, 0, H * hd, _p(k.hi), lo(k), k_bs, k_ts, 0, H * hd, _p(vt.hi), lo(vt), vt.hi.stride(0),
            _p(rel_h), _p(rel_w), kh, kw, _p(o), _p(s.hi) if s else None, _p(s.lo) if (s and s.lo is not None) else None,
            T * H * hd, H * hd, B, H, T, hd, float(scale), prec, _stream()), "attention_tc")
    return o, s


def relpos_bias(q: BF2, q_strides, table_t, axis, qh, qw, B, H, hd):
    """table_t: (qsize, hd, ksize) fp32.  Returns (B, H, qh*qw, ksize) fp32."""
    ksize = table_t.shape[-1]
    rel = torch.empty((B, H, qh * qw, ksize), dtype=torch.float32, device=table_t.device)
    with _timed("relpos_bias"):
        _lib.check(_lib.load().hipie_relpos_bias(_p(q.hi), _p(q.lo), q_strides[0], q_strides[1], q_strides[2], _p(table_t),
                                                 axis, qh, qw, ksize, _p(rel), B, H, hd, _stream()), "relpos_bias")
    return rel


def relpos_bias_tc(q: BF2, q_strides, table: BF2, axis, qh, qw, B, H, hd):
    """table: BF2 (qsize, ksize, hd) planes (split_weight of get_rel_pos output).  Returns (B, H, qh*qw, ksize) fp32."""
    ksize = table.hi.shape[1]
    rel = torch.empty((B, H, qh * qw, ksize), dtype=torch.float32, device=q.hi.device)
    with _timed("relpos_bias_tc"):
        _lib.check(_lib.load().hipie_relpos_bias_tc(_p(q.hi), _p(q.lo) if PREC == 3 else None, q_strides[0], q_strides[1], q_strides[2],
                                                    _p(table.hi), _p(table.lo), axis, qh, qw, ksize, _p(rel), B, H, hd, _stream()),
                   "relpos_bias_tc")
    return rel


def split_weight_f16(w: torch.Tensor) -> BF2:
    """fp16 hi / lo planes of a small constant table (rel-pos tables of the fp16 attention path); built once with torch at weight
    preparation time."""
    w = w.contiguous().float()
    hi = w.half()
    lo = (w - hi.float()).half()
    return BF2(hi, lo)


def relpos_bias_tc_f16(q_f16: torch.Tensor, q_strides, table: BF2, axis, qh, qw, B, H, hd):
    """q: one fp16 plane; table: fp16 hi/lo planes (qsize, ksize, hd).  Returns (B, H, qh*qw, ksize) fp32."""
    ksize = table.hi.shape[1]
    rel = torch.empty((B, H, qh * qw, ksize), dtype=torch.float32, device=q_f16.device)
    with _timed("relpos_bias_tc"):
        _lib.check(_lib.load().hipie_relpos_bias_tc_f16(_p(q_f16), q_strides[0], q_strides[1], q_strides[2], _p(table.hi), _p(table.lo), axis,
                                                        qh, qw, ksize, _p(rel), B, H, hd, _stream()), "relpos_bias_tc_f16")
    return rel


def msda_forward(value, spatial_shapes, level_start_index, sampling_locations, attention_weights):
    """Drop-in core op (reference signature minus im2col_step): fp32/fp64 tensors on CUDA."""
    N, S, M, D = value.shape
    _, Lq, _, L, P, _ = sampling_locations.shape
    dt = {torch.float32: 0, torch.float64: 1}[sampling_locations.dtype]
    vdt = 2 if value.dtype == torch.bfloat16 else dt
    out = torch.empty((N, Lq, M * D), dtype=sampling_locations.dtype, device=value.device)
    _lib.check(_lib.load().hipie_msda_forward(_p(value.contiguous()), _p(spatial_shapes.contiguous()),
                                              _p(level_start_index.contiguous()), _p(sampling_locations.contiguous()),
                                              _p(attention_weights.contiguous()), _p(out), N, S, M, D, L, Lq, P, dt, vdt,
                                              _stream()), "msda_forward")
    return out


MSDA_WINDOWS = False     # True: encoder calls gather from TMA-staged shared-memory windows (msda_win_kernel, bit-identical results);
                         # measured slower than the flat kernel so far (tools/msda_micro.py, profiles/r02_msda_micro.txt): off by default


def msda_fused(value, spatial_shapes, level_start_index, offs_logits, reference_points, M=8, D=32, L=4, P=4,
               want_split=True, shapes_host=None):
    """value (N,S,M*D) fp32|bf16|fp16; offs_logits (N,Lq,M*L*P*3) fp32; reference_points (N,Lq,L,2|4) fp32.
    shapes_host: the level (H, W) list on the host -- with it, encoder calls (Lq == S, 2-d reference points, fp32 value map) run the
    shared-memory window kernel."""
    N, S = value.shape[0], value.shape[1]
    Lq = offs_logits.shape[1]
    ref_dim = reference_points.shape[-1]
    vdt = 2 if value.dtype == torch.bfloat16 else (3 if value.dtype == torch.float16 else 0)
    dev = value.device
    if want_split:
        s = _empty_bf2((N, Lq, M * D), dev)
        out, out_lo = s.hi, s.lo
    else:
        s = None
        out, out_lo = torch.empty((N, Lq, M * D), dtype=torch.float32, device=dev), None
    fv = 4      # algorithmic bytes are counted on the fp32 value map of the reference op whatever the storage format
    # algorithmic bytes (SURVEY §8d): value map + offsets/logits (3 floats per sample) + output
    alg = float(N) * (S * M * D * fv + Lq * M * L * P * 3 * 4 + Lq * M * D * 4)
    offs_logits, reference_points = offs_logits.contiguous(), reference_points.contiguous()
    with _timed("msda_fused" + (":enc" if Lq == S else ":dec"), alg):
        done = False
        if MSDA_WINDOWS and shapes_host is not None and Lq == S and ref_dim == 2 and vdt == 0 and L == 4:
            sh = (ctypes.c_int * 8)(*[int(v) for hw in shapes_host for v in hw])
            rc = _lib.load().hipie_msda_encoder_forward(_p(value), sh, _p(offs_logits), _p(reference_points), _p(out), N, S, M, D, L, P,
                                                        1 if want_split else 0, _p(out_lo), 0, _stream())
            if rc == 0:
                done = True
            elif rc != -3:           # HIPIE_EUNSUPPORTED: windows do not fit -> flat kernel
                _lib.check(rc, "msda_encoder_forward")
        if not done:
            _lib.check(_lib.load().hipie_msda_fused_forward(_p(value), _p(spatial_shapes), _p(level_start_index),
                                                            _p(offs_logits), _p(reference_points), ref_dim,
                                                            _p(out), N, S, M, D, L, Lq, P, vdt, 1 if want_split else 0, _p(out_lo),
                                                            _stream()), "msda_fused_forward")
    return s if want_split else out


def condinst_masks(feats_nhwc, params, ref_px, Hf, Wf, stride=8):
    B, Q = params.shape[0], params.shape[1]
    out = torch.empty((B, Q, 2 * Hf, 2 * Wf), dtype=torch.float32, device=params.device)
    with _timed("condinst", float(out.numel()) * 4):
        _lib.check(_lib.load().hipie_condinst_masks(_p(feats_nhwc.contiguous()), _p(params.contiguous()), _p(ref_px.contiguous()),
                                                    _p(out), B, Q, Hf, Wf, stride, _stream()), "condinst_masks")
    return out


def seg_postprocess(masks_low, cls_prob, threshold, Hc, Wc, stride=4):
    """Fused semantic + panoptic tensor work for one image (hipie_seg_postprocess).
    masks_low (Q,h,w) f32 logits, cls_prob (Q,C) f32.  Returns sem (C,Hc,Wc), ids (Hc,Wc) i32 [-1 | 2q+inter], areas (3,Q) i32,
    scores (Q), labels (Q).  Any number of classes: vocabularies wider than one accumulator tile run as class chunks of the same kernel, each writing its own rows of `sem`; the panoptic argmax / areas depend on the
    per-query max over ALL classes only and are taken from the first chunk."""
    Q, h, w = masks_low.shape
    C = cls_prob.shape[1]
    dev = masks_low.device
    Qpad = (Q + 63) // 64 * 64
    masks_low = masks_low.contiguous()
    scores, labels = cls_prob.max(-1)
    sc = torch.zeros((Qpad,), dtype=torch.float32, device=dev)
    sc[:Q] = torch.where(scores > threshold, scores, torch.zeros_like(scores))
    sem = torch.empty((C, Hc, Wc), dtype=torch.float32, device=dev)
    ids = torch.empty((Hc, Wc), dtype=torch.int32, device=dev)
    areas = torch.empty((3, Q), dtype=torch.int32, device=dev)
    chunk = C if C <= 136 else 80
    for c0 in range(0, C, chunk):
        cc = min(chunk, C - c0)
        rows = 80 if cc <= 80 else 136
        pt = torch.zeros((rows, Qpad), dtype=torch.float32, device=dev)
        pt[:cc, :Q] = cls_prob[:, c0:c0 + cc].t()
        hi = pt.to(torch.bfloat16)
        lo = (pt - hi.float()).to(torch.bfloat16)
        first = c0 == 0
        ids_c = ids if first else torch.empty_like(ids)
        areas_c = areas if first else torch.empty_like(areas)
        with _timed("seg_postprocess", float(masks_low.numel() + cc * Hc * Wc + ids.numel()) * 4):
            _lib.check(_lib.load().hipie_seg_postprocess(_p(masks_low), _p(hi), _p(lo), _p(sc), _p(sem[c0:c0 + cc]), _p(ids_c), _p(areas_c),
                                                         Q, Qpad, cc, h, w, stride, Hc, Wc, _stream()), "seg_postprocess")
    return sem, ids, areas, scores, labels


def upsample_threshold(masks_low, threshold, Hc, Wc, stride=4):
    """(N,h,w) f32 logits -> (N,Hc,Wc) bool = sigmoid(bilinear x4) > threshold, cropped (hipie_upsample_threshold)."""
    N, h, w = masks_low.shape
    out = torch.empty((N, Hc, Wc), dtype=torch.bool, device=masks_low.device)
    with _timed("upsample_threshold", float(masks_low.numel()) * 4 + out.numel()):
        _lib.check(_lib.load().hipie_upsample_threshold(_p(masks_low.contiguous()), _p(out), N, h, w, stride, Hc, Wc, float(threshold),
                                                        _stream()), "upsample_threshold")
    return out


def sine_embed(pos, want_f32=False, want_split=True):
    """pos (..., 4) f32 (last dim contiguous, uniform row stride) -> (rows, 512) sine embedding in [y, x, w, h] order."""
    assert pos.shape[-1] == 4 and pos.stride(-1) == 1
    rows = pos.numel() // 4
    ld = pos.stride(-2) if pos.dim() > 1 else 4
    if pos.dim() > 2:
        assert pos.stride(-3) == ld * pos.shape[-2], "sine_embed: rows must be uniformly strided"
    out = torch.empty((rows, 512), dtype=torch.float32, device=pos.device) if want_f32 else None
    s = _empty_bf2((rows, 512), pos.device) if want_split else None
    _lib.check(_lib.load().hipie_sine_embed(_p(pos), ld, rows, _p(out), _p(s.hi) if s else None,
                                            _p(s.lo) if (s and s.lo is not None) else None, _stream()), "sine_embed")
    return out, s


def class_scores(logits, tok, cnt, masked=None, iou=None, max_pool=False, want_prob=True):
    """Token -> class pooling + masking + sqrt(sigmoid(cls) * sigmoid(iou)) + per-row max / argmax (hipie_class_scores).
    logits (R, Lt) f32; tok (C, maxlen) i32; cnt (C) i32; masked (C) i8 | None; iou (R) | None.
    Returns scores (R, C), prob (R, C) | None, row_max (R) | None, row_arg (R) i32 | None."""
    logits = logits.contiguous()
    R, Lt = logits.shape
    C, maxlen = tok.shape
    dev = logits.device
    scores = torch.empty((R, C), dtype=torch.float32, device=dev)
    prob = torch.empty((R, C), dtype=torch.float32, device=dev) if want_prob else None
    rmax = torch.empty((R,), dtype=torch.float32, device=dev) if want_prob else None
    rarg = torch.empty((R,), dtype=torch.int32, device=dev) if want_prob else None
    with _timed("class_scores"):
        _lib.check(_lib.load().hipie_class_scores(_p(logits), _p(tok), _p(cnt), _p(masked), _p(iou.contiguous()) if iou is not None else None,
                                                  _p(scores), _p(prob), _p(rmax), _p(rarg), R, Lt, C, maxlen, 1 if max_pool else 0, _stream()),
                   "class_scores")
    return scores, prob, rmax, rarg


def batched_nms(boxes_cxcywh, scores, cls, iou_threshold):
    """(B, N, 4) cxcywh boxes, (B, N) scores, (B, N) int32 classes -> keep (B, N) int32 (-1 padded, decreasing score), nkeep (B) int32."""
    boxes_cxcywh, scores, cls = boxes_cxcywh.contiguous(), scores.contiguous(), cls.contiguous()
    B, N = scores.shape
    keep = torch.empty((B, N), dtype=torch.int32, device=scores.device)
    nkeep = torch.empty((B,), dtype=torch.int32, device=scores.device)
    with _timed("batched_nms"):
        _lib.check(_lib.load().hipie_batched_nms(_p(boxes_cxcywh), _p(scores), _p(cls), _p(keep), _p(nkeep), B, N, float(iou_threshold), _stream()),
                   "batched_nms")
    return keep, nkeep


def topk(values, k, n_rows=None, n_cols_per_row=0):
    """values (R, n) f32 (row-contiguous) -> (R, k) values descending, (R, k) int32 indices; optional device-side valid row counts."""
    assert values.dim() == 2 and values.stride(1) == 1
    R, n = values.shape
    ov = torch.empty((R, k), dtype=torch.float32, device=values.device)
    oi = torch.empty((R, k), dtype=torch.int32, device=values.device)
    with _timed("topk"):
        _lib.check(_lib.load().hipie_topk(_p(values), values.stride(0), _p(n_rows), n_cols_per_row, R, n, k, _p(ov), _p(oi), _stream()), "topk")
    return ov, oi


# ---------------------------------------------------------------------------- MaskCLIP support (open_vocab/clip.py, hipie_img.py:811-868)
def maskclip_patch_mask(masks, S, P, bits, key_offset=1, up=1, crop=None):
    """Per-query patch masks into `bits` (Q, row_words) int32 (zeroed first): bit key_offset + patch set = patch masked OUT.
    masks (Q, h, w) f32 logits; up = 4 with crop = (Hc, Wc): the x4-upsampled, cropped maps are the source of the resize to S x S."""
    masks = masks.contiguous()
    Q, h, w = masks.shape
    Hc, Wc = (h, w) if up == 1 else (int(crop[0]), int(crop[1]))
    assert bits.dtype == torch.int32 and bits.is_contiguous() and bits.shape[0] >= Q
    with _timed("maskclip_patch_mask"):
        _lib.check(_lib.load().hipie_maskclip_patch_mask(_p(masks), Q, h, w, up, Hc, Wc, S, P, _p(bits), bits.shape[1], key_offset, _stream()),
                   "maskclip_patch_mask")
    return bits


def clip_patches(image01, S, P, mean, std):
    """(3, H, W) f32 image in 0..1 -> BF2 ((S/P)^2, 3*P*P padded to a multiple of 8) normalised patch rows of the S x S resize."""
    image01 = image01.contiguous()
    _, H, W = image01.shape
    G, K = S // P, 3 * P * P
    ld = (K + 7) // 8 * 8
    out = BF2(torch.zeros((G * G, ld), dtype=torch.bfloat16, device=image01.device),
              torch.zeros((G * G, ld), dtype=torch.bfloat16, device=image01.device) if PREC == 3 else None)
    m3, s3 = (ctypes.c_float * 3)(*mean), (ctypes.c_float * 3)(*std)
    with _timed("clip_patches"):
        _lib.check(_lib.load().hipie_clip_patches(_p(image01), H, W, S, P, ctypes.cast(m3, ctypes.c_void_p), ctypes.cast(s3, ctypes.c_void_p),
                                                  _p(out.hi), _p(out.lo) if out.lo is not None else None, ld, _stream()), "clip_patches")
    return out


def clip_fuse(raw, mask_embed, logit_scale, seg, scores, temp, overlap, alpha, beta, agg_add, mode, iou=None, fg_a=1.0, fg_b=1.0):
    """hipie_clip_fuse: CLIP logits (norm, scale, max over synonyms, softmax) fused with the model's class probabilities.
    mode 0 -> fused log-probs (R, C); mode 1 -> (prob, row_max, row_arg); mode 2 -> softmax(fused)."""
    raw, mask_embed, scores = raw.contiguous(), mask_embed.contiguous(), scores.contiguous()
    R, C = scores.shape
    out = torch.empty((R, C), dtype=torch.float32, device=scores.device)
    rmax = torch.empty((R,), dtype=torch.float32, device=scores.device) if mode == 1 else None
    rarg = torch.empty((R,), dtype=torch.int32, device=scores.device) if mode == 1 else None
    with _timed("clip_fuse"):
        _lib.check(_lib.load().hipie_clip_fuse(_p(raw), raw.shape[1], _p(mask_embed), mask_embed.shape[1], float(logit_scale), _p(seg), _p(scores),
                                               float(temp), _p(overlap), float(alpha), float(beta), 1 if agg_add else 0,
                                               _p(iou.contiguous()) if iou is not None else None, float(fg_a), float(fg_b), mode, _p(out), _p(rmax),
                                               _p(rarg), R, C, _stream()), "clip_fuse")
    return (out, rmax, rarg) if mode == 1 else out
