"""Python wrappers of the C-ABI hot-path operators (include/hipie_b200.h).

torch is used for device memory and streams only: every function takes CUDA tensors, passes raw
pointers to libhipie_b200.so on the current stream and returns freshly allocated outputs.  Nothing in
here computes on the CPU or through ATen; a missing library or a CPU tensor raises.
"""
import ctypes
from typing import Optional

import numpy as np
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
    """The operand planes of a tensor-core contraction: `hi` and an optional second plane `lo`.  The plane dtypes ARE the format
    (DESIGN.md 2-3); this class is the one place that knows which pairs exist and how the second plane is shaped:

        fmt          hi             lo               read by
        "bf16"       bf16           None             gemm prec 1
        "bf16x2"     bf16           bf16             gemm prec 3
        "f16"        fp16           None             gemm prec 2, the A operand of prec 4, attention_tc(f16=True)
        "f16x2"      fp16           fp16             the W operand of gemm prec 4, relpos_bias_tc_f16
        "f16+e4m3"   fp16 (.., K)   uint8 (.., 2K)   gemm prec 6; lo holds two e4m3 slots per element, interleaved in 32-column groups
    """

    __slots__ = ("hi", "lo")

    _PLANES = {"bf16": (torch.bfloat16, None), "bf16x2": (torch.bfloat16, torch.bfloat16), "f16": (torch.float16, None),
               "f16x2": (torch.float16, torch.float16), "f16+e4m3": (torch.float16, torch.uint8)}
    _FMT = {v: k for k, v in _PLANES.items()}

    def __init__(self, hi, lo=None):
        self.hi, self.lo = hi, lo

    @property
    def fmt(self):
        pair = (self.hi.dtype, None if self.lo is None else self.lo.dtype)
        if pair not in self._FMT:
            raise TypeError(f"BF2: no plane format has hi {pair[0]} with lo {pair[1]}")
        return self._FMT[pair]

    @staticmethod
    def _lo_shape(fmt, shape):
        """Shape of the second plane for the logical shape (.., K): two e4m3 slots per element, otherwise the same."""
        return tuple(shape[:-1]) + (2 * shape[-1],) if fmt == "f16+e4m3" else tuple(shape)

    @classmethod
    def empty(cls, shape, device, fmt=None, make=torch.empty):
        """Uninitialised planes of the logical shape (.., K); fmt None: the bf16 planes of the current precision mode."""
        fmt = ("bf16x2" if PREC == 3 else "bf16") if fmt is None else fmt
        dhi, dlo = cls._PLANES[fmt]
        hi = make(tuple(shape), dtype=dhi, device=device)
        return cls(hi, None if dlo is None else make(cls._lo_shape(fmt, shape), dtype=dlo, device=device))

    @classmethod
    def zeros(cls, shape, device, fmt=None):
        return cls.empty(shape, device, fmt, make=torch.zeros)

    @property
    def shape(self):
        return self.hi.shape

    def map(self, fn):
        """fn applied to each present plane (it sees an e4m3 plane at its own (.., 2K) shape)."""
        return BF2(fn(self.hi), None if self.lo is None else fn(self.lo))

    def view(self, *s):
        hi = self.hi.view(*s)
        return BF2(hi, None if self.lo is None else self.lo.view(self._lo_shape(self.fmt, hi.shape)))

    def __getitem__(self, idx):
        if self.fmt == "f16+e4m3":      # rows only: a column cut would split the 32-column slot groups of the e4m3 plane
            t = idx if isinstance(idx, tuple) else (idx,)
            if len(t) >= self.hi.dim() or any(i is None or i is Ellipsis for i in t):
                raise IndexError("BF2: fp16 + e4m3 planes can be cut along leading (row) dimensions only")
        return self.map(lambda t: t[idx])

    def float(self):
        f = self.hi.float()
        if self.fmt == "f16+e4m3":      # planes of an ACTIVATION (split_f16_e4m3): [e4m3(h) | e4m3(2^10 l)]
            K = self.hi.shape[-1]
            slot1 = self.lo.view(*self.lo.shape[:-1], K // 32, 2, 32)[..., 1, :].reshape(self.hi.shape)      # slots interleaved in 32-column groups
            return f + slot1.view(torch.float8_e4m3fn).float() / 1024.0
        return f if self.lo is None else f + self.lo.float()


def _pp(s: Optional[BF2]):
    """(hi, lo) pointer pair of optional planes: an absent value or an absent second plane is a null pointer."""
    return (None, None) if s is None else (_p(s.hi), _p(s.lo))


def split(x: torch.Tensor) -> BF2:
    x = x.contiguous()
    assert x.dtype == torch.float32
    out = BF2.empty(x.shape, x.device)
    _lib.check(_lib.load().hipie_split_bf16(_p(x), *_pp(out), x.numel(), _stream()), "split_bf16")
    return out


def split_weight(w: torch.Tensor) -> BF2:
    """Weights always carry both planes so the precision mode can be switched at run time."""
    w = w.contiguous().float()
    out = BF2.empty(w.shape, w.device, "bf16x2")
    _lib.check(_lib.load().hipie_split_bf16(_p(w), *_pp(out), w.numel(), _stream()), "split_bf16")
    return out


def split_f16_e4m3(x: torch.Tensor, weight=False) -> BF2:
    """Operand planes of a prec-6 GEMM (fp16 hi x hi pass + ONE e4m3 pass for both cross terms, DESIGN.md 3): hi = fp16(x) (rows, K),
    lo = uint8 storage of the e4m3 planes (rows, 2K): activations [e4m3(h) | e4m3(2^10 (x - h))], weights [e4m3(2^14 (w - h)) | e4m3(2^4 h)]."""
    x = x.contiguous().float()
    K = x.shape[-1]
    rows = x.numel() // K
    out = BF2.empty(x.shape, x.device, "f16+e4m3")
    _lib.check(_lib.load().hipie_split_f16_e4m3(_p(x), *_pp(out), rows, K, 1 if weight else 0, _stream()), "split_f16_e4m3")
    return out


def add_split(a, b=None, want_f32=False, want_split=True):
    a = a.contiguous()
    if b is not None:
        b = b.contiguous()
        assert a.shape == b.shape
    s = torch.empty_like(a) if want_f32 else None
    o = BF2.empty(a.shape, a.device) if want_split else None
    _lib.check(_lib.load().hipie_add_split(_p(a), _p(b), _p(s), *_pp(o), a.numel(), _stream()), "add_split")
    return s, o


_BF16, _F16 = ("bf16", "bf16x2"), ("f16", "f16x2", "f16+e4m3")       # every format whose first plane is bf16 / fp16
# gemm precision -> (formats A may have, formats W may have, hipie_gemm_args field A's second plane feeds, field W's feeds): a second
# plane the precision does not name is not read
_GEMM_PLANES = {1: (_BF16, _BF16, None, None),
                3: (("bf16x2",), ("bf16x2",), "a_lo", "w_lo"),
                2: (_F16, _F16, None, None),
                4: (_F16, ("f16x2",), None, "w_lo"),
                6: (("f16+e4m3",), ("f16+e4m3",), "a8", "w8")}
_PRODUCERS = {_BF16: "bf16 planes (split / split_weight / the default output of every kernel)",
              ("bf16x2",): "bf16 hi + lo planes (split / split_weight / kernel outputs under set_precision(3))",
              _F16: "fp16 planes (gemm(out_fp16=True) / layernorm(out_fp16=True) / row_softmax(out_fp16=True) / split_weight_f16)",
              ("f16x2",): "the weight's fp16 lo plane next to its fp16 hi plane (split_weight_f16)",
              ("f16+e4m3",): "fp16 + e4m3 planes (split_f16_e4m3 / layernorm(out_e4m3=True) / gemm(out_e4m3=True))"}


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
    if prec not in _GEMM_PLANES:
        raise RuntimeError(f"gemm: no precision {prec} (1, 2, 3, 4 or 6)")
    a_fmts, w_fmts, a_field, w_field = _GEMM_PLANES[prec]
    for name, x, fmts in (("A", a, a_fmts), ("W", w, w_fmts)):
        if x.fmt not in fmts:
            raise RuntimeError(f"gemm: prec={prec} takes {name} as {_PRODUCERS[fmts]}, got {x.fmt} planes")
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
    if out_e4m3:       # fp16 plane + e4m3 planes: the A operand of a following prec-6 GEMM
        assert not transposed and batch == 1 and out_split is None
        c_split = BF2.empty(ashape, dev, "f16+e4m3")
        out_fp16 = True
    elif out_fp16:     # one IEEE fp16 plane (operand of the single-pass fp16 contractions)
        c_split = out_split if out_split is not None else BF2.empty(ashape, dev, "f16")
        assert c_split.fmt == "f16"
    else:
        c_split = out_split if out_split is not None else (BF2.empty(ashape, dev) if want_split else None)
    second = {a_field: a.lo, w_field: w.lo}      # hipie_gemm_args field -> the second plane it points at (key None: a plane this precision does not read)
    if c_split is not None:
        second["c8" if out_e4m3 else "c_lo"] = c_split.lo
    ptr2 = lambda field: second[field].data_ptr() if second.get(field) is not None else None
    ld2 = lambda field: second[field].stride(-2) if second.get(field) is not None else 0
    c_bits = None
    if bits_threshold is not None:       # x > threshold, bit-packed along the contiguous output dimension
        c_bits = torch.zeros((batch, N, (M + 31) // 32) if transposed else (batch, rows_out, (N + 31) // 32), dtype=torch.int32, device=dev)
    if residual is not None and ldr is None:
        ldr = residual.stride(-2) if not transposed else residual.stride(-2)
    args = _lib.GemmArgs(
        a_hi=a.hi.data_ptr(), a_lo=ptr2("a_lo"), lda=lda, a_bstride=a_bstride,
        w_hi=w.hi.data_ptr(), w_lo=ptr2("w_lo"), ldw=ldw, w_bstride=w_bstride,
        bias=bias.data_ptr() if bias is not None else None,
        colscale=colscale.data_ptr() if colscale is not None else None,
        residual=residual.data_ptr() if residual is not None else None,
        ldr=ldr or 0, r_bstride=r_bstride,
        c_f32=c_f32.data_ptr() if c_f32 is not None else None,
        c_hi=c_split.hi.data_ptr() if c_split is not None else None, c_lo=ptr2("c_lo"),
        ldc=ldc_, c_bstride=cb,
        c_bits=c_bits.data_ptr() if c_bits is not None else None,
        bits_threshold=float(bits_threshold) if bits_threshold is not None else 0.0,
        M=M, N=N, K=K, batch=batch, act=act, prec=prec, alpha=float(alpha), transposed=1 if transposed else 0,
        c_row_map=row_map.data_ptr() if row_map is not None else None, t_row_group=t_row_group, t_row_pad=t_row_pad,
        relu_after_residual=1 if relu_after_residual else 0, c_fp16=1 if out_fp16 else 0,
        a8=ptr2("a8"), lda8=ld2("a8"), w8=ptr2("w8"), ldw8=ld2("w8"), c8=ptr2("c8"), ldc8=ld2("c8"))
    tag = {2: "gemm_tc[f16x1]", 4: "gemm_tc[f16x2]", 6: "gemm_tc[f16+e4m3]"}.get(prec, f"gemm_tc[p{prec}]") + (":mask_embed" if c_bits is not None else "")
    if profiler.enabled and profiler.shapes:
        tag += f" {M}x{N}x{K}" + (f"x{batch}" if batch > 1 else "") + ("T" if transposed else "")
    work = 2.0 * M * N * K * batch
    if c_bits is not None:   # the mask-embed contraction is HBM-bound (SURVEY 8d): report algorithmic bytes instead of flops
        work = float(batch) * ((M * K + N * K) * 2.0 * (2 if prec == 3 else 1) + M * N * 4.0 + M * N / 8.0)
    with _timed(tag, work):
        _lib.check(lib.hipie_gemm(ctypes.byref(args), _stream()), "gemm")
    if padded:
        if c_f32 is not None and out_f32 is None:
            c_f32 = c_f32[:, :rows_out]
        if c_split is not None and out_split is None:
            c_split = c_split[:, :rows_out]
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
        s = BF2.empty(oshape, x.device, "f16+e4m3")
    elif out_fp16:
        s = out_split if out_split is not None else BF2.empty(oshape, x.device, "f16")
        assert s.fmt == "f16"
    else:
        s = out_split if out_split is not None else (BF2.empty(oshape, x.device) if want_split else None)
    ssum = torch.empty_like(x) if (want_sum and add is not None) else None
    planes = 2 if (out_e4m3 or (PREC == 3 and not out_fp16)) else 1
    nbytes = x.numel() * 4.0 * (1 + (add is not None) + (ssum is not None) + (y is not None)) + (x.numel() * 2.0 * planes if s else 0.0)
    with _timed("layernorm", nbytes):
        if out_fp16:
            _lib.check(_lib.load().hipie_layernorm_f16(_p(x), _p(add), _p(gamma), _p(beta), float(eps), _p(ssum), _p(y), *_pp(s),
                                                       rows, C, _p(row_map), _stream()), "layernorm_f16")
        else:
            _lib.check(_lib.load().hipie_layernorm(_p(x), _p(add), _p(gamma), _p(beta), float(eps), _p(ssum), _p(y),
                                                   *_pp(s), rows, C, _p(row_map), _stream()), "layernorm")
    return y, s, ssum


_gn_ws = {}


def groupnorm_nhwc(x, gamma, beta, eps=1e-5, groups=32, relu=False, post_add=None, want_f32=True, want_split=False,
                   out_f32=None, y_bstride=None, add_bstride=None):
    """x: (N, HW, C) fp32 contiguous.  y_bstride / add_bstride: batch strides (elements) of out_f32 / post_add when they are views
    of larger buffers; the bf16 planes are always (N, HW, C), so a strided output takes want_split=False."""
    N, HW, C = x.shape
    if want_split and y_bstride is not None and y_bstride != HW * C:
        raise ValueError("groupnorm_nhwc: want_split writes (N, HW, C) planes and cannot follow y_bstride")
    dev = x.device
    key = (dev, N * groups, torch.cuda.current_stream(dev).cuda_stream)       # one workspace per stream: branches of the forward overlap
    ws = _gn_ws.get(key)
    if ws is None:
        ws = torch.empty(2 * N * groups, dtype=torch.float64, device=dev)
        _gn_ws[key] = ws
    y = out_f32 if out_f32 is not None else (torch.empty_like(x) if want_f32 else None)
    s = BF2.empty(x.shape, dev) if want_split else None
    yb = HW * C if y_bstride is None else y_bstride
    ab = HW * C if add_bstride is None else add_bstride
    _lib.check(_lib.load().hipie_groupnorm_nhwc(_p(x), _p(gamma), _p(beta), float(eps), _p(post_add), _p(y), *_pp(s),
                                                _p(ws), N, HW, C, groups, 1 if relu else 0, HW * C, yb, ab, _stream()),
               "groupnorm_nhwc")
    return y, s


def patchify(img, mean, std, P=16) -> BF2:
    B, _, H, W = img.shape
    img = img.contiguous()
    rows = B * (H // P) * (W // P)
    out = BF2.empty((rows, 3 * P * P), img.device)
    m = (ctypes.c_float * 3)(*[float(v) for v in mean])
    s = (ctypes.c_float * 3)(*[float(v) for v in std])
    _lib.check(_lib.load().hipie_patchify(_p(img), *_pp(out), B, H, W, P,
                                          ctypes.cast(m, ctypes.c_void_p), ctypes.cast(s, ctypes.c_void_p), _stream()),
               "patchify")
    return out


def im2col_nhwc(x, ksz=3, stride=1, pad=1) -> BF2:
    B, H, W, C = x.shape
    x = x.contiguous()
    Ho = (H + 2 * pad - ksz) // stride + 1
    Wo = (W + 2 * pad - ksz) // stride + 1
    out = BF2.empty((B * Ho * Wo, ksz * ksz * C), x.device)
    _lib.check(_lib.load().hipie_im2col_nhwc(_p(x), *_pp(out), B, H, W, C, ksz, stride, pad, _stream()),
               "im2col_nhwc")
    return out, Ho, Wo


def pixel_shuffle2(g, B, H, W, C, want_f32=True, want_split=False):
    g = g.contiguous()
    y = torch.empty((B, 2 * H, 2 * W, C), dtype=torch.float32, device=g.device) if want_f32 else None
    s = BF2.empty((B, 2 * H, 2 * W, C), g.device) if want_split else None
    _lib.check(_lib.load().hipie_pixel_shuffle2(_p(g), _p(y), *_pp(s), B, H, W, C, _stream()),
               "pixel_shuffle2")
    return y, s


def maxpool2_nhwc(x, want_f32=True, want_split=False):
    B, H, W, C = x.shape
    x = x.contiguous()
    y = torch.empty((B, H // 2, W // 2, C), dtype=torch.float32, device=x.device) if want_f32 else None
    s = BF2.empty((B, H // 2, W // 2, C), x.device) if want_split else None
    _lib.check(_lib.load().hipie_maxpool2_nhwc(_p(x), _p(y), *_pp(s), B, H, W, C, _stream()),
               "maxpool2_nhwc")
    return y, s


def maxpool3x3s2_nhwc(x, want_f32=True, want_split=False):
    B, H, W, C = x.shape
    x = x.contiguous()
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    y = torch.empty((B, Ho, Wo, C), dtype=torch.float32, device=x.device) if want_f32 else None
    s = BF2.empty((B, Ho, Wo, C), x.device) if want_split else None
    _lib.check(_lib.load().hipie_maxpool3x3s2_nhwc(_p(x), _p(y), *_pp(s), B, H, W, C, _stream()), "maxpool3x3s2_nhwc")
    return y, s


def row_softmax(x, colbias=None, rows_per_batch=None, clampv=50000.0, sub_rowmax=False, want_split=True, want_f32=False, out_fp16=False):
    n = x.shape[-1]
    rows = x.numel() // n
    x = x.contiguous()
    s = BF2.empty(x.shape, x.device, "f16") if out_fp16 else (BF2.empty(x.shape, x.device) if want_split else None)
    pf = torch.empty_like(x) if want_f32 else None
    nbytes = x.numel() * 4.0 * (1 + (pf is not None)) + (x.numel() * 2.0 * (2 if (s.lo is not None) else 1) if s else 0.0)
    with _timed("row_softmax", nbytes):
        _lib.check(_lib.load().hipie_row_softmax(_p(x), _p(colbias), rows, rows_per_batch or rows, n, float(clampv),
                                                 1 if sub_rowmax else 0, *_pp(s), _p(pf), 1 if out_fp16 else 0, _stream()),
                   "row_softmax")
    return pf, s


def attention(q: BF2, k: BF2, v: BF2, B, H, Tq, Tk, hd, q_strides, k_strides, v_strides, scale, rel_h=None, rel_w=None,
              kh=0, kw=0, key_bias=None, want_f32=False, want_split=True, prec=None, key_mask=None):
    """q/k/v: planes with explicit (batch, token, head) element strides; output (B, Tq, H*hd).
    key_mask: (B, Tq, ceil(Tk/32)) int32 bit words, bit set = key masked out for that query (boolean attn_mask, all heads)."""
    prec = PREC if prec is None else prec
    dev = q.hi.device
    o = torch.empty((B, Tq, H * hd), dtype=torch.float32, device=dev) if want_f32 else None
    s = BF2.empty((B, Tq, H * hd), dev) if want_split else None
    lo = lambda t: t.lo.data_ptr() if (t.lo is not None and prec == 3) else None
    args = _lib.AttnArgs(
        q_hi=q.hi.data_ptr(), q_lo=lo(q), k_hi=k.hi.data_ptr(), k_lo=lo(k), v_hi=v.hi.data_ptr(), v_lo=lo(v),
        q_bs=q_strides[0], q_ts=q_strides[1], q_hs=q_strides[2],
        k_bs=k_strides[0], k_ts=k_strides[1], k_hs=k_strides[2],
        v_bs=v_strides[0], v_ts=v_strides[1], v_hs=v_strides[2],
        rel_h=rel_h.data_ptr() if rel_h is not None else None, rel_w=rel_w.data_ptr() if rel_w is not None else None,
        kh=kh, kw=kw, key_bias=key_bias.data_ptr() if key_bias is not None else None,
        out_f32=o.data_ptr() if o is not None else None, out_hi=_pp(s)[0], out_lo=_pp(s)[1], o_bs=Tq * H * hd, o_ts=H * hd,
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
        assert q.fmt == k.fmt == vt.fmt == "f16"
        prec = 2
    dev = q.hi.device
    o = torch.empty((B, T, H * hd), dtype=torch.float32, device=dev) if want_f32 else None
    if out_e4m3:       # output as fp16 + e4m3 planes (the A operand of a prec-6 proj GEMM)
        s = BF2.empty((B, T, H * hd), dev, "f16+e4m3")
    else:
        s = BF2.empty((B, T, H * hd), dev) if want_split else None
    lo = lambda t: _p(t.lo) if (t.lo is not None and prec == 3) else None
    fn = _lib.load().hipie_attention_tc_planes if out_e4m3 else _lib.load().hipie_attention_tc
    with _timed("attention_tc[f16x1]" if f16 else f"attention_tc[p{prec}]", 4.0 * B * H * T * T * hd):
        _lib.check(fn(
            _p(q.hi), lo(q), q_bs, q_ts, 0, H * hd, _p(k.hi), lo(k), k_bs, k_ts, 0, H * hd, _p(vt.hi), lo(vt), vt.hi.stride(0),
            _p(rel_h), _p(rel_w), kh, kw, _p(o), *_pp(s), T * H * hd, H * hd, B, H, T, hd, float(scale), prec, _stream()), "attention_tc")
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
        _lib.check(_lib.load().hipie_relpos_bias_tc_f16(_p(q_f16), q_strides[0], q_strides[1], q_strides[2], *_pp(table), axis,
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
        s = BF2.empty((N, Lq, M * D), dev)
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
    s = BF2.empty((rows, 512), pos.device) if want_split else None
    _lib.check(_lib.load().hipie_sine_embed(_p(pos), ld, rows, _p(out), *_pp(s), _stream()), "sine_embed")
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
    out = BF2.zeros((G * G, ld), image01.device)
    m3, s3 = (ctypes.c_float * 3)(*mean), (ctypes.c_float * 3)(*std)
    with _timed("clip_patches"):
        _lib.check(_lib.load().hipie_clip_patches(_p(image01), H, W, S, P, ctypes.cast(m3, ctypes.c_void_p), ctypes.cast(s3, ctypes.c_void_p),
                                                  *_pp(out), ld, _stream()), "clip_patches")
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


# ---------------------------------------------------------------------------- SAM mask refinement (hipie_img.py:367-390, segment_anything 1.0)
def sam_attention(q, k, v, B, H, Tq, Tk, hd, q_bs, q_ld, kv_bs, kv_ld, q_index=None, kv_index=None, want_f32=False, want_split=True):
    """hipie_sam_attention: fp32 q / k / v row views (head h at columns [h*hd, (h+1)*hd)); q_index / kv_index (B) int32 map each output
    batch to its q / kv batch.  Returns (out_f32 (B, Tq, H*hd) or None, BF2 planes or None)."""
    dev = q.device
    o = torch.empty((B, Tq, H * hd), dtype=torch.float32, device=dev) if want_f32 else None
    s = BF2.empty((B, Tq, H * hd), dev) if want_split else None
    tag = "sam_attention:" + ("fewq" if Tq <= 32 else "fewk")
    with _timed(tag, 4.0 * B * H * Tq * Tk * hd):
        _lib.check(_lib.load().hipie_sam_attention(_p(q), q_bs, q_ld, _p(q_index), _p(k), _p(v), kv_bs, kv_ld, _p(kv_index), _p(o),
                                                   *_pp(s), Tq * H * hd, H * hd,
                                                   B, H, Tq, Tk, hd, float(hd ** -0.5), _stream()), "sam_attention")
    return o, s


def sam_masks(x, w, bias, hyper):
    """x (N, h, w, 64) f32 LayerNorm2d output of the first ConvT; w (64, 32, 2, 2), bias (32); hyper (N, 32) -> (N, 2h, 2w) mask-0
    logits, or hyper (N, M, 32) with M in {1, 3} -> (N, M, 2h, 2w): the upscaled features are computed once for the M masks."""
    x, w, bias, hyper = x.contiguous(), w.contiguous(), bias.contiguous(), hyper.contiguous()
    N, h, wd, C = x.shape
    single = hyper.dim() == 2
    M = 1 if single else hyper.shape[1]
    assert C == 64 and tuple(w.shape) == (64, 32, 2, 2) and tuple(hyper.shape) == ((N, 32) if single else (N, M, 32)) and M in (1, 3)
    out = torch.empty((N, M, 2 * h, 2 * wd), dtype=torch.float32, device=x.device)
    with _timed("sam_masks" if M == 1 else f"sam_masks[M={M}]", 2.0 * N * h * wd * 4 * 64 * 32):
        _lib.check(_lib.load().hipie_sam_masks(_p(x), _p(w), _p(bias), _p(hyper), _p(out), N, M, h, wd, _stream()), "sam_masks")
    return out[:, 0] if single else out


SAM_MASK_EMBED_WEIGHTS = ("0.weight", "0.bias", "1.weight", "1.bias", "3.weight", "3.bias", "4.weight", "4.bias", "6.weight", "6.bias")


def sam_mask_embed(masks, weights, emb, img_index=None, eps=1e-6):
    """hipie_sam_mask_embed: masks (N, 1, 4g, 4g) or (N, 4g, 4g) f32 mask inputs; weights: the ten prompt_encoder.mask_downscaling tensors
    in SAM_MASK_EMBED_WEIGHTS order; emb (B, g*g, 256) f32 token-major image embeddings; img_index (N) int32 image of each prompt (None:
    prompt n reads image n).  Returns src (N, g*g, 256) = emb[img] + mask_downscaling(masks), the per-prompt decoder image stream."""
    masks = masks.reshape(masks.shape[0], masks.shape[-2], masks.shape[-1]).float().contiguous()
    N, L = masks.shape[0], masks.shape[-1]
    g = L // 4
    assert masks.shape[-2] == L == 4 * g
    emb = emb.reshape(-1, g * g, 256).contiguous()
    ws = [t.float().contiguous() for t in weights]
    ptrs = (ctypes.c_void_p * 10)(*[t.data_ptr() for t in ws])
    for t in ws:
        _p(t)
    if img_index is not None:
        img_index = img_index.to(torch.int32).contiguous()
    src = torch.empty((N, g * g, 256), dtype=torch.float32, device=masks.device)
    with _timed("sam_mask_embed", float(N * g * g * 256 * 8)):
        _lib.check(_lib.load().hipie_sam_mask_embed(_p(masks), N, ctypes.cast(ptrs, ctypes.c_void_p), float(eps), _p(emb), _p(img_index), g,
                                                    _p(src), _stream()), "sam_mask_embed")
    return src


def sam_upscale(low, input_size, original_size, img_size=1024, return_logits=False, threshold=0.0):
    """hipie_sam_upscale: low (.., lh, lw) f32 logits of one image -> SamPredictor.postprocess_masks at original_size (bilinear to
    img_size^2, crop to input_size, bilinear to original_size); fp32 logits (.., H, W), or bool logit > threshold."""
    lead = tuple(low.shape[:-2])
    lh, lw = low.shape[-2:]
    low = low.reshape(-1, lh, lw).contiguous()
    N = low.shape[0]
    (h_in, w_in), (H, W) = (int(v) for v in input_size), (int(v) for v in original_size)
    out = torch.empty((N, H, W), dtype=torch.float32 if return_logits else torch.uint8, device=low.device)
    with _timed("sam_upscale", float(N * H * W * (4 if return_logits else 1))):
        _lib.check(_lib.load().hipie_sam_upscale(_p(low), N, lh, lw, img_size, h_in, w_in, H, W, float(threshold),
                                                 _p(out) if return_logits else None, None if return_logits else _p(out), _stream()),
                   "sam_upscale")
    out = out.view(lead + (H, W))
    return out if return_logits else out.view(torch.bool)


def sam_mask_stats(low, input_size, original_size, img_size=1024, threshold=0.0, offset=1.0):
    """hipie_sam_mask_stats: low (N, lh, lw) f32 logits of one crop -> (N, 8) int32 per mask of the sam_upscale chain at original_size:
    (count > threshold + offset, count > threshold - offset, area = count > threshold, x0, y0, x1, y1 inclusive (zeros when empty),
    row bands merged).  No pixel is stored."""
    low = low.contiguous()
    N, lh, lw = low.shape
    (h_in, w_in), (H, W) = (int(v) for v in input_size), (int(v) for v in original_size)
    stats = torch.empty((N, 8), dtype=torch.int32, device=low.device)
    with _timed("sam_mask_stats", float(N * H * W)):
        _lib.check(_lib.load().hipie_sam_mask_stats(_p(low), N, lh, lw, img_size, h_in, w_in, H, W, float(threshold), float(offset),
                                                    _p(stats), _stream()), "sam_mask_stats")
    return stats


def sam_mask_emit(low, geom, image_size, img_size=1024, threshold=0.0):
    """hipie_sam_mask_emit: low (K, lh, lw) f32 logits, geom (K, 6) int32 (crop x0, y0, crop_h, crop_w, h_in, w_in) on the device ->
    (K, H, W) bool masks at image_size, each the chain of sam_mask_stats inside its crop box and False outside."""
    low, geom = low.contiguous(), geom.contiguous()
    K, lh, lw = low.shape
    assert geom.shape == (K, 6) and geom.dtype == torch.int32 and geom.device == low.device
    H, W = (int(v) for v in image_size)
    out = torch.empty((K, H, W), dtype=torch.uint8, device=low.device)
    with _timed("sam_mask_emit", float(K * H * W)):
        _lib.check(_lib.load().hipie_sam_mask_emit(_p(low), _p(geom), K, lh, lw, img_size, H, W, float(threshold), _p(out), _stream()),
                   "sam_mask_emit")
    return out.view(torch.bool)


def nms_sorted(boxes_xyxy, iou_threshold):
    """hipie_nms_sorted: (N, 4) f32 xyxy boxes sorted by decreasing score -> int64 positions of the kept boxes, ascending (torchvision
    nms decisions).  Reads back the kept count."""
    boxes = boxes_xyxy.to(torch.float32).contiguous()
    N = boxes.shape[0]
    tiles = (N + 63) // 64
    ws = torch.empty((max(1, N * tiles),), dtype=torch.int64, device=boxes.device)
    keep = torch.empty((max(1, N),), dtype=torch.int32, device=boxes.device)
    nkeep = torch.empty((1,), dtype=torch.int32, device=boxes.device)
    with _timed("nms_sorted", float(N * N)):
        _lib.check(_lib.load().hipie_nms_sorted(_p(boxes), N, float(iou_threshold), _p(ws), ws.numel(), _p(keep), _p(nkeep), _stream()),
                   "nms_sorted")
    return keep[:int(nkeep.item())].long()


def sam_postprocess(low, box_image, geoms, img_size=1024):
    """low (N, lh, lw) f32 logits; box_image (N) int32 image index per box (host list or device tensor); geoms: per image
    (h_in, w_in, h_large, w_large, height, width) host tuples.  Returns one (n_i, height_i, width_i) uint8 tensor per image, boxes in
    order (box_image must be sorted)."""
    low = low.contiguous()
    N, lh, lw = low.shape
    dev = low.device
    bi = [int(i) for i in (box_image.tolist() if torch.is_tensor(box_image) else box_image)]
    counts = [bi.count(i) for i in range(len(geoms))]
    assert bi == sorted(bi), "sam_postprocess: boxes must be grouped by image"
    offs, sizes, total = [], [], 0
    for i, g in enumerate(geoms):
        sizes.append(g[4] * g[5])
        for _ in range(counts[i]):
            offs.append(total)
            total += g[4] * g[5]
    out = torch.empty((total,), dtype=torch.uint8, device=dev)
    if N:
        bi_d = torch.tensor(bi, dtype=torch.int32).to(dev, non_blocking=True)
        geom_d = torch.tensor([int(v) for g in geoms for v in g], dtype=torch.int32).to(dev, non_blocking=True)
        off_d = torch.tensor(offs, dtype=torch.int64).to(dev, non_blocking=True)
        with _timed("sam_postprocess", float(total)):
            _lib.check(_lib.load().hipie_sam_postprocess(_p(low), N, lh, lw, img_size, _p(bi_d), _p(geom_d), _p(off_d), max(sizes), _p(out),
                                                         _stream()), "sam_postprocess")
    res, o = [], 0
    for i, g in enumerate(geoms):
        n = counts[i] * sizes[i]
        res.append(out[o:o + n].view(counts[i], g[4], g[5]))
        o += n
    return res


def part_assign(sem, group, inst):
    """sem (C, H, W) f32; group (C) int fine id -> coarse id, Cc = group.max() = "no part" (host sequence or CUDA i32 tensor, values
    in 0..Cc); inst (N, H, W) uint8 / bool.  Returns fine (H, W) i32 = argmax over C (first index on ties), coarse (H, W) i32 =
    group[fine], cnt_fine (N, C) and cnt_coarse (N, Cc + 1) i32 per-instance pixel counts."""
    sem = sem.contiguous()
    C, H, W = sem.shape
    if sem.dtype != torch.float32:
        raise TypeError("part_assign: sem must be float32")
    if torch.is_tensor(group) and group.is_cuda:
        group_d = group.to(torch.int32).contiguous()
        Cc = int(group_d.max())                     # one host read; callers on the hot path pass the table from the host
    else:
        g = [int(v) for v in (group.tolist() if torch.is_tensor(group) else group)]
        Cc = max(g)
        if min(g) < 0:
            raise ValueError("part_assign: negative group id")
        group_d = torch.tensor(g, dtype=torch.int32).to(sem.device, non_blocking=True)
    if group_d.numel() != C:
        raise ValueError(f"part_assign: group has {group_d.numel()} entries for {C} classes")
    inst = inst.contiguous()
    if inst.dtype == torch.bool:
        inst = inst.view(torch.uint8)
    N = inst.shape[0]
    if inst.dtype != torch.uint8 or (N and tuple(inst.shape[1:]) != (H, W)):
        raise ValueError(f"part_assign: inst must be (N, {H}, {W}) uint8, got {tuple(inst.shape)} {inst.dtype}")
    dev = sem.device
    fine = torch.empty((H, W), dtype=torch.int32, device=dev)
    coarse = torch.empty((H, W), dtype=torch.int32, device=dev)
    cnt_fine = torch.empty((N, C), dtype=torch.int32, device=dev)
    cnt_coarse = torch.empty((N, Cc + 1), dtype=torch.int32, device=dev)
    with _timed("part_assign", float(C * H * W * 4 + N * H * W)):
        _lib.check(_lib.load().hipie_part_assign(_p(sem), C, H, W, _p(group_d), Cc, _p(inst) if N else None, N, _p(fine), _p(coarse),
                                                 _p(cnt_fine) if N else None, _p(cnt_coarse) if N else None, _stream()), "part_assign")
    return fine, coarse, cnt_fine, cnt_coarse


def part_masks(labels, inst, pairs):
    """labels (L, H, W) or (H, W) i32 label planes; inst (N, H, W) uint8 / bool; pairs: (P, 3) (plane, label, instance) host sequence
    or tensor ((P, 2) (label, instance) with a single plane).  Returns (P, H, W) uint8 = (labels[plane] == label) & inst[instance]."""
    labels = labels.contiguous()
    if labels.dim() == 2:
        labels = labels.unsqueeze(0)
    L, H, W = labels.shape
    if labels.dtype != torch.int32:
        raise TypeError("part_masks: labels must be int32")
    inst = inst.contiguous()
    if inst.dtype == torch.bool:
        inst = inst.view(torch.uint8)
    N = inst.shape[0]
    pr = [[int(v) for v in p] for p in (pairs.tolist() if torch.is_tensor(pairs) else pairs)]
    pr = [p if len(p) == 3 else [0] + p for p in pr]
    P = len(pr)
    if any(not (0 <= pl < L and 0 <= n < N) for pl, _, n in pr):
        raise ValueError(f"part_masks: plane outside 0..{L - 1} or instance outside 0..{N - 1}")
    if P and (inst.dtype != torch.uint8 or tuple(inst.shape[1:]) != (H, W)):
        raise ValueError(f"part_masks: inst must be (N, {H}, {W}) uint8, got {tuple(inst.shape)} {inst.dtype}")
    out = torch.empty((P, H, W), dtype=torch.uint8, device=labels.device)
    if P:
        pairs_d = torch.tensor(pr, dtype=torch.int32).to(labels.device, non_blocking=True)
        with _timed("part_masks", float(P * H * W * 6)):
            _lib.check(_lib.load().hipie_part_masks(_p(labels), L, H, W, _p(inst), N, _p(pairs_d), P, _p(out), _stream()), "part_masks")
    return out


def label_words(M):
    """32-bit words per pixel of hipie_label_cover's label bit sets for M label planes."""
    return 1 if M <= 32 else 2 if M <= 64 else 4 if M <= 128 else 8


def label_cover(labels):
    """hipie_label_cover: labels (M, H, W) uint8 / bool label planes (M may be 0) -> bits (label_words(M), H, W) i32 per-pixel label
    bit sets, sem_raw (H, W) i32 = the vote map's argmax (0 = background, else 1 + the first covering plane; background where 20 or more
    planes cover the pixel).  M > 255 is refused by the library."""
    labels = labels.contiguous()
    if labels.dtype == torch.bool:
        labels = labels.view(torch.uint8)
    if labels.dim() != 3 or labels.dtype != torch.uint8:
        raise ValueError(f"label_cover: labels must be (M, H, W) uint8, got {tuple(labels.shape)} {labels.dtype}")
    M, H, W = labels.shape
    bits = torch.empty((label_words(M), H, W), dtype=torch.int32, device=labels.device)
    sem_raw = torch.empty((H, W), dtype=torch.int32, device=labels.device)
    with _timed("label_cover", float(M * H * W)):
        _lib.check(_lib.load().hipie_label_cover(_p(labels) if M else None, M, H, W, _p(bits), _p(sem_raw), _stream()), "label_cover")
    return bits, sem_raw


def sam_vote(masks, bits, M, first_part, acc, area, inter, raw, base):
    """hipie_sam_vote on one chunk of at most 64 masks (Kc, H, W) uint8 / bool, masks base .. base + Kc - 1: accumulates into acc (K, M + 1),
    area (K), inter (K) int64 (zeroed by the caller) the exact fixed-point pooled sums (value * 2^32), areas and part-covered pixel counts,
    and sets raw (H, W) i32 (-1 = uncovered so far) to the first covering mask.  bits from label_cover; labels >= first_part are parts."""
    masks = masks.contiguous()
    if masks.dtype == torch.bool:
        masks = masks.view(torch.uint8)
    Kc, H, W = masks.shape
    K = acc.shape[0]
    if masks.dtype != torch.uint8 or tuple(bits.shape) != (label_words(M), H, W) or bits.dtype != torch.int32:
        raise ValueError(f"sam_vote: masks (Kc, H, W) uint8 and bits ({label_words(M)}, H, W) i32 expected, got "
                         f"{tuple(masks.shape)} {masks.dtype} / {tuple(bits.shape)} {bits.dtype}")
    for t, shape in ((acc, (K, M + 1)), (area, (K,)), (inter, (K,))):
        if t.dtype != torch.int64 or tuple(t.shape) != shape or not t.is_contiguous():
            raise ValueError(f"sam_vote: accumulator of shape {shape} int64 expected, got {tuple(t.shape)} {t.dtype}")
    if raw.dtype != torch.int32 or tuple(raw.shape) != (H, W) or not raw.is_contiguous():
        raise ValueError(f"sam_vote: raw must be ({H}, {W}) int32")
    with _timed("sam_vote", float(Kc * H * W + bits.numel() * 4)):
        _lib.check(_lib.load().hipie_sam_vote(_p(masks) if Kc else None, Kc, H, W, _p(bits), M, int(first_part), int(base), K, _p(acc),
                                              _p(area), _p(inter), _p(raw), _stream()), "sam_vote")


def _error_counter(err, device, what):
    if err is None:
        return torch.zeros(1, dtype=torch.int64, device=device), True
    if err.dtype != torch.int64 or err.numel() != 1 or not err.is_contiguous():
        raise ValueError(f"{what}: err must be a one-element int64 tensor")
    return err, False


def _raise_on_errors(err, what, detail):
    n = int(err.item())
    if n:
        raise ValueError(f"{what}: {n} pixels {detail}")


def semseg_confusion(sem, gt, ignore_label, conf=None, err=None):
    """hipie_semseg_confusion: adds one image to conf ((C + 1, C + 1) int64, rows = predictions, columns = GT; zeros when None) from
    sem (C, H, W) f32 and gt (H, W) int32: pred = torch.argmax(sem, 0), gt == ignore_label -> column C.  GT labels outside 0..C-1 that
    are not ignore_label are counted in err (a one-element int64 counter on the device, accumulated); without err the call allocates one,
    waits for the kernel and raises on them.  Returns conf."""
    if sem.dim() != 3 or sem.dtype != torch.float32:
        raise ValueError(f"semseg_confusion: sem must be (C, H, W) float32, got {tuple(sem.shape)} {sem.dtype}")
    C, H, W = sem.shape
    if not 1 <= C <= SEMSEG_MAX_CLASSES:
        raise ValueError(f"semseg_confusion: {C} classes (1 .. {SEMSEG_MAX_CLASSES})")
    if gt.dtype != torch.int32 or tuple(gt.shape) != (H, W):
        raise ValueError(f"semseg_confusion: gt must be ({H}, {W}) int32, got {tuple(gt.shape)} {gt.dtype}")
    if conf is None:
        conf = torch.zeros((C + 1, C + 1), dtype=torch.int64, device=sem.device)
    elif conf.dtype != torch.int64 or tuple(conf.shape) != (C + 1, C + 1) or not conf.is_contiguous():
        raise ValueError(f"semseg_confusion: conf must be ({C + 1}, {C + 1}) int64")
    err, check = _error_counter(err, sem.device, "semseg_confusion")
    sem, gt = sem.contiguous(), gt.contiguous()
    with _timed("semseg_confusion", float(sem.numel() * 4 + gt.numel() * 4)):
        _lib.check(_lib.load().hipie_semseg_confusion(_p(sem), C, H, W, _p(gt), int(ignore_label), _p(conf), _p(err), _stream()),
                   "semseg_confusion")
    if check:
        _raise_on_errors(err, "semseg_confusion", f"carry a GT label outside 0..{C - 1} that is not the ignore label {ignore_label}")
    return conf


PAIRS_MAX_GT, PAIRS_MAX_PRED, PAIRS_MAX_TABLE = 4096, 65535, 1 << 24
SEMSEG_MAX_CLASSES = 4096


def panoptic_pairs(pred, gt_rgb, gt_ids, S, err=None):
    """hipie_panoptic_pairs: pred (H, W) int32 segment ids (0 = VOID, 1..S), gt_rgb (H, W, 3) uint8 RGB-coded GT, gt_ids the ascending
    positive int32 ids listed in the image's segments_info (a device tensor or a sequence) -> table (n_gt + 2, S + 1) int64 of pixel
    counts: row 0 = GT VOID, rows 1..n_gt = gt_ids, row n_gt + 1 = GT ids present but not listed; column 0 = prediction VOID.  Predictions
    outside 0..S are counted in err (as semseg_confusion); without err the call waits and raises on them.  Sizes beyond the PAIRS_MAX_*
    limits (hipie_panoptic_pairs's) raise."""
    if pred.dim() != 2 or pred.dtype != torch.int32:
        raise ValueError(f"panoptic_pairs: pred must be (H, W) int32, got {tuple(pred.shape)} {pred.dtype}")
    H, W = pred.shape
    if gt_rgb.dtype != torch.uint8 or tuple(gt_rgb.shape) != (H, W, 3):
        raise ValueError(f"panoptic_pairs: gt_rgb must be ({H}, {W}, 3) uint8, got {tuple(gt_rgb.shape)} {gt_rgb.dtype}")
    if not torch.is_tensor(gt_ids):
        ids = [int(i) for i in gt_ids]
        if any(i <= 0 for i in ids) or any(a >= b for a, b in zip(ids, ids[1:])):
            raise ValueError("panoptic_pairs: gt_ids must be positive and strictly ascending")
        gt_ids = torch.tensor(ids, dtype=torch.int32).to(pred.device, non_blocking=True)
    if gt_ids.dtype != torch.int32 or gt_ids.dim() != 1:
        raise ValueError("panoptic_pairs: gt_ids must be a 1-D int32 tensor")
    n_gt, S = gt_ids.numel(), int(S)
    err, check = _error_counter(err, pred.device, "panoptic_pairs")
    if not (0 <= S <= PAIRS_MAX_PRED and n_gt <= PAIRS_MAX_GT and (n_gt + 2) * (S + 1) <= PAIRS_MAX_TABLE):
        raise ValueError(f"panoptic_pairs: {n_gt} listed GT segments and {S} predicted segments exceed the limits (n_gt <= "
                         f"{PAIRS_MAX_GT}, S <= {PAIRS_MAX_PRED}, (n_gt + 2) (S + 1) <= {PAIRS_MAX_TABLE})")
    table = torch.zeros((n_gt + 2, S + 1), dtype=torch.int64, device=pred.device)
    pred, gt_rgb, gt_ids = pred.contiguous(), gt_rgb.contiguous(), gt_ids.contiguous()
    with _timed("panoptic_pairs", float(pred.numel() * 7)):
        _lib.check(_lib.load().hipie_panoptic_pairs(_p(pred), _p(gt_rgb), H, W, _p(gt_ids) if n_gt else None, n_gt, S, _p(table), _p(err),
                                                    _stream()), "panoptic_pairs")
    if check:
        _raise_on_errors(err, "panoptic_pairs", f"carry a predicted segment id outside 0..{S}")
    return table


# ---- instance mask overlaps (COCO AP_segm): one bit layout for predictions and GTs, owned here and by hipie_mask_words
MASK_MAX_PRED, MASK_MAX_GT = 1024, 4096


def mask_words(H, W):
    """u32 words per packed mask: the row-major pixels of an H x W mask, 32 per word, zero-padded to whole 256-bit chunks."""
    return (int(H) * int(W) + 255) // 256 * 8


def _check_hw(what, H, W):
    if not (H > 0 and W > 0 and H * W < (1 << 31)):
        raise ValueError(f"{what}: bad image size {H} x {W} (H * W < 2^31)")


def mask_pack(masks):
    """hipie_mask_pack: masks (N, H, W) uint8 / bool -> (bits (N, mask_words(H, W)) int32, area (N,) int32 pixel counts).  N <= 1024;
    N = 0 returns empty tensors without a launch."""
    masks = masks.contiguous()
    if masks.dtype == torch.bool:
        masks = masks.view(torch.uint8)
    if masks.dim() != 3 or masks.dtype != torch.uint8:
        raise ValueError(f"mask_pack: masks must be (N, H, W) uint8, got {tuple(masks.shape)} {masks.dtype}")
    N, H, W = masks.shape
    _check_hw("mask_pack", H, W)
    if N > MASK_MAX_PRED:
        raise ValueError(f"mask_pack: {N} masks (at most {MASK_MAX_PRED})")
    bits = torch.empty((N, mask_words(H, W)), dtype=torch.int32, device=masks.device)
    area = torch.zeros(N, dtype=torch.int32, device=masks.device)
    if N:
        with _timed("mask_pack", float(masks.numel())):
            _lib.check(_lib.load().hipie_mask_pack(_p(masks), N, H, W, _p(bits), _p(area), _stream()), "mask_pack")
    return bits, area


def rle_ends(runs, H, W):
    """Host side of rle_expand: a sequence of COCO run-length lists (column-major counts, background first) -> (ends int32, offsets
    int64 (M + 1)) numpy arrays, the cumulative run ends of every list back to back.  A list with a negative count or not summing to
    H * W raises."""
    _check_hw("rle_ends", H, W)
    if len(runs) > MASK_MAX_GT:
        raise ValueError(f"rle_ends: {len(runs)} GT masks (at most {MASK_MAX_GT})")
    ends, offsets = [], [0]
    for i, r in enumerate(runs):
        r = np.asarray(r, dtype=np.int64).reshape(-1)
        e = np.cumsum(r)
        if (r < 0).any() or not len(e) or e[-1] != H * W:
            raise ValueError(f"rle_ends: run list {i} sums to {int(e[-1]) if len(e) else 0}, the image has {H} x {W} = {H * W} pixels")
        ends.append(e.astype(np.int32))
        offsets.append(offsets[-1] + len(e))
    return (np.concatenate(ends) if ends else np.zeros(0, np.int32)), np.asarray(offsets, dtype=np.int64)


def rle_expand(ends, offsets, H, W, err=None):
    """hipie_rle_expand: device ends (int32) / offsets (int64, M + 1) from rle_ends -> bits (M, mask_words(H, W)) int32.  Lists whose
    last end is not H * W are counted in err (as semseg_confusion); without err the call waits and raises on them.  M <= 4096; M = 0
    returns an empty tensor without a launch."""
    _check_hw("rle_expand", H, W)
    if offsets.dtype != torch.int64 or offsets.dim() != 1 or ends.dtype != torch.int32 or ends.dim() != 1:
        raise ValueError("rle_expand: ends must be 1-D int32 and offsets 1-D int64")
    M = offsets.numel() - 1
    if not 0 <= M <= MASK_MAX_GT:
        raise ValueError(f"rle_expand: {M} GT masks (at most {MASK_MAX_GT})")
    bits = torch.empty((M, mask_words(H, W)), dtype=torch.int32, device=ends.device)
    if M == 0:
        return bits
    err, check = _error_counter(err, ends.device, "rle_expand")
    ends, offsets = ends.contiguous(), offsets.contiguous()
    with _timed("rle_expand", float(bits.numel() * 4)):
        _lib.check(_lib.load().hipie_rle_expand(_p(ends), _p(offsets), M, H, W, _p(bits), _p(err), _stream()), "rle_expand")
    if check and int(err.item()):
        raise ValueError(f"rle_expand: {int(err.item())} run lists do not sum to {H} x {W} = {H * W} pixels")
    return bits


def mask_overlaps(pred_bits, gt_bits, H, W):
    """hipie_mask_overlaps: pred_bits (N, KW) and gt_bits (M, KW) int32 from mask_pack / rle_expand -> inter (N, M) int32 pixel counts of
    every pair's intersection (b1 MMA, K split over CTAs, exact).  N = 0 or M = 0 returns an empty table without a launch."""
    _check_hw("mask_overlaps", H, W)
    KW = mask_words(H, W)
    for name, t, lim in (("pred_bits", pred_bits, MASK_MAX_PRED), ("gt_bits", gt_bits, MASK_MAX_GT)):
        if t.dtype != torch.int32 or t.dim() != 2 or t.shape[1] != KW or not t.is_contiguous():
            raise ValueError(f"mask_overlaps: {name} must be contiguous (rows, {KW}) int32, got {tuple(t.shape)} {t.dtype}")
        if t.shape[0] > lim:
            raise ValueError(f"mask_overlaps: {t.shape[0]} rows of {name} (at most {lim})")
    N, M = pred_bits.shape[0], gt_bits.shape[0]
    inter = torch.zeros((N, M), dtype=torch.int32, device=pred_bits.device)
    if N and M:
        with _timed("mask_overlaps", float((N + M) * KW * 4)):
            _lib.check(_lib.load().hipie_mask_overlaps(_p(pred_bits), N, _p(gt_bits), M, H, W, _p(inter), _stream()), "mask_overlaps")
    return inter
