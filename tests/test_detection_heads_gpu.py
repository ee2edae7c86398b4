"""GPU: the kernels that turn decoder states into detections, at the geometry a forward launches them with, each against an fp64
restatement computed from exactly the operands the kernel reads.

| Launcher | Branch / instance | Taken when | Tests |
|---|---|---|---|
| `hipie_msda_fused_forward` (msda.cu) | `msda_fast_kernel<BV, true, REFDIM, SPLIT>`, all 12 | value fp32 / bf16 / fp16 x ref_dim 2 / 4 x fp32 out / bf16 hi-lo | `test_msda_instances_by_kernel_name`, `test_msda_fused_instances` (M = 4, 8, 16), `test_msda_encoder_geometry`, `test_msda_decoder_geometry` |
| same | bounds test `h > -1 && w > -1 && h < H && w < W`, per-corner zero padding, float -> int clamps | borders, corners, offsets +-1e6 / +-inf / NaN, 1 x 1, 1 x 7, 7 x 1 levels | `test_msda_sampling_edges` |
| `hipie_msda_forward` | `msda_fast_kernel<BV, false, 2, false>` (fast path) on non-square levels | fp32, D = 32, L = P = 4, M % 4 == 0 | `test_msda_instances_by_kernel_name`, `test_msda_sampling_edges` |
| `hipie_condinst_masks` (misc.cu) | prefetch of the next 4 pixels, ragged last pass | Hf * Wf > 256 x 4, Hf * Wf % 1024 != 0 | `test_condinst_shapes` |
| same | generic upsampling | Wo % 4 != 0 (odd Wf) | `test_condinst_shapes` |
| same | shared-memory limit (host check) | Hf * Wf * 4 <= 200 KB | `test_condinst_shared_memory_limit` |
| `hipie_class_scores` (select.cu) | 64 / 128 / 256 threads, strided classes, cross-warp arg-max, lowest index among ties | C < 128 / < 256 / >= 256 | `test_class_scores` |
| `hipie_batched_nms` | (score desc, index asc) order, class offsets near 1700, 0/0 IoU, N at the shared-memory limit | N <= NMS_MAX = 1216 | `test_batched_nms`, `test_batched_nms_refuses_past_limit` |
| all of the above | what one c1 forward launches | ViT-H, 1024 x 1024, 80 classes | `test_census_c1_forward` |

The MSDeformAttn instances are identified by kernel name in one torch.profiler session (`test_msda_instances_by_kernel_name`);
the other MSDeformAttn tests reach the same instances through the same launcher arguments (value dtype, ref_dim, want_split:
msda.cu hipie_msda_fused_forward) and check them numerically.  That profiler session and the census's model forward run in a
child process (`_in_child`): after either, torch.profiler can stop delivering device activity in the process, and the test
files that run after this one identify kernels by their traces.  The CondInst and class_scores branches are identified by
restating the launcher's predicate.  Reduced-precision value maps are compared against the operator on the rounded values, and
the bf16 hi / lo output planes must equal ops.split of the same call's fp32 output bit for bit.
"""
import json
import re
import sys
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

_T0 = time.time()
BUDGET_S = 300.0
U = 2.0 ** -24                                   # fp32 unit roundoff

VDT = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}
BV = {"f32": 0, "bf16": 1, "f16": 2}            # msda_fast_kernel's BF16V template argument


@pytest.fixture(scope="module")
def ops(cuda):
    from hipie_b200 import ops as o
    o.set_precision(3)
    return o


def _budget(need):
    if time.time() - _T0 + need > BUDGET_S:
        pytest.skip(f"time budget: {time.time() - _T0:.0f}s used, case needs ~{need:.0f}s")


def _msda_instances(names):
    """{(BF16V, FUSED, REFDIM, SPLIT)} of the msda_fast_kernel instances among the recorded names (demangled or mangled)."""
    got = set()
    for n in names:
        for m in re.finditer(r"msda_fast_kernel<(\d),(true|false),(\d),(true|false)>", n):
            got.add((int(m[1]), m[2] == "true", int(m[3]), m[4] == "true"))
        for m in re.finditer(r"msda_fast_kernelILi(\d)ELb([01])ELi(\d)ELb([01])E", n):
            got.add((int(m[1]), m[2] == "1", int(m[3]), m[4] == "1"))
    return got


# ------------------------------------------------------------------------------------------ MSDeformAttn: fp64 restatement
def _lsi(shapes, dev):
    st = [0]
    for h, w in shapes[:-1]:
        st.append(st[-1] + h * w)
    return torch.tensor(shapes, dtype=torch.long, device=dev), torch.tensor(st, dtype=torch.long, device=dev)


def msda_ref64(value, shapes, loc, w):
    """The reference CUDA operator's per-tap semantics in fp64 (ms_deform_im2col_cuda.cuh: bilinear helper and im2col loop):
    pixel = loc * size - 0.5; a tap counts only if h > -1 && w > -1 && h < H && w < W (false for NaN and +-inf), and then each
    of its four corners reads the value map only inside the level, zero outside.
    value (N, S, M, D); loc (N, Lq, M, L, P, 2) normalised (x, y); w (N, Lq, M, L, P) -> (N, Lq, M * D)."""
    value, loc, w = value.double(), loc.double(), w.double()
    N, S, M, D = value.shape
    Lq, L, P = loc.shape[1], loc.shape[3], loc.shape[4]
    dev = value.device
    out = torch.zeros(N, Lq, M, D, dtype=torch.float64, device=dev)
    n_i = torch.arange(N, device=dev).view(N, 1, 1, 1)
    m_i = torch.arange(M, device=dev).view(1, 1, M, 1)
    start = 0
    for l, (H, W) in enumerate(shapes):
        vl = value[:, start:start + H * W].permute(0, 2, 1, 3)              # (N, M, HW, D)
        x = loc[:, :, :, l, :, 0] * W - 0.5
        y = loc[:, :, :, l, :, 1] * H - 0.5
        inside = (y > -1) & (x > -1) & (y < H) & (x < W)
        x, y = torch.where(inside, x, 0.0), torch.where(inside, y, 0.0)
        x0, y0 = x.floor(), y.floor()
        lx, ly = x - x0, y - y0
        wl = torch.where(inside, w[:, :, :, l], 0.0)
        for dy, dx, bw in ((0, 0, (1 - ly) * (1 - lx)), (0, 1, (1 - ly) * lx), (1, 0, ly * (1 - lx)), (1, 1, ly * lx)):
            yy, xx = y0 + dy, x0 + dx
            ok = (yy >= 0) & (yy <= H - 1) & (xx >= 0) & (xx <= W - 1)
            idx = (yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1)).long()       # (N, Lq, M, P)
            out += ((wl * bw * ok)[..., None] * vl[n_i, m_i, idx]).sum(3)
        start += H * W
    return out.reshape(N, Lq, M * D)


def msda_front64(offs, logits, refp, shapes):
    """The fused front half of MSDeformAttn.forward in fp64 (ms_deform_attn.py:97-109): softmax over L * P, then
    ref + off / (W, H) for 2-d reference points, ref + off / P * wh * 0.5 for 4-d boxes.
    offs (N, Lq, M, L, P, 2); logits (N, Lq, M, L * P); refp (N, Lq, L, 2 | 4) -> loc, w."""
    N, Lq, M, L, P, _ = offs.shape
    offs, refp = offs.double(), refp.double()
    w = torch.softmax(logits.double(), -1).view(N, Lq, M, L, P)
    if refp.shape[-1] == 2:
        norm = torch.tensor([[w_, h_] for h_, w_ in shapes], dtype=torch.float64, device=offs.device)
        loc = refp[:, :, None, :, None, :] + offs / norm[None, None, None, :, None, :]
    else:
        loc = refp[:, :, None, :, None, :2] + offs / P * refp[:, :, None, :, None, 2:] * 0.5
    return loc, w


def _pack(offs, logits):
    N, Lq = offs.shape[:2]
    return torch.cat([offs.reshape(N, Lq, -1), logits.reshape(N, Lq, -1)], -1).float().contiguous()


def _msda_tol(value, shapes, loc=None):
    """A priori bound of the fp32 kernel against fp64.  Every output is a combination of 64 bilinear taps with weights summing to
    1: the products and sums cost <= 72 u max|v|.  Where the pixel coordinate is not exact in fp32, it is off by
    <= 2 u (W |loc| + 1) per axis, and moving a tap by d pixels changes it by <= 2 max|v| d per axis (bilinear is continuous at
    the borders too).  loc None: coordinates are exact."""
    vmax = float(value.float().abs().max())
    if loc is None:
        return 72 * U * vmax
    f = loc[torch.isfinite(loc)].abs()
    lmax = min(float(f.max()) if f.numel() else 0.0, 2.0)
    wmax = max(max(h, w) for h, w in shapes)
    return U * vmax * (72 + 8 * (wmax * lmax + 1))


def _check_split(ops, s, out):
    ref = ops.split(out)
    assert torch.equal(s.hi, ref.hi) and torch.equal(s.lo, ref.lo), "split planes differ from ops.split of the fp32 output"


def test_msda_restatement_matches_oracle(cuda):
    """msda_ref64 against ms_deform_attn_core (grid_sample) on finite locations, and against the scalar restatement of the
    reference CUDA kernel on a tiny case that includes borders and non-finite locations."""
    from hipie_oracle.msda import ms_deform_attn_core, ms_deform_attn_scalar
    g = torch.Generator().manual_seed(11)
    shapes = [(6, 5), (3, 8), (1, 1), (4, 1)]
    S = sum(h * w for h, w in shapes)
    N, Lq, M, D, L, P = 2, 13, 4, 3, 4, 4
    value = torch.randn(N, S, M, D, generator=g, dtype=torch.float64)
    loc = torch.rand(N, Lq, M, L, P, 2, generator=g, dtype=torch.float64) * 1.6 - 0.3
    w = torch.rand(N, Lq, M, L, P, generator=g, dtype=torch.float64)
    ref = ms_deform_attn_core(value, torch.tensor(shapes), loc, w)
    assert (msda_ref64(value, shapes, loc, w) - ref).abs().max() < 1e-12
    special = torch.tensor([0.0, 1.0, -0.5 / 6, -1e6, float("inf"), float("-inf"), float("nan"), 1e6], dtype=torch.float64)
    every7 = loc.view(-1)[::7]
    every7.copy_(special[torch.arange(every7.numel()) % len(special)])
    sc = ms_deform_attn_scalar(value, torch.tensor(shapes), _lsi(shapes, "cpu")[1], loc, w)
    assert (msda_ref64(value, shapes, loc, w) - sc).abs().max() < 1e-12


# ------------------------------------------------------------------------------------------ MSDeformAttn: every fused instance
POW2_LEVELS = [(16, 32), (8, 16), (4, 8), (2, 4)]
FUSED_CASES = [(v, rd, M) for v in ("f32", "bf16", "f16") for rd in (2, 4) for M in (4, 8, 16)]


def _run_fused(ops, value, shapes, packed, refp, M):
    """ops.msda_fused with the fp32 output (instance <BV, true, ref_dim, false>) and with the split output (<BV, true, ref_dim,
    true>) -> (fp32 output, BF2 planes)."""
    sh, lsi = _lsi(shapes, value.device)
    N, S = value.shape[:2]
    return tuple(ops.msda_fused(value.reshape(N, S, -1), sh, lsi, packed, refp, M=M, want_split=sp) for sp in (False, True))


def _msda_instance_counts():
    """Launch every launcher argument combination once inside one profiler session -> [(launched instance counts, expected)]:
    the 12 instances of hipie_msda_fused_forward (value fp32 / bf16 / fp16 x ref_dim 2 / 4 x fp32 / split output) and the 2 of
    hipie_msda_forward's fast path (value fp32 / bf16).  A trace without any device activity is taken once more."""
    from torch.profiler import ProfilerActivity, profile
    from hipie_b200 import ops
    cuda = torch.device("cuda:0")
    g = torch.Generator(device="cuda").manual_seed(1)
    shapes, N, Lq, M, L, P = POW2_LEVELS, 1, 8, 8, 4, 4
    S = sum(h * w for h, w in shapes)
    sh, lsi = _lsi(shapes, cuda)
    value = torch.randn(N, S, M * 32, device=cuda, generator=g)
    packed = torch.randn(N, Lq, M * L * P * 3, device=cuda, generator=g)
    refp = {rd: torch.rand(N, Lq, L, rd, device=cuda, generator=g) for rd in (2, 4)}
    loc = torch.rand(N, Lq, M, L, P, 2, device=cuda, generator=g)
    w = torch.rand(N, Lq, M, L, P, device=cuda, generator=g)
    calls, want = [], {}
    for v in ("f32", "bf16", "f16"):
        for rd in (2, 4):
            for sp in (False, True):
                calls.append(lambda v=v, rd=rd, sp=sp: ops.msda_fused(value.to(VDT[v]), sh, lsi, packed, refp[rd], M=M, want_split=sp))
                want[(BV[v], True, rd, sp)] = 1
    for v in ("f32", "bf16"):
        calls.append(lambda v=v: ops.msda_forward(value.to(VDT[v]).view(N, S, M, 32), sh, lsi, loc, w))
        want[(BV[v], False, 2, False)] = 1
    for _ in range(2):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for c in calls:
                c()
            torch.cuda.synchronize()
        got = {}
        for e in prof.key_averages():
            for inst in _msda_instances([e.key.replace(" ", "")]):
                got[inst] = got.get(inst, 0) + e.count
        if got:
            break
    return sorted(got.items()), sorted(want.items())


def _in_child(mode):
    """Run one of this file's __main__ modes in a fresh Python process on the same device -> its JSON result.  torch.profiler
    sessions and whole-model forwards stay out of the test process: after either, torch.profiler can stop delivering device
    activity in that process, and the test files that run after this one identify kernels by their traces."""
    import os
    import subprocess
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    env = dict(os.environ, PYTHONDONTWRITEBYTECODE="1", PYTHONPATH=os.pathsep.join([root, os.path.join(root, "oracle"), here]))
    torch.cuda.empty_cache()                                 # the child needs the memory this process has cached
    r = subprocess.run([sys.executable, "-s", os.path.abspath(__file__), mode], cwd=root, env=env, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_msda_instances_by_kernel_name(cuda):
    """Every launcher argument combination reaches its own msda_fast_kernel instance, each launched once and recorded once."""
    got, want = _in_child("--instances")
    assert got == want, (got, want)


@pytest.mark.parametrize("vdt,ref_dim,M", FUSED_CASES)
def test_msda_fused_instances(ops, cuda, vdt, ref_dim, M):
    """Each of the 12 instances of hipie_msda_fused_forward, at M = 4, 8, 16 head groups of four (a wrong head-group index that
    happens to be right for M = 8 fails at 4 or 16)."""
    g = torch.Generator(device="cuda").manual_seed(100 * M + ref_dim + BV[vdt])
    shapes = POW2_LEVELS
    S = sum(h * w for h, w in shapes)
    N, Lq, L, P = 2, 97, 4, 4
    value = torch.randn(N, S, M, 32, device=cuda, generator=g).to(VDT[vdt])
    offs = torch.randn(N, Lq, M, L, P, 2, device=cuda, generator=g) * 3
    logits = torch.randn(N, Lq, M, L * P, device=cuda, generator=g) * 2
    if ref_dim == 2:
        refp = torch.rand(N, Lq, L, 2, device=cuda, generator=g)
    else:
        refp = torch.cat([torch.rand(N, Lq, L, 2, device=cuda, generator=g) * 1.2 - 0.1,
                          torch.rand(N, Lq, L, 2, device=cuda, generator=g) * 0.8], -1)
    out, s = _run_fused(ops, value, shapes, _pack(offs, logits), refp, M)
    loc, w = msda_front64(offs, logits, refp, shapes)
    ref = msda_ref64(value, shapes, loc, w)                                # the op on exactly the (rounded) values read
    err = (out.double() - ref).abs().max().item()
    assert err <= _msda_tol(value, shapes, loc), (err, _msda_tol(value, shapes, loc))
    _check_split(ops, s, out)


# ------------------------------------------------------------------------------------------ MSDeformAttn: sampling edges
DEGENERATE_LEVELS = [(1, 1), (1, 7), (7, 1), (3, 5)]
NONFINITE = (1e6, -1e6, float("inf"), float("-inf"), float("nan"))


def _edge_coords(n):
    """Pixel coordinates at and next to the border of an axis of n pixels (exact in fp32 for power-of-two n)."""
    return [-1.0, -1.0 + 2 ** -10, -0.5, 0.0, n - 1.0, n - 0.5, n - 2 ** -10, float(n)]


def _edge_pixels(shapes, N, Lq, M, P, g):
    """(N, Lq, M, L, P, 2) pixel coordinates: every pair of edge coordinates (each axis, and so every corner) many times over,
    in a shuffled order, and ~10 % of the coordinates replaced by +-1e6, +-inf or NaN.  Returns (pixels, non-finite mask)."""
    L = len(shapes)
    px = torch.empty(N, Lq, M, L, P, 2, dtype=torch.float64)
    for l, (H, W) in enumerate(shapes):
        pairs = torch.tensor([(x, y) for x in _edge_coords(W) for y in _edge_coords(H)], dtype=torch.float64)
        n = N * Lq * M * P
        sel = torch.randperm(n, generator=g) % len(pairs)
        px[:, :, :, l] = pairs[sel].view(N, Lq, M, P, 2)
    bad = torch.rand(px.shape, generator=g) < 0.1
    pick = torch.randint(0, len(NONFINITE), px.shape, generator=g)
    px = torch.where(bad, torch.tensor(NONFINITE, dtype=torch.float64)[pick], px)
    return px, bad


@pytest.mark.parametrize("levels", ["pow2", "degenerate"])
@pytest.mark.parametrize("path,vdt", [("forward", "f32"), ("forward", "bf16"), ("fused", "f32"), ("fused", "bf16"), ("fused", "f16")])
def test_msda_sampling_edges(ops, cuda, path, vdt, levels):
    """Taps exactly on level borders and corners, just inside and just outside, far away and non-finite, on non-square and
    1 x 1 / 1 x 7 / 7 x 1 levels.  With power-of-two widths the fp32 pixel coordinate is exact, so only the accumulation can
    differ from fp64.  Non-finite taps must contribute exactly zero: the output is finite and matches the restatement."""
    shapes = POW2_LEVELS[:3] + [(1, 1)] if levels == "pow2" else DEGENERATE_LEVELS
    shapes = [(h, w) if i % 2 else (w, h) for i, (h, w) in enumerate(shapes)]       # tall and wide levels
    g = torch.Generator().manual_seed(7 + BV[vdt] + (path == "fused"))
    S = sum(h * w for h, w in shapes)
    N, Lq, M, L, P = 2, 64, 8, 4, 4
    px, bad = _edge_pixels(shapes, N, Lq, M, P, g)
    size = torch.tensor([[w, h] for h, w in shapes], dtype=torch.float64).view(1, 1, 1, L, 1, 2)
    value = torch.randn(N, S, M, 32, generator=g).to(VDT[vdt]).to(cuda)
    sh, lsi = _lsi(shapes, cuda)
    if path == "forward":
        loc = (px + 0.5) / size
        w = torch.softmax(torch.randn(N, Lq, M, L * P, generator=g), -1).view(N, Lq, M, L, P)
        out = ops.msda_forward(value, sh, lsi, loc.float().to(cuda), w.to(cuda))      # fast path: <BV, false, 2, false>
        loc64, w64 = loc.float().double(), w.double()
    else:
        # reference points at the origin: loc = off / W, pixel = off - 0.5 (exact for power-of-two W)
        offs = px + 0.5
        logits = torch.randn(N, Lq, M, L * P, generator=g) * 2
        refp = torch.zeros(N, Lq, L, 2)
        out, s = _run_fused(ops, value, shapes, _pack(offs, logits).to(cuda), refp.to(cuda), M)
        _check_split(ops, s, out)
        loc64, w64 = msda_front64(offs.float(), logits, refp, shapes)
    assert bool(torch.isfinite(out).all())
    ref = msda_ref64(value, shapes, loc64.to(cuda), w64.to(cuda))
    tol = _msda_tol(value, shapes, None if levels == "pow2" else loc64)
    err = (out.double() - ref).abs().max().item()
    assert err <= tol, (err, tol)
    # the non-finite taps contribute exactly zero: the same call with their weights zeroed (forward path) agrees bit for bit
    if path == "forward":
        w0 = torch.where(bad.any(-1), 0.0, w)
        loc0 = torch.where(bad, 0.5, loc)
        out0 = ops.msda_forward(value, sh, lsi, loc0.float().to(cuda), w0.to(cuda))
        assert torch.equal(out, out0)


# ------------------------------------------------------------------------------------------ MSDeformAttn: production geometry
C1_LEVELS = [(128, 128), (64, 64), (32, 32), (16, 16)]                    # c1 encoder, 1024 x 1024 input: S = 21760
ENC_CASES = [(v, r) for v in ("f32", "f16", "bf16") for r in ("full", "ragged")]
DEC_CASES = [(v, Lq) for v in ("f32", "bf16", "f16") for Lq in (910, 300)]


def _encoder_ref_points(shapes, ratios, dev):
    """Deformable-DETR encoder reference points (get_reference_points): pixel centres of every level over the valid region,
    times the valid ratios of every level.  ratios (N, L, 2) as (x, y)."""
    refs = []
    for l, (H, W) in enumerate(shapes):
        ry, rx = torch.meshgrid(torch.linspace(0.5, H - 0.5, H, device=dev), torch.linspace(0.5, W - 0.5, W, device=dev), indexing="ij")
        ry = ry.reshape(1, -1) / (ratios[:, None, l, 1] * H)
        rx = rx.reshape(1, -1) / (ratios[:, None, l, 0] * W)
        refs.append(torch.stack((rx, ry), -1))
    ref = torch.cat(refs, 1)
    return (ref[:, :, None] * ratios[:, None]).contiguous()


@pytest.mark.parametrize("vdt,ratios", ENC_CASES)
def test_msda_encoder_geometry(ops, cuda, vdt, ratios):
    """The c1 encoder call: Lq = S = 21760 over 128^2 ... 16^2 levels, 2-d reference points, N = 2.  'ragged': image 1 is
    valid on 96 x 80 of 128 x 128 (ratios 0.75, 0.625 on every level) and its padded value rows are zero, as msda_layer makes
    them."""
    _budget(10)
    g = torch.Generator(device="cuda").manual_seed(21760 + BV[vdt])
    shapes, N, M, L, P = C1_LEVELS, 2, 8, 4, 4
    S = sum(h * w for h, w in shapes)
    rat = torch.ones(N, L, 2, device=cuda)
    value = torch.randn(N, S, M, 32, device=cuda, generator=g)
    if ratios == "ragged":
        rat[1, :, 0], rat[1, :, 1] = 0.75, 0.625
        pad, st = [], 0
        for H, W in shapes:
            yy, xx = torch.meshgrid(torch.arange(H, device=cuda), torch.arange(W, device=cuda), indexing="ij")
            pad.append(((xx >= W * 0.75) | (yy >= H * 0.625)).reshape(-1))
        value[1][torch.cat(pad)] = 0.0
    value = value.to(VDT[vdt])
    refp = _encoder_ref_points(shapes, rat, cuda)
    offs = torch.randn(N, S, M, L, P, 2, device=cuda, generator=g) * 2
    offs = torch.where(torch.rand(offs.shape, device=cuda, generator=g) < 0.01, offs * 20, offs)
    logits = torch.randn(N, S, M, L * P, device=cuda, generator=g) * 2
    out, s = _run_fused(ops, value, shapes, _pack(offs, logits), refp, M)
    loc, w = msda_front64(offs, logits, refp, shapes)
    ref = msda_ref64(value, shapes, loc, w)
    err, tol = (out.double() - ref).abs().max().item(), _msda_tol(value, shapes, loc)
    assert err <= tol, (err, tol)
    _check_split(ops, s, out)


@pytest.mark.parametrize("vdt,Lq", DEC_CASES)
def test_msda_decoder_geometry(ops, cuda, vdt, Lq):
    """The decoder cross-attention: Lq = 910 (DINO: 900 queries + 10 background) or 300 (MaskDINO) 4-d boxes over the c1
    memory, including boxes with w, h in {0, 2^-20} and boxes reaching past [0, 1]."""
    _budget(5)
    g = torch.Generator(device="cuda").manual_seed(Lq + BV[vdt])
    shapes, N, M, L, P = C1_LEVELS, 2, 8, 4, 4
    S = sum(h * w for h, w in shapes)
    value = torch.randn(N, S, M, 32, device=cuda, generator=g).to(VDT[vdt])
    box = torch.cat([torch.rand(N, Lq, 2, device=cuda, generator=g) * 1.4 - 0.2,
                     torch.rand(N, Lq, 2, device=cuda, generator=g) * 1.5], -1)
    box[:, 0::7, 2:] = 0.0
    box[:, 1::7, 2] = 2.0 ** -20
    box[:, 2::7, 3] = 0.0
    box[:, 3::7, 2:] = 2.0 ** -20
    refp = box[:, :, None].expand(N, Lq, L, 4).contiguous()
    offs = torch.randn(N, Lq, M, L, P, 2, device=cuda, generator=g) * 2
    logits = torch.randn(N, Lq, M, L * P, device=cuda, generator=g) * 2
    out, s = _run_fused(ops, value, shapes, _pack(offs, logits), refp, M)
    loc, w = msda_front64(offs, logits, refp, shapes)
    ref = msda_ref64(value, shapes, loc, w)
    err, tol = (out.double() - ref).abs().max().item(), _msda_tol(value, shapes, loc)
    assert err <= tol, (err, tol)
    _check_split(ops, s, out)


# ------------------------------------------------------------------------------------------ CondInst
CI_THREADS, CI_PX = 256, 4              # condinst_kernel: 256 threads x 4 pixels per pass


def _condinst_branch(Hf, Wf):
    """misc.cu condinst_kernel: passes of 1024 coarse pixels (the next pass's features prefetched when there is one), and the
    16-byte upsampling loop when Wo = 2 Wf is a multiple of 4, the generic one otherwise."""
    return -(-Hf * Wf // (CI_THREADS * CI_PX)), (2 * Wf) % 4


def condinst_ref64(feats, params, ref_px, stride=8):
    """(fp64 reference, a priori bound) on the CPU.  The reference is the oracle's dynamic_mask_with_coords in fp64; the bound is
    the same MLP on |weights| and |inputs| (sum of |terms| of every layer: ReLU of non-negative values is the identity), taken
    through the same aligned_bilinear, which is a convex combination.  The fp32 kernel may differ by <= 64 u of it."""
    from hipie_oracle.condinst import (aligned_bilinear, compute_locations, dynamic_mask_with_coords, mask_heads_forward,
                                       parse_dynamic_params)
    feats, params, ref_px = feats.double().cpu(), params.double().cpu(), ref_px.double().cpu()
    B, C, H, W = feats.shape
    Q = ref_px.shape[1]
    ref = dynamic_mask_with_coords(feats, ref_px, params, stride=stride)
    locs = compute_locations(H, W, stride=stride).double()
    bounds = []
    for b in range(B):
        rel = (ref_px[b].reshape(Q, 1, 2) - locs.reshape(1, H * W, 2)).float().double().abs().permute(0, 2, 1)     # (Q, 2, HW)
        x = torch.cat([rel, feats[b].abs().reshape(1, C, H * W).expand(Q, C, H * W)], 1).reshape(1, Q * (C + 2), H, W)
        ws, bs = parse_dynamic_params(params[b].abs())
        a = mask_heads_forward(x, ws, bs, Q).reshape(Q, 1, H, W)
        bounds.append(aligned_bilinear(a, 2)[:, 0])
    return ref, torch.stack(bounds) * 64 * U


CONDINST_CASES = [(128, 128, 128), (160, 160, 48), (64, 64, 910), (100, 76, 40), (37, 45, 40), (32, 32, 16), (25, 41, 16),
                  (1, 1, 8), (1, 64, 8), (1, 37, 8)]


@pytest.mark.parametrize("Hf,Wf,Q", CONDINST_CASES)
def test_condinst_shapes(ops, cuda, Hf, Wf, Q):
    """128^2 (c1), 160^2 (1280-pixel inputs), 64^2 (R50 512): several passes with the prefetch; 100 x 76: a ragged last pass;
    37 x 45 and 25 x 41 (one pixel past one pass): the generic upsampling; 32 x 32: exactly one pass; 1 x 1, 1 x W.  Reference
    points inside, far left / above and far beyond W * stride.  (The fp64 oracle runs on the CPU: Q = 910 at 64^2 costs what
    Q = 230 does at 128^2.)"""
    _budget(5 if Q > 100 else 2)
    g = torch.Generator().manual_seed(Hf * 1000 + Wf)
    B = 2
    feats = torch.randn(B, 8, Hf, Wf, generator=g)
    params = torch.randn(B, Q, 169, generator=g) * 0.3
    ref_px = torch.rand(B, Q, 2, generator=g) * torch.tensor([Wf * 8.0, Hf * 8.0])
    ref_px[:, 0::5] = -torch.rand(B, len(range(0, Q, 5)), 2, generator=g) * 300
    ref_px[:, 1::5] = torch.tensor([Wf * 8.0, Hf * 8.0]) + torch.rand(B, len(range(1, Q, 5)), 2, generator=g) * 300
    out = ops.condinst_masks(feats.permute(0, 2, 3, 1).contiguous().to(cuda), params.to(cuda), ref_px.to(cuda), Hf, Wf)
    ref, bound = condinst_ref64(feats, params, ref_px)
    err = out.cpu().double() - ref
    assert bool((err.abs() <= bound).all()), (err.abs() / bound).max().item()
    passes, rem = _condinst_branch(Hf, Wf)
    assert (passes, rem) == {(128, 128): (16, 0), (160, 160): (25, 0), (64, 64): (4, 0), (100, 76): (8, 0), (37, 45): (2, 2),
                             (32, 32): (1, 0), (25, 41): (2, 2), (1, 1): (1, 2), (1, 64): (1, 0), (1, 37): (1, 2)}[(Hf, Wf)]


def test_condinst_shared_memory_limit(ops, cuda):
    """The coarse logits of one (query, image) live in shared memory: Hf * Wf * 4 <= 200 KB.  160 x 320 is exactly at the limit
    and runs; 3 x 17067 is one pixel over and is refused on the host before any launch."""
    _budget(5)
    g = torch.Generator().manual_seed(5)
    Hf, Wf = 160, 320
    assert Hf * Wf * 4 == 200 * 1024
    feats = torch.randn(1, 8, Hf, Wf, generator=g)
    params = torch.randn(1, 2, 169, generator=g) * 0.3
    ref_px = torch.tensor([[[700.0, 500.0], [-50.0, 2000.0]]])
    out = ops.condinst_masks(feats.permute(0, 2, 3, 1).contiguous().to(cuda), params.to(cuda), ref_px.to(cuda), Hf, Wf)
    ref, bound = condinst_ref64(feats, params, ref_px)
    assert bool(((out.cpu().double() - ref).abs() <= bound).all())
    Hf, Wf = 3, 17067
    assert Hf * Wf == 200 * 1024 // 4 + 1
    f = torch.zeros(1, Hf * Wf, 8, device=cuda)
    with pytest.raises(RuntimeError, match="bad sizes"):
        ops.condinst_masks(f, params[:, :1].to(cuda), ref_px[:, :1].to(cuda), Hf, Wf)


# ------------------------------------------------------------------------------------------ class_scores
def _cs_threads(C):
    """select.cu hipie_class_scores: 256 threads from C = 256, 128 from C = 128, 64 below."""
    return 256 if C >= 256 else (128 if C >= 128 else 64)


CS_CLASSES = [80, 127, 128, 150, 255, 256, 847]


def _cs_tables(C, Lt, maxlen, g):
    """Token spans of 1 ... maxlen tokens, padded with the first token; every 9th class absent (cnt 0); the last class's span
    ends at token Lt - 1."""
    cnt = torch.randint(1, maxlen + 1, (C,), generator=g, dtype=torch.int32)
    cnt[4::9] = 0
    cnt[C - 1] = maxlen
    tok = torch.zeros(C, maxlen, dtype=torch.int32)
    for c in range(C):
        n = max(int(cnt[c]), 1)
        start = Lt - n if c == C - 1 else int(torch.randint(0, Lt - maxlen, (1,), generator=g))
        tok[c, :n] = torch.arange(start, start + n, dtype=torch.int32)
        tok[c, n:] = start
    return tok, cnt


def _cs_tie_rows(C, threads, R, Lt, tok, cnt, g):
    """(R, Lt) logits: mostly randn * 3; saturated spans (>= 17: sigmoid == 1.0f exactly, <= -104: 0.0f) on groups of classes
    chosen so that exact prob ties fall across lanes of one warp, across warps, and on the classes one thread strides over."""
    logits = torch.randn(R, Lt, generator=g) * 3
    present = [c for c in range(C) if cnt[c] > 0]
    for r in range(R):
        kind = r % 5
        if kind == 0:                       # across lanes of warp 0
            grp = [present[1], present[3]]
        elif kind == 1:                     # across warps: class t and t + 32 (different warps of the block)
            grp = [c for c in present if c in (5, 37, 69)] or present[:2]
        elif kind == 2:                     # one thread's strided classes: t, t + threads (C > threads)
            grp = [c for c in present if c % threads == 7][:3]
            grp = grp if len(grp) > 1 else [present[-3], present[-1]]
        elif kind == 3:                     # random group, anywhere
            k = int(torch.randint(2, 6, (1,), generator=g))
            grp = [present[int(i)] for i in torch.randperm(len(present), generator=g)[:k]]
        else:                               # everything saturated low: every prob ties at its minimum
            logits[r] = -110.0 - torch.rand(Lt, generator=g)
            continue
        for c in grp:
            t = tok[c, :int(cnt[c])].long()
            logits[r, t] = 17.0 + torch.rand(len(t), generator=g) * 5
    return logits


@pytest.mark.parametrize("C", CS_CLASSES)
@pytest.mark.parametrize("Lt,max_pool", [(256, False), (256, True), (4096, False), (4096, True)])
def test_class_scores(ops, cuda, C, Lt, max_pool):
    """R = 2 x 910 rows.  Scores against fp64 within n u sum|l| (max pooling: exactly); prob against fp64 of the returned scores;
    row_max is exactly the maximum of the returned prob and row_arg the lowest index of it.  FG, BG and no masking."""
    _budget(2)
    g = torch.Generator().manual_seed(C * 7 + Lt + max_pool)
    R, maxlen = 2 * 910, 6
    threads = _cs_threads(C)
    assert C > 32 and (threads > 64) == (C >= 128) and (threads > 128) == (C >= 256)
    tok, cnt = _cs_tables(C, Lt, maxlen, g)
    logits = _cs_tie_rows(C, threads, R, Lt, tok, cnt, g)
    iou = torch.randn(R, generator=g)
    thing = torch.rand(C, generator=g) < 0.7
    tie_rows = 0
    for mode, masked in (("FG", ~thing), ("BG", thing), (None, None)):
        m8 = None if masked is None else masked.to(torch.int8).to(cuda)
        sc, prob, rmax, rarg = ops.class_scores(logits.to(cuda), tok.to(cuda), cnt.to(cuda), masked=m8, iou=iou.to(cuda),
                                                max_pool=max_pool)
        # fp64 restatement of the pooling
        lg = logits.to(cuda).double()[:, tok.long().to(cuda)]                    # (R, C, maxlen)
        valid = (torch.arange(maxlen, device=cuda)[None, :] < cnt.to(cuda)[:, None].long())[None]
        n = cnt.to(cuda).double().clamp(min=1)
        if max_pool:
            ref = torch.where(valid, lg, -float("inf")).amax(-1)
        else:
            ref = torch.where(valid, lg, 0.0).sum(-1) / n
        ref = torch.where(cnt.to(cuda)[None] > 0, ref, 0.0)
        tol = n * U * torch.where(valid, lg.abs(), 0.0).sum(-1)
        if masked is not None:
            ref = torch.where(masked.to(cuda)[None], -9999.0, ref)
            tol = torch.where(masked.to(cuda)[None], 0.0, tol)
        err = (sc.double() - ref).abs()
        if max_pool:
            assert bool((err == 0).all()), mode
        else:
            assert bool((err <= tol).all()), (mode, (err - tol).max().item())
        pref = torch.sqrt(torch.sigmoid(sc.double()) * torch.sigmoid(iou.to(cuda).double())[:, None])
        assert (prob.double() - pref).abs().max().item() < 8 * U, mode
        assert torch.equal(rmax, prob.max(1).values), mode
        cols = torch.arange(C, device=cuda, dtype=torch.int32).expand(R, C)
        first = torch.where(prob == rmax[:, None], cols, C).min(1).values
        assert torch.equal(rarg, first), (mode, int((rarg != first).sum()))
        tie_rows += int(((prob == rmax[:, None]).sum(1) > 1).sum())
    assert tie_rows >= R, "the tie rows did not tie"                   # without masking nearly every row ties


# ------------------------------------------------------------------------------------------ batched_nms
NMS_MAX = 1216                          # select.cu: the largest N whose pair bit matrix fits the 220 KB of shared memory
NMS_CASES = [900, 910, NMS_MAX]


def nms_ref32(boxes, scores, cls, thr):
    """Greedy class-aware NMS restated in numpy float32 with torchvision's coordinate-offset arithmetic
    (boxes + cls * (max + 1), IoU = inter / (area_a + area_b - inter) > thr) and the order (score desc, index asc).
    Returns (keep, smallest |IoU - thr| over the pairs the greedy pass decided on, in fp64)."""
    f = np.float32
    cx, cy, w, h = (boxes[:, i].astype(f) for i in range(4))
    x1, y1, x2, y2 = cx - f(0.5) * w, cy - f(0.5) * h, cx + f(0.5) * w, cy + f(0.5) * h
    mx = max(x1.max(), y1.max(), x2.max(), y2.max())
    off = cls.astype(f) * (mx + f(1))
    x1, y1, x2, y2 = x1 + off, y1 + off, x2 + off, y2 + off
    area = (x2 - x1) * (y2 - y1)
    order = np.lexsort((np.arange(len(scores)), -scores.astype(np.float64)))
    removed = np.zeros(len(scores), bool)
    keep, margin = [], np.inf
    with np.errstate(invalid="ignore", divide="ignore"):
        for k, i in enumerate(order):
            if removed[i]:
                continue
            keep.append(i)
            j = order[k + 1:]
            iw = np.maximum(np.minimum(x2[i], x2[j]) - np.maximum(x1[i], x1[j]), f(0))
            ih = np.maximum(np.minimum(y2[i], y2[j]) - np.maximum(y1[i], y1[j]), f(0))
            inter = iw * ih
            iou = inter / (area[i] + area[j] - inter)
            d = np.abs(iou.astype(np.float64) - thr)[~removed[j]]          # decisions still open
            d = d[np.isfinite(d)]
            if d.size:
                margin = min(margin, float(d.min()))
            removed[j] |= iou > f(thr)
    return np.array(keep, dtype=np.int64), margin


def _nms_batch(N, g):
    """B = 8 images, each a different regime: distinct scores (0, 1), classes up to 846 (1, 5), clusters of overlapping
    same-class boxes with equal scores and exact duplicates (2, 6), zero-area boxes (3), boxes outside [0, 1] (4, 7)."""
    B = 8
    boxes = torch.cat([torch.rand(B, N, 2, generator=g) * 0.8 + 0.1, torch.rand(B, N, 2, generator=g) * 0.3 + 0.02], -1)
    scores = torch.rand(B, N, generator=g)
    cls = torch.randint(0, 4, (B, N), generator=g, dtype=torch.int32)
    cls[1] = torch.randint(0, 847, (N,), generator=g, dtype=torch.int32)
    cls[1, :4] = 846
    cls[5] = torch.randint(800, 847, (N,), generator=g, dtype=torch.int32)
    for b in (0, 1, 5):                                      # near-duplicates so that suppression happens
        boxes[b, N // 2:N // 2 + N // 4] = boxes[b, :N // 4] + torch.randn(N // 4, 4, generator=g) * 0.01
        cls[b, N // 2:N // 2 + N // 4] = cls[b, :N // 4]
    for b in (2, 6):                                         # clusters of 8: one score, jittered boxes, two exact duplicates
        nc = N // 8
        base = boxes[b, :nc].repeat_interleave(8, 0)
        jit = torch.randn(nc * 8, 4, generator=g) * (0.004 if b == 2 else 0.02)
        boxes[b, :nc * 8] = base + jit
        boxes[b, 1:nc * 8:8] = boxes[b, 0:nc * 8:8]
        boxes[b, 5:nc * 8:8] = boxes[b, 3:nc * 8:8]
        scores[b, :nc * 8] = scores[b, :nc].repeat_interleave(8, 0)
        cls[b, :nc * 8] = cls[b, :nc].repeat_interleave(8, 0)
        perm = torch.randperm(N, generator=g)                # ties far apart in index order
        boxes[b], scores[b], cls[b] = boxes[b, perm], scores[b, perm], cls[b, perm]
    boxes[3, ::3, 2] = 0.0                                   # zero width, zero height, both; and exact duplicates of them
    boxes[3, 1::3, 3] = 0.0
    boxes[3, 2::6, 2:] = 0.0
    boxes[3, 5::6] = boxes[3, 2::6][:len(boxes[3, 5::6])]
    scores[3, 5::6] = scores[3, 2::6][:len(scores[3, 5::6])]
    for b in (4, 7):
        boxes[b, :, :2] = torch.rand(N, 2, generator=g) * 3 - 1
        boxes[b, :, 2:] = torch.rand(N, 2, generator=g) * 1.5
        boxes[b, N // 2:] = boxes[b, :N - N // 2] + torch.randn(N - N // 2, 4, generator=g) * 0.02
    return boxes, scores, cls


@pytest.mark.parametrize("N", NMS_CASES)
def test_batched_nms(ops, cuda, N):
    """Against the float32 restatement on every image (the contract: equal scores resolve by index), and against torchvision's
    coordinate-offset batched NMS (what torchvision.ops.batched_nms runs below 4000 box coordinates on the CPU; above, it
    switches to a per-class loop whose IoUs round differently) on every image whose scores are all distinct."""
    from torchvision.ops.boxes import _batched_nms_coordinate_trick as tv_batched_nms
    _budget(5)
    g = torch.Generator().manual_seed(N)
    boxes, scores, cls = _nms_batch(N, g)
    keep, nkeep = ops.batched_nms(boxes.to(cuda), scores.to(cuda), cls.to(cuda), 0.7)
    keep, nkeep = keep.cpu(), nkeep.cpu()
    n_tv = 0
    for b in range(boxes.shape[0]):
        ref, margin = nms_ref32(boxes[b].numpy(), scores[b].numpy(), cls[b].numpy(), 0.7)
        assert margin > 1e-6, (b, margin)                     # no decision sits within fp32 contraction of the threshold
        n = int(nkeep[b])
        assert n == len(ref), (b, n, len(ref))
        assert torch.equal(keep[b, :n].long(), torch.from_numpy(ref)), b
        assert bool((keep[b, n:] == -1).all())
        if len(torch.unique(scores[b])) == N:
            n_tv += 1
            cx, cy, w, h = boxes[b].unbind(-1)
            xyxy = torch.stack([cx - 0.5 * w, cy - 0.5 * h, cx + 0.5 * w, cy + 0.5 * h], -1)
            assert torch.equal(keep[b, :n].long(), tv_batched_nms(xyxy, scores[b], cls[b].long(), 0.7)), b
    assert n_tv >= 4


def test_batched_nms_refuses_past_limit(ops, cuda):
    """One box past NMS_MAX is refused on the host, before any launch."""
    boxes = torch.rand(1, NMS_MAX + 1, 4, device=cuda)
    with pytest.raises(RuntimeError, match="outside"):
        ops.batched_nms(boxes, torch.rand(1, NMS_MAX + 1, device=cuda), torch.zeros(1, NMS_MAX + 1, dtype=torch.int32, device=cuda), 0.7)


# ------------------------------------------------------------------------------------------ census
COVERED = ({("msda_fused", v, rd, sp, False) for v, rd, _ in FUSED_CASES for sp in (False, True)}
           | {("msda_fused", v, 2, sp, True) for v, _ in ENC_CASES for sp in (False, True)}
           | {("msda_forward", v) for v in ("f32", "bf16")}
           | {("condinst", p > 1, r) for p, r in (_condinst_branch(h, w) for h, w, _ in CONDINST_CASES)}
           | {("class_scores", _cs_threads(C)) for C in CS_CLASSES}
           | {("batched_nms", N) for N in NMS_CASES})


class _Census:
    """Wraps the five head-kernel launchers of ops for one forward and records each call's key: the kernel instance plus the
    launcher's size class."""

    NAMES = ("msda_fused", "msda_forward", "condinst_masks", "class_scores", "batched_nms")

    def __init__(self, ops):
        self.ops, self.calls = ops, {}
        self.orig = {n: getattr(ops, n) for n in self.NAMES}

    def __enter__(self):
        for n in self.NAMES:
            setattr(self.ops, n, getattr(self, "_" + n))
        return self

    def __exit__(self, *exc):
        for n, f in self.orig.items():
            setattr(self.ops, n, f)
        return False

    def _put(self, key, shape):
        self.calls.setdefault(key, set()).add(shape)

    @staticmethod
    def _vdt(t):
        return {torch.float32: "f32", torch.bfloat16: "bf16", torch.float16: "f16"}[t.dtype]

    def _msda_fused(self, value, shapes, lsi, offs_logits, refp, *a, **kw):
        split = kw.get("want_split", True)
        self._put(("msda_fused", self._vdt(value), refp.shape[-1], split, offs_logits.shape[1] == value.shape[1]),
                  f"N={value.shape[0]} Lq={offs_logits.shape[1]} S={value.shape[1]}")
        return self.orig["msda_fused"](value, shapes, lsi, offs_logits, refp, *a, **kw)

    def _msda_forward(self, value, *a, **kw):
        self._put(("msda_forward", self._vdt(value)), f"S={value.shape[1]}")
        return self.orig["msda_forward"](value, *a, **kw)

    def _condinst_masks(self, feats, params, ref_px, Hf, Wf, *a, **kw):
        p, r = _condinst_branch(Hf, Wf)
        self._put(("condinst", p > 1, r), f"B={params.shape[0]} Q={params.shape[1]} {Hf}x{Wf}")
        return self.orig["condinst_masks"](feats, params, ref_px, Hf, Wf, *a, **kw)

    def _class_scores(self, logits, tok, *a, **kw):
        self._put(("class_scores", _cs_threads(tok.shape[0])), f"R={logits.shape[0]} Lt={logits.shape[1]} C={tok.shape[0]}")
        return self.orig["class_scores"](logits, tok, *a, **kw)

    def _batched_nms(self, boxes, scores, *a, **kw):
        self._put(("batched_nms", scores.shape[1]), f"B={scores.shape[0]}")
        return self.orig["batched_nms"](boxes, scores, *a, **kw)


def _census_c1_forward():
    """One c1 forward (ViT-H, 1024 x 1024, 80 classes, synthetic weights, built as test_operating_range_c1 builds it) with the
    head-kernel launchers wrapped -> {key: set of shapes}."""
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
    with torch.no_grad(), _Census(ops) as cen:
        model(inputs)
    torch.cuda.synchronize()
    return cen.calls


def test_census_c1_forward(cuda):
    """Every head-kernel key one c1 forward launches is one this file tests (the forward runs in a child process, see
    _in_child)."""
    _budget(90)
    rec = _in_child("--census")
    calls = {tuple(k): set(v) for k, v in rec["calls"]}
    print(f"\n[census] c1 forward on {rec['device']}: head-kernel keys launched")
    for key, shapes in sorted(calls.items(), key=str):
        print(f"  {str(key):44s} {'covered' if key in COVERED else 'NOT COVERED':12s} {', '.join(sorted(shapes))}")
    assert {k[0] for k in calls} >= {"msda_fused", "condinst", "class_scores", "batched_nms"}, calls
    missing = set(calls) - COVERED
    assert not missing, missing


if __name__ == "__main__" and sys.argv[1:] == ["--census"]:
    print(json.dumps(dict(device=torch.cuda.get_device_name(0), calls=[[list(k), sorted(v)] for k, v in _census_c1_forward().items()])))
elif __name__ == "__main__" and sys.argv[1:] == ["--instances"]:
    print(json.dumps([[[list(k), n] for k, n in part] for part in _msda_instance_counts()]))
