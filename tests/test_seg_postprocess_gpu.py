"""GPU: the kernels that turn mask logits into what a user gets back (postproc.cu), at the geometry a forward launches them
with, against an fp64 restatement computed from exactly the fp32 logits and class probabilities the kernels read.

| Launcher | Branch / instance | Taken when | Tests |
|---|---|---|---|
| `hipie_seg_postprocess` | `seg_post_kernel<10>` | C <= 80 | `test_seg_geometry` (C = 1, 8, 80), `test_seg_crop_sweep`, `test_seg_scores` |
| same | `seg_post_kernel<17>` | 80 < C <= 136 | `test_seg_geometry` (C = 81, 136, Q = 8192) |
| `ops.seg_postprocess` | class chunks of 80, last one narrower | C > 136 | `test_seg_class_chunks` (C = 137, 150, 847) |
| same | both double-buffer parities of the 64-query chunks | Qpad / 64 odd and even | `test_seg_geometry` (Q = 1 ... 1200) |
| same | shared-memory limit (host check) | 3 * Qpad * 4 + tiles <= 220 KB | `test_seg_refuses_past_shared_memory` |
| same | ragged last CTA row / column, Hc or Wc = 1, crops 0..31 | image not a multiple of 32 x 8 | `test_seg_geometry`, `test_seg_crop_sweep` |
| same | argmax fallback to the first kept query, tie rule, flag | underflowed sigmoid, duplicate masks | `test_seg_scores`, `test_seg_constant_maps` |
| same | winner's flag recomputed after the argmax, bit for bit the count's sigmoid | every kept winner | `test_seg_flag_matches_count_at_the_edge` |
| `hipie_upsample_threshold` | grid-stride loop over `num_sms * 32` blocks | N * Hc * ceil((Wc + 2) / 4) > num_sms * 32 * 256 | `test_upsample_threshold_geometry`, `test_upsample_threshold_grid_cap` |
| `fused_sem_pano_launch` + `_finish` | the panoptic merge from the counters | every fused forward | `test_merge_matches_reference`, `test_merge_overlap_ratio` |
| all of the above | what one c1 forward launches | ViT-H, 1024 x 1024, 80 classes | `test_census_c1_forward` |

Every launch of `hipie_seg_postprocess` with C <= 136 goes through `_launch`, which surrounds `sem`, `ids` and `areas` with
sentinels and guard elements: every pixel of the crop must be written, and neither the guard nor `sem` rows >= C touched.

Ambiguity band (derived from the arithmetic, not fitted).  u = 2^-24; M = the largest |tap| of the four low-resolution taps a
pixel reads.  The kernel stages -log2(e) * logit (two roundings) and interpolates with two differences and two fma, the
weights being exact multiples of 1/8: its logit is within 8 u M of the fp64 one.  The fp32 reference `sigmoid(x) >= 0.5`
holds while fp32 rounds 1 + exp(-x) to 2, i.e. for x >= about -1.8e-7; with exp / ex2 / rcp within 2 ulp that edge lies in
[-4 * 2^-23, 2^-23].  A (pixel, query) pair is *predicate-ambiguous* when its fp64 logit is within 8 u M of that interval.
The kernel's sigmoid is within (1 - s) 8 u M (interpolation) + 8 u (ex2.approx, the add, rcp.approx) relative of the fp64
one, the product with the score adds u, and rcp.approx.ftz flushes results below 2^-126 to 0: a product p is within
p r + score 2^-125 with r = (1 - s) 8 u M + 9 u.  A pixel is *argmax-ambiguous* when some other kept query's upper bound
reaches the restated winner's lower bound.  Outside the band the ids must be equal; each counter may differ from the
restatement by at most that query's count of ambiguous pixels.

`sem` is bf16x3 (hi*hi + hi*lo + lo*hi): each term is within 2^-16 of p_qc s_q (split residuals 2 * 2^-18, the missing lo*lo
2^-18), the sigmoid error above is within 8 u (M_q + 1) relative, and the fp32 tensor-core accumulation over 3 Qpad / 16
mma steps costs <= 2 ulp per step relative to the sum of terms: per element the bound is
sum_q p_qc s_q (2^-16 + 8 u (M_q + 1) + 2 * 3 Qpad / 16 * 2^-23).

The census's model forward runs in a child process (`_in_child`), as in test_detection_heads_gpu.py.
"""
import json
import sys
import time
import types

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

_T0 = None                                           # set when the first test of this file starts (_clock)
BUDGET_S = 300.0
U = 2.0 ** -24
SIG_LO, SIG_HI = -4 * 2.0 ** -23, 2.0 ** -23        # logits where the fp32 `sigmoid >= 0.5` may go either way
TINY = 2.0 ** -125                                   # absolute error of a product (rcp.approx.ftz)
SEM_SENT, ID_SENT, AREA_SENT, U8_SENT = -12345.0, -7, -9, 0xAB
GUARD = 4099


@pytest.fixture(scope="module")
def ops(cuda):
    from hipie_b200 import ops as o
    o.set_precision(3)
    return o


@pytest.fixture(scope="module", autouse=True)
def _clock():
    """Start the time budget at this file's first test, not at collection: in a whole-suite run the files collected before it
    run first."""
    global _T0
    _T0 = time.time()


def _budget(need):
    if time.time() - _T0 + need > BUDGET_S:
        pytest.skip(f"time budget: {time.time() - _T0:.0f}s used, case needs ~{need:.0f}s")


def _smem(nt, qpad):
    """launch_seg_post's shared-memory size: taps, P^T hi / lo double buffers, scores, three counter rows."""
    return 2 * 64 * 27 * 4 + 4 * nt * 8 * 72 * 2 + 2 * 64 * 4 + 3 * qpad * 4


def _kept(prob, thr):
    sc = prob.max(-1)[0]
    return torch.where(sc > thr, sc, torch.zeros_like(sc))


def _launch(ops, masks, prob, thr, Hc, Wc):
    """One hipie_seg_postprocess launch (C <= 136), exactly as ops.seg_postprocess prepares it, with `sem`, `ids` and `areas`
    followed by sentinel guards (and `sem` by the unused accumulator rows) -> sem (C, Hc, Wc), ids (Hc, Wc), areas (3, Q)."""
    from hipie_b200 import _lib
    Q, h, w = masks.shape
    C = prob.shape[1]
    dev = masks.device
    Qpad = (Q + 63) // 64 * 64
    rows = 80 if C <= 80 else 136
    pt = torch.zeros((rows, Qpad), dtype=torch.float32, device=dev)
    pt[:C, :Q] = prob.t()
    hi = pt.to(torch.bfloat16)
    lo = (pt - hi.float()).to(torch.bfloat16)
    sc = torch.zeros((Qpad,), dtype=torch.float32, device=dev)
    sc[:Q] = _kept(prob, thr)
    plane = Hc * Wc
    sem = torch.full((rows * plane + GUARD,), SEM_SENT, dtype=torch.float32, device=dev)
    ids = torch.full((plane + GUARD,), ID_SENT, dtype=torch.int32, device=dev)
    areas = torch.full((3 * Q + GUARD,), AREA_SENT, dtype=torch.int32, device=dev)
    _lib.check(_lib.load().hipie_seg_postprocess(ops._p(masks.contiguous()), ops._p(hi), ops._p(lo), ops._p(sc), ops._p(sem),
                                                 ops._p(ids), ops._p(areas), Q, Qpad, C, h, w, 4, Hc, Wc, ops._stream()),
               "seg_postprocess")
    assert bool((sem[C * plane:] == SEM_SENT).all()), "sem written past row C - 1"
    assert bool((ids[plane:] == ID_SENT).all()) and bool((areas[3 * Q:] == AREA_SENT).all()), "guard written"
    sem, ids = sem[:C * plane].view(C, Hc, Wc), ids[:plane].view(Hc, Wc)
    assert bool((sem != SEM_SENT).all()) and bool((ids != ID_SENT).all()), "pixel of the crop not written"
    return sem, ids, areas[:3 * Q].view(3, Q)


# ------------------------------------------------------------------------------------------ fp64 restatement
def _axis(n_out, n_in, dev):
    """align_corners=False x4 source taps of each output index: i0, i1, weight of i1 (fp64)."""
    src = ((torch.arange(n_out, device=dev, dtype=torch.float64) + 0.5) * 0.25 - 0.5).clamp(min=0)
    i0 = src.floor().long().clamp(max=n_in - 1)
    i1 = (i0 + 1).clamp(max=n_in - 1)
    return i0, i1, src - i0


def _up64(m, ax, ay):
    """(q, h, w) -> fp64 bilinear x4 (align_corners=False), cropped, and the largest |tap| each pixel reads."""
    (y0, y1, ly), (x0, x1, lx) = ay, ax
    m = m.double()
    r0, r1 = m[:, y0], m[:, y1]
    t00, t01, t10, t11 = r0[:, :, x0], r0[:, :, x1], r1[:, :, x0], r1[:, :, x1]
    ly, lx = ly.view(1, -1, 1), lx.view(1, 1, -1)
    x = (1 - ly) * ((1 - lx) * t00 + lx * t01) + ly * ((1 - lx) * t10 + lx * t11)
    mag = torch.maximum(torch.maximum(t00.abs(), t01.abs()), torch.maximum(t10.abs(), t11.abs()))
    return x, mag


def _at64(m, ay, ax, yy, xx):
    """The same at the pixels (yy, xx) only -> (q, n)."""
    y0, y1, ly = (a[yy] for a in ay)
    x0, x1, lx = (a[xx] for a in ax)
    t00, t01, t10, t11 = (m[:, a, b].double() for a, b in ((y0, x0), (y0, x1), (y1, x0), (y1, x1)))
    x = (1 - ly) * ((1 - lx) * t00 + lx * t01) + ly * ((1 - lx) * t10 + lx * t11)
    mag = torch.maximum(torch.maximum(t00.abs(), t01.abs()), torch.maximum(t10.abs(), t11.abs()))
    return x, mag


def _pred_amb(x, mag):
    eps = 8 * U * mag
    return (x >= SIG_LO - eps) & (x <= SIG_HI + eps)


def restate(masks, prob, thr, Hc, Wc, chunk=64):
    """fp64 restatement of seg_post_kernel from the fp32 operands it reads.  Returns a dict: sem (C, Hc, Wc), tol (its
    per-element bound), ids (the restated 2 q + flag, -1 without kept queries), band (pixels where ids may differ), area
    (3, Q) and allow (3, Q) = the per-query count of ambiguous pixels."""
    Q, h, w = masks.shape
    C = prob.shape[1]
    dev = masks.device
    Qpad = (Q + 63) // 64 * 64
    ax, ay = _axis(Wc, w, dev), _axis(Hc, h, dev)
    ksc = _kept(prob, thr).double()
    keep = ksc > 0
    P = prob.double()
    Mq = masks.abs().flatten(1).amax(1).double()
    wq = 2.0 ** -16 + 8 * U * (Mq + 1) + 2 * 3 * Qpad / 16 * 2.0 ** -23
    HW = Hc * Wc
    sem = torch.zeros(C, HW, dtype=torch.float64, device=dev)
    tol = torch.zeros(C, HW, dtype=torch.float64, device=dev)
    orig = torch.zeros(Q, dtype=torch.long, device=dev)
    amb1 = torch.zeros(Q, dtype=torch.long, device=dev)
    best = torch.full((HW,), -1.0, dtype=torch.float64, device=dev)
    win = torch.full((HW,), -1, dtype=torch.long, device=dev)
    low_w = torch.zeros(HW, dtype=torch.float64, device=dev)
    x_w = torch.zeros(HW, dtype=torch.float64, device=dev)
    mag_w = torch.zeros(HW, dtype=torch.float64, device=dev)
    top_u = torch.full((2, HW), -float("inf"), dtype=torch.float64, device=dev)
    top_i = torch.full((2, HW), -1, dtype=torch.long, device=dev)
    for q0 in range(0, Q, chunk):
        q1 = min(Q, q0 + chunk)
        x, mag = _up64(masks[q0:q1], ax, ay)
        x, mag = x.view(q1 - q0, HW), mag.view(q1 - q0, HW)
        s = torch.sigmoid(x)
        sem += P[q0:q1].t() @ s
        tol += (P[q0:q1] * wq[q0:q1, None]).t() @ s
        orig[q0:q1] = (x >= 0).sum(1)
        amb1[q0:q1] = _pred_amb(x, mag).sum(1)
        k = ksc[q0:q1, None]
        p = torch.where(k > 0, s * k, torch.full_like(s, -1.0))
        r = (1 - s) * 8 * U * mag + 9 * U
        upper = torch.where(k > 0, p * (1 + r) + k * TINY, torch.full_like(s, -float("inf")))
        cmax, carg = p.max(0)                       # first maximal index, as torch.argmax
        upd = cmax > best
        sel = carg.view(1, HW)
        best = torch.where(upd, cmax, best)
        win = torch.where(upd, carg + q0, win)
        low_w = torch.where(upd, (p * (1 - r) - k * TINY).gather(0, sel)[0], low_w)
        x_w = torch.where(upd, x.gather(0, sel)[0], x_w)
        mag_w = torch.where(upd, mag.gather(0, sel)[0], mag_w)
        cu, ci = torch.cat([top_u, upper]), torch.cat([top_i, torch.arange(q0, q1, device=dev).view(-1, 1).expand(-1, HW)])
        top_u, j = cu.topk(2, dim=0)
        top_i = ci.gather(0, j)
    out = dict(sem=sem.view(C, Hc, Wc), tol=tol.view(C, Hc, Wc))
    area = torch.zeros(3, Q, dtype=torch.long, device=dev)
    allow = torch.zeros(3, Q, dtype=torch.long, device=dev)
    area[1], allow[1] = orig, amb1
    if not bool(keep.any()):
        out.update(ids=torch.full((Hc, Wc), -1, dtype=torch.long, device=dev), band=torch.zeros(Hc, Wc, dtype=torch.bool, device=dev),
                   area=area, allow=allow, n_arg=0, n_pred=0)
        return out
    flag = x_w >= 0
    other_u = torch.where(top_i[0] == win, top_u[1], top_u[0])
    amb_arg = other_u >= low_w
    amb_flag = _pred_amb(x_w, mag_w)
    area[0] = torch.bincount(win, minlength=Q)
    area[2] = torch.bincount(win[flag], minlength=Q)
    # queries that could own an argmax-ambiguous pixel: the winner and every kept query whose upper bound reaches it
    pix = amb_arg.nonzero()[:, 0]
    contend = torch.zeros(Q, dtype=torch.long, device=dev)
    for c0 in range(0, pix.numel(), 1 << 14):
        pp = pix[c0:c0 + (1 << 14)]
        for q0 in range(0, Q, 1024):
            q1 = min(Q, q0 + 1024)
            xs, mag = _at64(masks[q0:q1], ay, ax, pp // Wc, pp % Wc)
            s = torch.sigmoid(xs)
            k = ksc[q0:q1, None]
            up = s * k * (1 + (1 - s) * 8 * U * mag + 9 * U) + k * TINY
            c = (k > 0) & ((up >= low_w[pp]) | (torch.arange(q0, q1, device=dev).view(-1, 1) == win[pp]))
            contend[q0:q1] += c.sum(1)
    allow[0] = contend
    allow[2] = contend + torch.bincount(win[amb_flag], minlength=Q)
    out.update(ids=(2 * win + flag.long()).view(Hc, Wc), band=(amb_arg | amb_flag).view(Hc, Wc), area=area, allow=allow,
               n_arg=int(amb_arg.sum()), n_pred=int(amb1.sum()))
    return out


def _check(sem, ids, areas, ref, label=""):
    """The exact assertions shared by every case."""
    ids, areas = ids.long(), areas.long()
    Q = areas.shape[1]
    own = ids >= 0
    assert torch.equal(areas[0], torch.bincount((ids[own] >> 1).flatten(), minlength=Q)), "mask area != pixels owned"
    odd = own & (ids & 1).bool()
    assert torch.equal(areas[2], torch.bincount((ids[odd] >> 1).flatten(), minlength=Q)), "intersection area != odd ids"
    assert bool((areas[2] <= areas[1]).all()), "intersection area > original area"
    assert bool((areas[2] <= areas[0]).all())
    band = ref["band"]
    bad = (ids != ref["ids"]) & ~band
    assert not bool(bad.any()), f"{int(bad.sum())} ids outside the band differ, first at {bad.nonzero()[0].tolist()}"
    d = (areas - ref["area"]).abs()
    over = d > ref["allow"]
    assert not bool(over.any()), f"counter beyond its allowance: (row, q) {over.nonzero()[:4].tolist()}"
    err = (sem.double() - ref["sem"]).abs()
    assert bool((err <= ref["tol"]).all()), f"sem beyond its bound: max err {err.max():.3e}, worst ratio {(err / ref['tol']).max():.2f}"
    print(f"[{label}] band pixels {int(band.sum())} (argmax {ref['n_arg']}), predicate-ambiguous pairs {ref['n_pred']}, "
          f"max |counter - restated| {d.max(1)[0].tolist()} within {ref['allow'].max(1)[0].tolist()}")


def _data(Q, C, h, w, seed, dev, scale=4.0):
    g = torch.Generator(device=dev).manual_seed(seed)
    masks = torch.randn(Q, h, w, device=dev, generator=g) * scale
    prob = torch.softmax(torch.randn(Q, C, device=dev, generator=g) * 3, -1)
    return masks, prob


# ------------------------------------------------------------------------------------------ seg_post_kernel: geometry
GEOMETRY = [  # Q, C, h, w, Hc, Wc, object-mask threshold
    (1, 1, 24, 20, 96, 80, 0.25), (63, 8, 24, 20, 93, 78, 0.25), (64, 80, 24, 20, 94, 79, 0.25), (64, 80, 24, 20, 94, 79, 0.01),
    (65, 80, 10, 16, 39, 63, 0.25), (129, 81, 24, 40, 95, 157, 0.25), (129, 81, 24, 40, 95, 157, 0.01),
    (70, 136, 12, 40, 48, 160, 0.25), (64, 80, 2, 2, 8, 8, 0.25), (5, 8, 2, 2, 1, 1, 0.01), (7, 80, 2, 9, 1, 36, 0.25),
    (7, 81, 9, 2, 36, 1, 0.25), (1200, 80, 256, 256, 1024, 1024, 0.25), (1200, 80, 256, 256, 1024, 1024, 0.01),
    (129, 136, 171, 256, 683, 1024, 0.25), (65, 81, 256, 171, 1024, 683, 0.01), (8192, 136, 48, 48, 190, 187, 0.25),
]


@pytest.mark.parametrize("Q,C,h,w,Hc,Wc,thr", GEOMETRY)
def test_seg_geometry(ops, cuda, Q, C, h, w, Hc, Wc, thr):
    """Q across the 64-query chunks (1, 63, 64, 65, 129, 1200 = 19 chunks, 8192), both accumulator tiles, Hc / Wc of every residue
    mod 4, Hc or Wc = 1, h = w = 2, last CTA row / column with one block inside (39 x 63), the production image sizes, the model's
    object-mask threshold 0.25 and the demo's 0.01."""
    _budget(20 if Q * Hc * Wc > 1e8 else 3)
    masks, prob = _data(Q, C, h, w, Q + C + h, cuda)
    sem, ids, areas = _launch(ops, masks, prob, thr, Hc, Wc)
    _check(sem, ids, areas, restate(masks, prob, thr, Hc, Wc), f"Q={Q} C={C} {Hc}x{Wc} thr={thr}")


def test_seg_crop_sweep(ops, cuda):
    """Crops 4h - Hc and 4w - Wc from 0 to 31 (every residue mod 4 in both axes) on one 9 x 10 low-resolution grid."""
    _budget(10)
    masks, prob = _data(70, 13, 9, 10, 31, cuda)
    for cy in range(32):
        cx = 31 - cy
        Hc, Wc = max(36 - cy, 1), max(40 - cx, 1)
        sem, ids, areas = _launch(ops, masks, prob, 0.25, Hc, Wc)
        _check(sem, ids, areas, restate(masks, prob, 0.25, Hc, Wc), f"crop {cy},{cx}")


@pytest.mark.parametrize("C", [137, 150, 847])
def test_seg_class_chunks(ops, cuda, C):
    """Vocabularies wider than one accumulator tile: ops.seg_postprocess runs class chunks of 80 (the last one 57, 70, 47)."""
    _budget(5)
    masks, prob = _data(129, C, 24, 30, C, cuda)
    sem, ids, areas, scores, labels = ops.seg_postprocess(masks, prob, 0.01, 95, 118)
    assert torch.equal(labels, prob.max(-1)[1])
    _check(sem, ids, areas, restate(masks, prob, 0.01, 95, 118), f"C={C}")


@pytest.mark.parametrize("nt,Qok", [(10, 13696), (17, 11008)])
def test_seg_refuses_past_shared_memory(ops, cuda, nt, Qok):
    """The largest Qpad whose counters fit the 220 KB of shared memory is launched; one 64-query chunk more is refused with an
    error before any launch, and writes nothing but the zeroed counters."""
    from hipie_b200 import _lib
    assert _smem(nt, Qok) <= 220 * 1024 < _smem(nt, Qok + 64)
    C = 80 if nt == 10 else 136
    Q = Qok + 1
    masks, prob = _data(Q, C, 2, 2, nt, cuda)
    plane = 8 * 8
    sem = torch.full((C * plane,), SEM_SENT, device=cuda)
    ids = torch.full((plane,), ID_SENT, dtype=torch.int32, device=cuda)
    areas = torch.zeros((3 * Q,), dtype=torch.int32, device=cuda)
    pt = torch.zeros((C, Q + 63), dtype=torch.bfloat16, device=cuda)
    sc = torch.zeros((Q + 63,), device=cuda)
    n0 = _lib.launch_count()
    rc = _lib.load().hipie_seg_postprocess(ops._p(masks), ops._p(pt), ops._p(pt), ops._p(sc), ops._p(sem), ops._p(ids), ops._p(areas),
                                           Q, (Q + 63) // 64 * 64, C, 2, 2, 4, 8, 8, ops._stream())
    torch.cuda.synchronize()
    assert rc != 0 and b"shared memory" in _lib.load().hipie_last_error()
    assert _lib.launch_count() == n0
    assert bool((sem == SEM_SENT).all()) and bool((ids == ID_SENT).all())
    m2, p2 = masks[:Qok], prob[:Qok]
    s2, i2, a2 = _launch(ops, m2, p2, 0.25, 8, 8)
    _check(s2, i2, a2, restate(m2, p2, 0.25, 8, 8), f"Qpad={Qok}")


# ------------------------------------------------------------------------------------------ scores and logits
def _fp32_chain(masks, prob, thr, Hc, Wc):
    """The reference op chain in fp32 (hipie_img.py panoptic_inference on F.interpolate): ids and the three counters."""
    Q, h, w = masks.shape
    up = F.interpolate(masks[:, None], size=(4 * h, 4 * w), mode="bilinear", align_corners=False)[:, 0, :Hc, :Wc]
    sg = up.sigmoid()
    sc = _kept(prob, thr)
    keep = sc > 0
    if not bool(keep.any()):
        return (torch.full((Hc, Wc), -1, dtype=torch.long, device=masks.device),
                torch.stack([torch.zeros(Q, dtype=torch.long, device=masks.device), (sg >= 0.5).flatten(1).sum(1),
                             torch.zeros(Q, dtype=torch.long, device=masks.device)]))
    kidx = keep.nonzero()[:, 0]
    win = kidx[(sc[keep].view(-1, 1, 1) * sg[keep]).argmax(0)]
    inter = sg.gather(0, win[None])[0] >= 0.5
    own = win[None] == torch.arange(Q, device=masks.device).view(Q, 1, 1)
    areas = torch.stack([own.flatten(1).sum(1), (sg >= 0.5).flatten(1).sum(1), (own & (sg >= 0.5)).flatten(1).sum(1)])
    return 2 * win + inter.long(), areas


CONSTANTS = [-3e-8, 3e-8, -1e-6, 0.0, 100.0, -100.0, 1e4, -1e4]


def _rows(scores, thr, dev, C=128):
    """Class-probability rows whose maximum is the given score; None = exactly the threshold (not kept, the test is `>`)."""
    out = []
    for s in scores:
        r = torch.zeros(C)
        if s is None:
            r[:round(1 / thr)] = thr
        else:
            r[:] = (1 - s) / (C - 1)
            r[0] = s
        out.append(r)
    return torch.stack(out).to(dev)


@pytest.mark.parametrize("thr", [0.25, 0.01])
def test_seg_constant_maps(ops, cuda, thr):
    """Constant logit maps interpolate exactly, so ids and counters must equal the fp32 reference with no band: logits in the
    band where fp32 rounds sigmoid to 0.5 (-3e-8, 3e-8, 0 are inside, -1e-6 is not), saturated +-100 / +-1e4 where the products
    tie at the score, sigmoid underflow (every kept product 0 -> first kept query, flag 0), exact zeros.  Query 0 scores exactly
    the threshold and is not kept; 0.005 is below either threshold."""
    Hc, Wc = 37, 45
    for c in CONSTANTS:                                           # one kept query, index 2
        masks = torch.full((4, 10, 12), c, device=cuda)
        prob = _rows([None, 0.005, 0.6, 0.005], thr, cuda)
        sem, ids, areas = _launch(ops, masks, prob, thr, Hc, Wc)
        rid, rar = _fp32_chain(masks, prob, thr, Hc, Wc)
        assert torch.equal(ids.long(), rid), (c, ids.unique().tolist(), rid.unique().tolist())
        assert torch.equal(areas.long(), rar), (c, areas.tolist(), rar.tolist())
    # several kept queries: equal scores tie at +100 / +1e4 / 0 / 0.5 -> lowest index; all underflowed -> first kept (index 1)
    for vals, want in (((100.0, 100.0, 100.0), 1), ((1e4, 1e4, -1e4), 1), ((0.0, 0.0, 0.0), 1), ((-1e4, -1e4, -1e4), 1),
                       ((-100.0, -100.0, -100.0), 1), ((-100.0, 100.0, 100.0), 2), ((-3e-8, -3e-8, 3e-8), 1)):
        masks = torch.stack([torch.full((10, 12), v, device=cuda) for v in (5.0,) + vals])
        prob = _rows([None, 0.7, 0.7, 0.7], thr, cuda)
        sem, ids, areas = _launch(ops, masks, prob, thr, Hc, Wc)
        rid, rar = _fp32_chain(masks, prob, thr, Hc, Wc)
        assert torch.equal(ids.long(), rid) and torch.equal(areas.long(), rar), (vals, ids.unique().tolist(), rid.unique().tolist())
        assert bool(((ids >> 1) == want).all()), (vals, ids.unique().tolist())


def test_seg_scores(ops, cuda):
    """No query kept; a score exactly at the threshold (not kept: `>`); the first kept query not at index 0 and a kept query
    whose sigmoid underflows everywhere; duplicated masks with equal scores (the lower index takes every pixel the copy would)
    and with different scores; logits +-100 and +-1e4."""
    Q, h, w, Hc, Wc = 40, 16, 20, 62, 77
    masks, prob = _data(Q, 8, h, w, 9, cuda)
    flat = torch.full((Q, 8), 1 / 8, device=cuda)                       # 1/8 == threshold: nothing kept
    sem, ids, areas = _launch(ops, masks, flat, 0.125, Hc, Wc)
    assert bool((ids == -1).all()) and not bool(areas[0].any()) and not bool(areas[2].any())
    _check(sem, ids, areas, restate(masks, flat, 0.125, Hc, Wc), "none kept")
    p, m = prob.clone(), masks.clone()
    p[:3] = 1 / 8
    p[5] = _rows([0.5], 0.125, cuda, C=8)[0]
    m[5] = -1e4
    sem, ids, areas = _launch(ops, m, p, 0.125, Hc, Wc)
    _check(sem, ids, areas, restate(m, p, 0.125, Hc, Wc), "underflow")
    assert areas[:, 5].tolist() == [0, 0, 0]
    # duplicated masks: q 7 copies q 4 with the same class probabilities -> never wins; its original area equals q 4's
    m, p = masks.clone(), prob.clone()
    p[4] = _rows([0.95], 0.25, cuda, C=8)[0]
    m[7], p[7] = m[4], p[4]
    sem, ids, areas = _launch(ops, m, p, 0.25, Hc, Wc)
    assert int(areas[0, 4]) > 0 and not bool(((ids >> 1) == 7).any()) and int(areas[1, 7]) == int(areas[1, 4])
    p_off = p.clone()
    p_off[7] = 1 / 8                                                       # the copy not kept: ids and owners unchanged
    _, ids2, areas2 = _launch(ops, m, p_off, 0.25, Hc, Wc)
    assert torch.equal(ids, ids2) and torch.equal(areas[:, :7], areas2[:, :7]) and torch.equal(areas[0], areas2[0])
    # the copy with a higher score takes every pixel the original won
    p[7] = _rows([0.99], 0.25, cuda, C=8)[0]
    sem, ids, areas = _launch(ops, m, p, 0.25, Hc, Wc)
    _check(sem, ids, areas, restate(m, p, 0.25, Hc, Wc), "duplicate, higher score")
    assert not bool(((ids >> 1) == 4).any()) and int(areas[0, 7]) > 0
    for big in (100.0, 1e4):                                               # saturated logits
        m = torch.sign(masks) * big
        sem, ids, areas = _launch(ops, m, prob, 0.25, Hc, Wc)
        _check(sem, ids, areas, restate(m, prob, 0.25, Hc, Wc), f"+-{big}")


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_seg_flag_matches_count_at_the_edge(ops, cuda, seed):
    """One kept query owns every pixel, so each pixel counted in its original area must carry the intersection flag and vice
    versa: intersection area == original area exactly.  The logits put the interpolated value at the sigmoid >= 0.5 edge from
    large taps that cancel (columns a, b with 5/8 a + 3/8 b = eps, |a| up to 30, eps in [-4e-7, 2e-7]), where one rounding more or
    less in the tap arithmetic moves the value across the edge: a flag computed by other arithmetic than the count's fails."""
    h, w = 64, 64
    g = torch.Generator().manual_seed(seed)
    a = torch.rand(h, 1, generator=g, dtype=torch.float64) * 29 + 1
    eps = torch.rand(h, 1, generator=g, dtype=torch.float64) * 6e-7 - 4e-7
    m = torch.empty(1, h, w, dtype=torch.float32)
    m[0, :, 0::2] = a.float()
    m[0, :, 1::2] = (-5 / 3 * a.float().double() + 8 / 3 * eps).float()
    prob = _rows([0.9], 0.25, cuda, C=8)
    sem, ids, areas = _launch(ops, m.to(cuda), prob, 0.25, 4 * h, 4 * w)
    assert bool((ids >> 1 == 0).all())
    n_in = int(areas[1, 0])
    assert 0 < n_in < 16 * h * w
    assert int(areas[2, 0]) == n_in and int(areas[0, 0]) == 16 * h * w, areas[:, 0].tolist()
    print(f"[edge seed {seed}] {n_in} of {16 * h * w} pixels inside")


# ------------------------------------------------------------------------------------------ upsample_threshold
def _ut_launch(ops, masks, thr, Hc, Wc):
    from hipie_b200 import _lib
    N, h, w = masks.shape
    out = torch.full((N * Hc * Wc + GUARD,), U8_SENT, dtype=torch.uint8, device=masks.device)
    _lib.check(_lib.load().hipie_upsample_threshold(ops._p(masks.contiguous()), ops._p(out), N, h, w, 4, Hc, Wc, float(thr),
                                                    ops._stream()), "upsample_threshold")
    assert bool((out[N * Hc * Wc:] == U8_SENT).all()), "guard written"
    o = out[:N * Hc * Wc].view(N, Hc, Wc)
    assert bool((o <= 1).all()), "pixel of the crop not written"
    return o.bool()


def _ut_check(masks, out, thr, Hc, Wc, label):
    """Exact equality with fp64 sigmoid > thr outside the band: the kernel's logit (fp32 products and sums of exact weights) is
    within 8 u M of the fp64 one, and expf / the add / the division move the sigmoid by <= 6 u, i.e. the logit by
    <= 6 u / (1 - thr) <= 16 u."""
    import math
    t32 = float(torch.tensor(thr, dtype=torch.float32))
    x0 = math.log(t32 / (1 - t32))
    N = masks.shape[0]
    ax, ay = _axis(Wc, masks.shape[2], masks.device), _axis(Hc, masks.shape[1], masks.device)
    nb = 0
    for n0 in range(0, N, 16):
        x, mag = _up64(masks[n0:n0 + 16], ax, ay)
        band = (x - x0).abs() <= 8 * U * mag + 16 * U
        want = torch.sigmoid(x) > t32
        bad = (out[n0:n0 + 16] != want) & ~band
        assert not bool(bad.any()), f"{label}: {int(bad.sum())} pixels differ outside the band"
        nb += int(band.sum())
    print(f"[{label}] band pixels {nb}")


UT_GEOMETRY = [(1, 256, 256, 1024, 1024), (100, 256, 256, 1024, 1024), (100, 171, 256, 683, 1024), (1, 256, 171, 1024, 683),
               (7, 24, 20, 90, 77), (3, 2, 2, 1, 1), (5, 2, 9, 1, 36)]


@pytest.mark.parametrize("N,h,w,Hc,Wc", UT_GEOMETRY)
def test_upsample_threshold_geometry(ops, cuda, N, h, w, Hc, Wc):
    """N = 1 and 100 at the production sizes (100 x 1024 x 257 threads run the grid-stride loop), thresholds 0.5 and 0.3."""
    _budget(8 if N * Hc * Wc > 1e7 else 2)
    g = torch.Generator(device=cuda).manual_seed(N + h + w)
    masks = torch.randn(N, h, w, device=cuda, generator=g) * 3
    for thr in (0.5, 0.3):
        out = _ut_launch(ops, masks, thr, Hc, Wc)
        _ut_check(masks, out, thr, Hc, Wc, f"N={N} {Hc}x{Wc} thr={thr}")


def test_upsample_threshold_crops(ops, cuda):
    """Every crop 4h - Hc, 4w - Wc from 0 to 31."""
    g = torch.Generator(device=cuda).manual_seed(3)
    masks = torch.randn(3, 9, 10, device=cuda, generator=g) * 3
    for cy in range(32):
        Hc, Wc = max(36 - cy, 1), max(40 - (31 - cy), 1)
        _ut_check(masks, _ut_launch(ops, masks, 0.5, Hc, Wc), 0.5, Hc, Wc, f"crop {cy}")


@pytest.mark.parametrize("delta", [-1, 1])
def test_upsample_threshold_grid_cap(ops, cuda, delta):
    """A total of work items just under and just over the grid cap num_sms * 32 * 256 (Wc <= 2: one item per output row)."""
    cap = torch.cuda.get_device_properties(0).multi_processor_count * 32 * 256
    Hc = cap + delta
    h = (Hc + 3) // 4
    g = torch.Generator(device=cuda).manual_seed(delta + 2)
    masks = torch.randn(1, h, 2, device=cuda, generator=g) * 3
    out = _ut_launch(ops, masks, 0.5, Hc, 2)
    _ut_check(masks, out, 0.5, Hc, 2, f"total {Hc} vs cap {cap}")


# ------------------------------------------------------------------------------------------ the panoptic merge end to end
def _shell(thr=0.25):
    from hipie_b200.modeling.hipie_img import HIPIE_IMG
    m = types.SimpleNamespace(object_mask_threshold=thr, overlap_threshold=0.8, mask_stride=4)
    for f in ("fused_sem_pano_launch", "fused_sem_pano_finish", "semantic_inference", "panoptic_inference"):
        setattr(m, f, types.MethodType(getattr(HIPIE_IMG, f), m))
    return m


def _merge(m, mask_cls, mask_low, Hc, Wc, is_thing):
    pend = m.fused_sem_pano_launch(mask_cls, mask_low, (Hc, Wc))
    sem, (seg, info) = m.fused_sem_pano_finish(pend, pend["host_d"].cpu(), is_thing)
    h, w = mask_low.shape[1:]
    up = F.interpolate(mask_low[:, None], size=(4 * h, 4 * w), mode="bilinear", align_corners=False)[:, 0, :Hc, :Wc]
    rseg, rinfo = m.panoptic_inference(mask_cls, up, is_thing)
    return pend, seg, info, rseg, rinfo


@pytest.mark.parametrize("C", [80, 133, 150])
def test_merge_matches_reference(ops, cuda, C):
    """fused_sem_pano_launch + _finish against panoptic_inference on the same (mask_cls, mask_low), Q = 1200, 1024 x 1024:
    identical segments_info, panoptic_seg equal outside the band.  Each query is a blob of positive logits over noise, so that
    some segments survive the overlap test and some do not."""
    _budget(25)
    Q, h, w, Hc, Wc = 1200, 256, 256, 1024, 1024
    g = torch.Generator(device=cuda).manual_seed(C)
    yy, xx = torch.meshgrid(torch.arange(h, device=cuda), torch.arange(w, device=cuda), indexing="ij")
    cy, cx = torch.rand(Q, 1, 1, device=cuda, generator=g) * h, torch.rand(Q, 1, 1, device=cuda, generator=g) * w
    rad = 4 + torch.rand(Q, 1, 1, device=cuda, generator=g) * 20
    blob = ((yy - cy) ** 2 + (xx - cx) ** 2 < rad ** 2).float()
    mask_low = torch.randn(Q, h, w, device=cuda, generator=g) * 1.5 - 6 + 12 * blob
    mask_cls = torch.softmax(torch.randn(Q, C, device=cuda, generator=g) * 3, -1)
    is_thing = {c + 1: c % 3 != 0 for c in range(C)}
    m = _shell()
    pend, seg, info, rseg, rinfo = _merge(m, mask_cls, mask_low, Hc, Wc, is_thing)
    assert info == rinfo
    assert len(info) > 10, len(info)
    ref = restate(mask_low, mask_cls, 0.25, Hc, Wc)
    bad = (seg != rseg) & ~ref["band"]
    assert not bool(bad.any()), int(bad.sum())
    print(f"[merge C={C}] {len(info)} segments, band pixels {int(ref['band'].sum())}, differing {int((seg != rseg).sum())}")


@pytest.mark.parametrize("extra,kept", [(False, True), (True, False)])
def test_merge_overlap_ratio(ops, cuda, extra, kept):
    """Step-shaped logits whose sign is unambiguous after the upsample: query 1 is inside the mask on all 40 columns, query 0
    (higher score) owns the first 8 (9 with `extra`), so mask_area / original_area of query 1 is exactly 32 / 40 = 0.8 (kept)
    or 31 / 40 (dropped)."""
    w, Wc = 10, 40
    mask_low = torch.full((2, 2, w), -8.0, device=cuda)
    mask_low[0, :, :2] = 8.0
    if extra:
        mask_low[0, :, 2] = -2.0                  # pixel 8: 0.375 * 8 + 0.625 * -2 > 0, q 0 wins; pixel 9 does not
    mask_low[1] = 8.0
    mask_cls = torch.tensor([[0.9, 0.05, 0.05], [0.1, 0.5, 0.4]], device=cuda)
    is_thing = {1: True, 2: True, 3: True}
    pend, seg, info, rseg, rinfo = _merge(_shell(), mask_cls, mask_low, 1, Wc, is_thing)
    areas = pend["host_d"][:3].cpu()
    assert areas[:, 1].tolist() == [31 if extra else 32, 40, 31 if extra else 32], areas.tolist()
    assert info == rinfo and torch.equal(seg, rseg)
    assert [s["category_id"] for s in info] == ([0, 1] if kept else [0])


# ------------------------------------------------------------------------------------------ census
TESTED_C = {1, 8, 80, 81, 136, 137, 150, 847}


def _census_c1_forward():
    """One c1 forward (ViT-H, 1024 x 1024, 80 classes, synthetic weights) with ops.seg_postprocess and ops.upsample_threshold
    wrapped -> [(name, Q, C, h, w, Hc, Wc)]."""
    from hipie_oracle import hparams, synth
    from hipie_oracle.model import HipieOracle
    from hipie_b200 import ops
    from hipie_b200.modeling.hipie_img import HIPIE_IMG
    calls = []
    seg, ut = ops.seg_postprocess, ops.upsample_threshold

    def seg_w(masks_low, cls_prob, threshold, Hc, Wc, stride=4):
        calls.append(("seg_postprocess", *masks_low.shape[:1], cls_prob.shape[1], *masks_low.shape[1:], Hc, Wc))
        return seg(masks_low, cls_prob, threshold, Hc, Wc, stride)

    def ut_w(masks_low, threshold, Hc, Wc, stride=4):
        calls.append(("upsample_threshold", masks_low.shape[0], 0, *masks_low.shape[1:], Hc, Wc))
        return ut(masks_low, threshold, Hc, Wc, stride)

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
    ops.seg_postprocess, ops.upsample_threshold = seg_w, ut_w
    try:
        with torch.no_grad():
            model(inputs)
    finally:
        ops.seg_postprocess, ops.upsample_threshold = seg, ut
    torch.cuda.synchronize()
    return calls


def _in_child(mode):
    """Run one of this file's __main__ modes in a fresh Python process on the same device -> its JSON result (a whole-model
    forward stays out of the test process, see test_detection_heads_gpu.py)."""
    import os
    import subprocess
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    env = dict(os.environ, PYTHONDONTWRITEBYTECODE="1", PYTHONPATH=os.pathsep.join([root, os.path.join(root, "oracle"), here]))
    torch.cuda.empty_cache()
    r = subprocess.run([sys.executable, "-s", os.path.abspath(__file__), mode], cwd=root, env=env, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_census_c1_forward(cuda):
    """Every seg_postprocess / upsample_threshold call of one c1 forward falls inside what this file tests: a tested class count,
    Q within the tested range of its accumulator tile, an image no larger than the tested production sizes, N <= 100."""
    _budget(90)
    rec = _in_child("--census")
    calls = [tuple(c) for c in rec["calls"]]
    print(f"\n[census] c1 forward on {rec['device']}: {calls}")
    assert any(c[0] == "seg_postprocess" for c in calls) and any(c[0] == "upsample_threshold" for c in calls), calls
    qmax = {10: 1200, 17: 8192}
    for name, Q, C, h, w, Hc, Wc in calls:
        assert 4 * h - 32 < Hc <= 4 * h and 4 * w - 32 < Wc <= 4 * w and Hc <= 1024 and Wc <= 1024, (name, h, w, Hc, Wc)
        if name == "seg_postprocess":
            assert C in TESTED_C and Q <= (8192 if C > 136 else qmax[10 if C <= 80 else 17]), (Q, C)
        else:
            assert Q <= 100, Q


if __name__ == "__main__" and sys.argv[1:] == ["--census"]:
    print(json.dumps(dict(device=torch.cuda.get_device_name(0), calls=[list(c) for c in _census_c1_forward()])))
