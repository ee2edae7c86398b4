"""COCO instance evaluation on the host, without torch: GT annotation decoding (pycocotools maskApi.c / COCO.annToRLE) and the matching
and averaging of pycocotools' COCOeval (evaluateImg, accumulate, summarize) with detectron2's _derive_coco_results.  The pixel work
(every prediction x GT mask intersection) runs on the device (ops.mask_pack / rle_expand / mask_overlaps); this module takes the
resulting integer tables.  Quirks are kept, see DESIGN.md "Evaluation".

    rle_from_string, polygon_runs, merge_runs, ann_to_runs   one column-major run list per GT (counts, background first)
    bbox_iou, mask_iou                                       maskApi.c bbIou / rleIou from boxes or from intersection counts
    evaluate_image                                           COCOeval.evaluateImg for one (image, category, area range)
    image_records                                            every (category, area range) record of one image and task
    accumulate, summarize, derive_results                    COCOeval.accumulate / summarize and _derive_coco_results
"""
import math

import numpy as np

# Params.setDetParams (pycocotools cocoeval.py), built exactly as there
IOU_THRS = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
REC_THRS = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
MAX_DETS = [1, 10, 100]
AREA_RNG = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
AREA_LBL = ["all", "small", "medium", "large"]
METRICS = ["AP", "AP50", "AP75", "APs", "APm", "APl"]

# ---------------------------------------------------------------------------------------------------------------------------------
# GT masks as run lists


def rle_from_string(s, h=None, w=None):
    """maskApi.c rleFrString: the compressed COCO RLE string -> counts (uint32).  Each character - 48 carries 5 bits, 0x20 continues
    the value, 0x10 in its last character is the sign; from the fourth count on the value is a delta to the count two before."""
    if isinstance(s, str):
        s = s.encode("ascii")
    cnts = []
    p = 0
    while p < len(s):
        x, k, more = 0, 0, True
        while more:
            c = s[p] - 48
            x |= (c & 0x1f) << (5 * k)
            more = bool(c & 0x20)
            p += 1
            k += 1
            if not more and (c & 0x10):
                x |= -1 << (5 * k)
        if len(cnts) > 2:
            x += cnts[-2]
        cnts.append(x & 0xffffffff)                            # (uint) x
    return np.asarray(cnts, dtype=np.uint32)


def polygon_runs(xy, h, w):
    """maskApi.c rleFrPoly: one polygon [x0, y0, x1, y1, ...] -> counts.  The vertices are scaled x5 and rounded, the boundary is
    walked densely, the points where it crosses a pixel column are downsampled and the sorted column-major positions become runs."""
    xy = np.asarray(xy, dtype=np.float64)
    k = len(xy) // 2
    scale = 5.0
    x = [int(scale * xy[2 * j] + .5) for j in range(k)]       # C casts truncate toward zero
    y = [int(scale * xy[2 * j + 1] + .5) for j in range(k)]
    x.append(x[0])
    y.append(y[0])
    u, v = [], []
    for j in range(k):
        xs, xe, ys, ye = x[j], x[j + 1], y[j], y[j + 1]
        dx, dy = abs(xe - xs), abs(ys - ye)
        flip = (dx >= dy and xs > xe) or (dx < dy and ys > ye)
        if flip:
            xs, xe, ys, ye = xe, xs, ye, ys
        if dx == 0 and dy == 0:                                 # a repeated vertex: s = 0 / 0, and (int) NaN is INT_MIN on x86-64
            u.append(xs)
            v.append(-(1 << 31))
        elif dx >= dy:
            s = (ye - ys) / dx
            for d in range(dx + 1):
                t = dx - d if flip else d
                u.append(t + xs)
                v.append(int(ys + s * t + .5))
        else:
            s = (xe - xs) / dy
            for d in range(dy + 1):
                t = dy - d if flip else d
                v.append(t + ys)
                u.append(int(xs + s * t + .5))
    bx, by = [], []
    for j in range(1, len(u)):
        if u[j] == u[j - 1]:
            continue
        xd = float(u[j] if u[j] < u[j - 1] else u[j] - 1)
        xd = (xd + .5) / scale - .5
        if math.floor(xd) != xd or xd < 0 or xd > w - 1:
            continue
        yd = float(v[j] if v[j] < v[j - 1] else v[j - 1])
        yd = (yd + .5) / scale - .5
        yd = 0.0 if yd < 0 else (float(h) if yd > h else yd)
        bx.append(int(xd))
        by.append(int(math.ceil(yd)))
    a = sorted([(bx[j] * h + by[j]) & 0xffffffff for j in range(len(bx))] + [h * w])
    prev = 0
    for j in range(len(a)):
        a[j], prev = a[j] - prev, a[j]
    b = [a[0]]
    j = 1
    while j < len(a):
        if a[j] > 0:
            b.append(a[j])
            j += 1
        else:
            j += 1
            if j < len(a):
                b[-1] += a[j]
                j += 1
    return np.asarray(b, dtype=np.uint32)


def _fg_intervals(counts):
    c = np.asarray(counts, dtype=np.int64)
    e = np.cumsum(c)
    s = e - c
    return s[1::2], e[1::2]


def merge_runs(runs, n):
    """maskApi.c rleMerge with intersect = 0: the union of run lists over n pixels, as counts."""
    starts, ends = [], []
    for r in runs:
        s, e = _fg_intervals(r)
        keep = e > s
        starts.append(s[keep])
        ends.append(e[keep])
    s, e = np.concatenate(starts) if starts else np.zeros(0, np.int64), np.concatenate(ends) if ends else np.zeros(0, np.int64)
    order = np.argsort(s, kind="stable")
    s, e = s[order], e[order]
    out, pos = [], 0
    i = 0
    while i < len(s):
        a, b = s[i], e[i]
        i += 1
        while i < len(s) and s[i] <= b:
            b = max(b, e[i])
            i += 1
        out += [a - pos, b - a]
        pos = b
    out.append(n - pos)
    return np.asarray(out, dtype=np.uint32)


def runs_area(counts):
    """maskApi.c rleArea: the foreground pixels of a run list."""
    return int(np.asarray(counts, dtype=np.int64)[1::2].sum())


def ann_to_runs(ann, h, w):
    """COCO.annToRLE of one annotation on an h x w image -> counts: polygons (frPyObjects: a first entry of 4 numbers makes the list
    boxes) merged into one mask, uncompressed `counts` lists as they are, compressed strings through rle_from_string.  An RLE whose
    `size` is not (h, w) raises."""
    segm = ann["segmentation"]
    if isinstance(segm, list):
        if not segm:
            raise ValueError(f"annotation {ann.get('id')}: empty polygon list")
        if len(segm[0]) == 4:                                   # frBbox: [x, y, w, h] -> its four corners
            segm = [[b[0], b[1], b[0], b[1] + b[3], b[0] + b[2], b[1] + b[3], b[0] + b[2], b[1]] for b in segm]
        return merge_runs([polygon_runs(p, h, w) for p in segm], h * w)
    if tuple(segm["size"]) != (h, w):
        raise ValueError(f"annotation {ann.get('id')}: RLE of size {tuple(segm['size'])} on a {h} x {w} image")
    if isinstance(segm["counts"], list):
        return np.asarray(segm["counts"], dtype=np.int64)
    return rle_from_string(segm["counts"], h, w)


# ---------------------------------------------------------------------------------------------------------------------------------
# IoUs


def bbox_iou(dt, gt, iscrowd):
    """maskApi.c bbIou in float64: dt (D, 4), gt (G, 4) XYWH -> (D, G); a crowd GT's union is the detection's area."""
    d = np.asarray(dt, dtype=np.float64).reshape(-1, 4)[:, None, :]
    g = np.asarray(gt, dtype=np.float64).reshape(-1, 4)[None, :, :]
    crowd = np.asarray(iscrowd, dtype=bool).reshape(1, -1)
    w = np.minimum(d[..., 2] + d[..., 0], g[..., 2] + g[..., 0]) - np.maximum(d[..., 0], g[..., 0])
    h = np.minimum(d[..., 3] + d[..., 1], g[..., 3] + g[..., 1]) - np.maximum(d[..., 1], g[..., 1])
    i = w * h
    da, ga = d[..., 2] * d[..., 3], g[..., 2] * g[..., 3]
    u = np.where(crowd, da, da + ga - i)
    with np.errstate(divide="ignore", invalid="ignore"):
        o = i / u
    return np.where((w > 0) & (h > 0), o, 0.0)


def mask_iou(inter, dt_area, gt_area, iscrowd):
    """maskApi.c rleIou from the integer intersections inter (D, G) and areas: i / (da + ga - i), i / da for a crowd GT, 0 where i = 0."""
    inter = np.asarray(inter, dtype=np.int64)
    da = np.asarray(dt_area, dtype=np.int64)[:, None]
    ga = np.asarray(gt_area, dtype=np.int64)[None, :]
    u = np.where(np.asarray(iscrowd, dtype=bool)[None, :], da, da + ga - inter)
    u = np.where(inter == 0, 1, u)
    return inter.astype(np.float64) / u.astype(np.float64)


# ---------------------------------------------------------------------------------------------------------------------------------
# COCOeval


def evaluate_image(ious, gt_ids, gt_crowd, gt_area, dt_scores, dt_area, a_rng, max_det=MAX_DETS[-1]):
    """COCOeval.evaluateImg for one (image, category, area range).  GTs in annotation order, detections in prediction order; ious (D,
    G) over the same orders (rows = detections).  Returns None when there is neither, else (scores, matched (T, D) bool, ignored (T, D)
    bool, npig): detections sorted by -score (mergesort) and cut at max_det, matched = matched to a GT with a non-zero id (dtMatches
    stores the GT id), npig = GTs not ignored."""
    G, D = len(gt_ids), len(dt_scores)
    if G == 0 and D == 0:
        return None
    gt_area = np.asarray(gt_area, dtype=np.float64)
    ignore = np.array([1 if (c or gt_area[j] < a_rng[0] or gt_area[j] > a_rng[1]) else 0 for j, c in enumerate(gt_crowd)], dtype=np.int64)
    gtind = np.argsort(ignore, kind="mergesort")
    dtind = np.argsort([-s for s in dt_scores], kind="mergesort")[:max_det]
    gt_ig = ignore[gtind]
    crowd = [int(gt_crowd[j]) for j in gtind]
    ids = [gt_ids[j] for j in gtind]
    scores = np.asarray([dt_scores[i] for i in dtind], dtype=np.float64)
    T, Dk = len(IOU_THRS), len(dtind)
    dtm = np.zeros((T, Dk))
    dt_ig = np.zeros((T, Dk))
    if D and G:
        iou_m = np.asarray(ious, dtype=np.float64)[dtind][:, gtind]
        gtm = np.zeros((T, G))
        for tind, t in enumerate(IOU_THRS):
            for dind in range(Dk):
                iou = min([t, 1 - 1e-10])
                m = -1
                for gind in range(G):
                    if gtm[tind, gind] > 0 and not crowd[gind]:
                        continue
                    if m > -1 and gt_ig[m] == 0 and gt_ig[gind] == 1:
                        break
                    if iou_m[dind, gind] < iou:
                        continue
                    iou = iou_m[dind, gind]
                    m = gind
                if m == -1:
                    continue
                dt_ig[tind, dind] = gt_ig[m]
                dtm[tind, dind] = ids[m]
                gtm[tind, m] = 1 + dind                        # a detection id (1-based, never 0)
    da = np.asarray(dt_area, dtype=np.float64)[dtind]
    out = np.array([a < a_rng[0] or a > a_rng[1] for a in da]).reshape((1, Dk))
    dt_ig = np.logical_or(dt_ig, np.logical_and(dtm == 0, np.repeat(out, T, 0)))
    return scores, dtm != 0, dt_ig, int(np.count_nonzero(gt_ig == 0))


def image_records(cat_ids, gts, dts, ious):
    """Every record of one image and task: {(k, a): evaluate_image(...)} for k over the indices of cat_ids (the instance JSON's sorted
    category ids) and the four area ranges, None entries left out.  gts: list of dicts (id, category_id, iscrowd, area) in annotation
    order; dts: list of dicts (category_id, score, area) in prediction order; ious (len(dts), len(gts)) over all pairs (pairs of
    different categories are never read).  Detections of one category are cut at the best 100, as COCOeval.computeIoU does."""
    ious = np.asarray(ious, dtype=np.float64).reshape(len(dts), len(gts))
    out = {}
    for k, c in enumerate(cat_ids):
        gi = [j for j, g in enumerate(gts) if g["category_id"] == c]
        di = [i for i, d in enumerate(dts) if d["category_id"] == c]
        if not gi and not di:
            continue
        order = np.argsort([-dts[i]["score"] for i in di], kind="mergesort")[:MAX_DETS[-1]]
        di = [di[i] for i in order]
        sub = ious[np.ix_(di, gi)] if di and gi else np.zeros((len(di), len(gi)))
        for a, rng in enumerate(AREA_RNG):
            out[(k, a)] = evaluate_image(sub, [gts[j]["id"] for j in gi], [gts[j].get("iscrowd", 0) for j in gi], [gts[j]["area"] for j in gi],
                                         [dts[i]["score"] for i in di], [dts[i]["area"] for i in di], rng)
    return out


def accumulate(per_image, K):
    """COCOeval.accumulate over the records of every image: per_image is a list of (image_id, image_records(...)); images are
    concatenated in ascending image-id order before the mergesort, as COCOeval indexes evalImgs by the sorted imgIds.  -> (precision
    (T, R, K, A, M), recall (T, K, A, M), scores (T, R, K, A, M)), -1 where a category has no GT."""
    T, R, A, M = len(IOU_THRS), len(REC_THRS), len(AREA_RNG), len(MAX_DETS)
    precision = -np.ones((T, R, K, A, M))
    recall = -np.ones((T, K, A, M))
    scores = -np.ones((T, R, K, A, M))
    per_image = sorted(per_image, key=lambda x: x[0])
    for k in range(K):
        for a in range(A):
            E = [rec[(k, a)] for _, rec in per_image if rec.get((k, a)) is not None]
            if not E:
                continue
            for m, max_det in enumerate(MAX_DETS):
                dt_scores = np.concatenate([e[0][0:max_det] for e in E])
                inds = np.argsort(-dt_scores, kind="mergesort")
                dt_scores_sorted = dt_scores[inds]
                dtm = np.concatenate([e[1][:, 0:max_det] for e in E], axis=1)[:, inds]
                dt_ig = np.concatenate([e[2][:, 0:max_det] for e in E], axis=1)[:, inds]
                npig = sum(e[3] for e in E)
                if npig == 0:
                    continue
                tps = np.logical_and(dtm, np.logical_not(dt_ig))
                fps = np.logical_and(np.logical_not(dtm), np.logical_not(dt_ig))
                tp_sum = np.cumsum(tps, axis=1).astype(dtype=float)
                fp_sum = np.cumsum(fps, axis=1).astype(dtype=float)
                for t, (tp, fp) in enumerate(zip(tp_sum, fp_sum)):
                    nd = len(tp)
                    rc = tp / npig
                    pr = tp / (fp + tp + np.spacing(1))
                    recall[t, k, a, m] = rc[-1] if nd else 0
                    pr = pr.tolist()
                    for i in range(nd - 1, 0, -1):
                        if pr[i] > pr[i - 1]:
                            pr[i - 1] = pr[i]
                    idx = np.searchsorted(rc, REC_THRS, side="left")
                    q, ss = np.zeros((R,)), np.zeros((R,))
                    valid = idx < nd                           # the reference's loop stops at the first index past the end
                    n_ok = int(np.argmin(valid)) if not valid.all() else R
                    if n_ok:
                        q[:n_ok] = np.asarray(pr)[idx[:n_ok]]
                        ss[:n_ok] = dt_scores_sorted[idx[:n_ok]]
                    precision[t, :, k, a, m] = q
                    scores[t, :, k, a, m] = ss
    return precision, recall, scores


def summarize(precision, recall):
    """COCOeval.summarize (_summarizeDets) -> the 12 stats; -1 where nothing counts."""
    def _summarize(ap=1, iou_thr=None, area_rng="all", max_dets=100):
        aind = [i for i, r in enumerate(AREA_LBL) if r == area_rng]
        mind = [i for i, m in enumerate(MAX_DETS) if m == max_dets]
        s = precision if ap == 1 else recall
        if iou_thr is not None:
            s = s[np.where(iou_thr == IOU_THRS)[0]]
        s = s[:, :, :, aind, mind] if ap == 1 else s[:, :, aind, mind]
        return -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
    stats = np.zeros((12,))
    stats[0] = _summarize(1)
    stats[1] = _summarize(1, iou_thr=.5, max_dets=MAX_DETS[2])
    stats[2] = _summarize(1, iou_thr=.75, max_dets=MAX_DETS[2])
    stats[3] = _summarize(1, area_rng="small", max_dets=MAX_DETS[2])
    stats[4] = _summarize(1, area_rng="medium", max_dets=MAX_DETS[2])
    stats[5] = _summarize(1, area_rng="large", max_dets=MAX_DETS[2])
    stats[6] = _summarize(0, max_dets=MAX_DETS[0])
    stats[7] = _summarize(0, max_dets=MAX_DETS[1])
    stats[8] = _summarize(0, max_dets=MAX_DETS[2])
    stats[9] = _summarize(0, area_rng="small", max_dets=MAX_DETS[2])
    stats[10] = _summarize(0, area_rng="medium", max_dets=MAX_DETS[2])
    stats[11] = _summarize(0, area_rng="large", max_dets=MAX_DETS[2])
    return stats


def derive_results(stats, precision, class_names):
    """detectron2 COCOEvaluator._derive_coco_results: AP, AP50, AP75, APs, APm, APl x 100 (NaN for -1), then AP-<name> per category
    from precision[:, :, k, area all, maxDets 100] when there are at least two names.  stats None (no predictions at all) -> every metric
    NaN.  The names index the categories by position, as the reference does."""
    if stats is None:
        return {m: float("nan") for m in METRICS}
    res = {m: float(stats[i] * 100 if stats[i] >= 0 else "nan") for i, m in enumerate(METRICS)}
    if class_names is None or len(class_names) <= 1:
        return res
    if len(class_names) != precision.shape[2]:
        raise ValueError(f"derive_results: {len(class_names)} class names for {precision.shape[2]} categories")
    for k, name in enumerate(class_names):
        p = precision[:, :, k, 0, -1]
        p = p[p > -1]
        ap = np.mean(p) if p.size else float("nan")
        res["AP-" + str(name)] = float(ap * 100)
    return res


def evaluate_records(per_image, cat_ids, class_names, any_predictions):
    """accumulate + summarize + derive_results of one task."""
    if not any_predictions:
        return derive_results(None, None, class_names)
    precision, recall, _ = accumulate(per_image, len(cat_ids))
    return derive_results(summarize(precision, recall), precision, class_names)
