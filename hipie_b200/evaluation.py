"""Semantic and panoptic evaluation on the device: the reference's `train_net.py --eval-only` path for the segmentation benchmarks of
its README (ADE-150 PQ / mIoU, COCO PQ / mIoU, ADE-847, PAS-21, CTX-59, CTX-459 mIoU).

The reference runs detectron2's SemSegEvaluator (detectron2/evaluation/sem_seg_evaluation.py) and COCOPanopticEvaluator
(detectron2/evaluation/panoptic_evaluation.py + panopticapi) on the host: an argmax map copied to the host and np.bincount per image, a
PNG encoded per image, written to disk at evaluate() and decoded again for np.unique.  Here the per-pixel reductions are
ops.semseg_confusion / ops.panoptic_pairs on the model's outputs; the confusion matrix stays on the device until evaluate(), and each
image's pair table (a few KB) is copied asynchronously into pinned memory and matched on the host one or more images later.  The metrics
are computed from those counters exactly as the reference computes them, quirks included (DESIGN.md, "Evaluation").

    SemSegEvaluator / COCOPanopticEvaluator   reset() / process(inputs, outputs) / evaluate(), the reference's DatasetEvaluator surface
    COCOInstanceEvaluator                     AP_bbox / AP_segm (COCOEvaluator / InstanceSegEvaluator): mask overlaps on the device,
                                              COCOeval's matching on the host (cocoeval.py)
    PRESETS, load_records                     readers for the reference's dataset layouts under a data root
    preset_vocabulary                         the test mapper's vocabulary of a preset (coco_dataset_mapper_uni.py:196-215, 556-566)
    evaluate_dataset                          the eval-only driver; `python -m hipie_b200.evaluation` is its command line
"""
import argparse
import collections
import json
import os
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch
import torch.distributed as dist

from . import cocoeval, ops
from .data import ResizeShortestEdge, create_queries_and_maps, get_openseg_labels
from .hostio import PinnedArena
from .parallel import shard_indices
from .predictor import cat2ind

VOID = 0

# ---------------------------------------------------------------------------------------------------------------------------------
# metrics from the counters (host, float64)


def semseg_metrics(conf, class_names):
    """SemSegEvaluator.evaluate (sem_seg_evaluation.py:133-160) on a (C + 1, C + 1) int64 confusion matrix (rows = predictions, columns =
    GT, last row / column = ignore).  Its quirks are kept: the mIoU numerator sums the IoU of classes with GT pixels, its denominator
    counts classes with GT or predicted pixels; classes without GT pixels get NaN IoU and ACC; every value is x 100."""
    conf = np.asarray(conf, dtype=np.int64)
    C = conf.shape[0] - 1
    if len(class_names) != C:
        raise ValueError(f"semseg_metrics: {len(class_names)} class names for a {C}-class matrix")
    acc = np.full(C, np.nan, dtype=np.float64)
    iou = np.full(C, np.nan, dtype=np.float64)
    tp = conf.diagonal()[:-1].astype(np.float64)
    pos_gt = np.sum(conf[:-1, :-1], axis=0).astype(np.float64)
    class_weights = pos_gt / np.sum(pos_gt)
    pos_pred = np.sum(conf[:-1, :-1], axis=1).astype(np.float64)
    acc_valid = pos_gt > 0
    acc[acc_valid] = tp[acc_valid] / pos_gt[acc_valid]
    iou_valid = (pos_gt + pos_pred) > 0
    union = pos_gt + pos_pred - tp
    iou[acc_valid] = tp[acc_valid] / union[acc_valid]
    macc = np.sum(acc[acc_valid]) / np.sum(acc_valid)
    miou = np.sum(iou[acc_valid]) / np.sum(iou_valid)
    fiou = np.sum(iou[acc_valid] * class_weights[acc_valid])
    pacc = np.sum(tp) / np.sum(pos_gt)
    res = {"mIoU": 100 * miou, "fwIoU": 100 * fiou}
    for i, name in enumerate(class_names):
        res[f"IoU-{name}"] = 100 * iou[i]
    res["mACC"] = 100 * macc
    res["pACC"] = 100 * pacc
    for i, name in enumerate(class_names):
        res[f"ACC-{name}"] = 100 * acc[i]
    return res


class PQStat:
    """panopticapi's PQStat as arrays over the dataset's category ids: int64 tp / fp / fn and float64 IoU sums (the accumulators that
    are summed over ranks)."""

    def __init__(self, category_ids):
        self.ids = list(category_ids)
        self.index = {c: i for i, c in enumerate(self.ids)}
        n = len(self.ids)
        self.counts = np.zeros((n, 3), dtype=np.int64)       # tp, fp, fn
        self.iou = np.zeros(n, dtype=np.float64)

    def add_image(self, table, gt_ids, gt_segments, pred_segments, image_id=None):
        """pq_compute_single_core on one image's pair table.  table (n_gt + 2, S + 1): rows VOID, gt_ids (ascending), unlisted; columns
        pred ids 0..S.  gt_segments: {id: segment_info of the GT JSON (category_id, iscrowd, area)} in segments_info order;
        pred_segments: {id: dataset category id} of the listed predicted segments."""
        table = np.asarray(table, dtype=np.int64)
        S = table.shape[1] - 1
        pred_area = table.sum(0)
        for p in range(1, S + 1):
            if pred_area[p] and p not in pred_segments:
                raise KeyError(f"In the image with ID {image_id} segment with ID {p} is presented in PNG and not presented in JSON.")
        for p, cat in pred_segments.items():
            if not (1 <= p <= S) or pred_area[p] == 0:
                raise KeyError(f"In the image with ID {image_id} the following segment IDs {[p]} are presented in JSON and not presented "
                               "in PNG.")
            if cat not in self.index:
                raise KeyError(f"In the image with ID {image_id} segment with ID {p} has unknown category_id {cat}.")
        row_of = {g: r + 1 for r, g in enumerate(gt_ids)}
        gt_matched, pred_matched = set(), set()
        for r, g in enumerate(gt_ids, 1):                   # np.unique order of gt * 2^24 + pred: ascending GT id, then pred id
            info = gt_segments[g]
            for p in np.nonzero(table[r])[0].tolist():
                if p not in pred_segments or info.get("iscrowd", 0) == 1 or info["category_id"] != pred_segments[p]:
                    continue
                inter = table[r, p]
                union = pred_area[p] + info["area"] - inter - table[VOID, p]
                iou = inter / union
                if iou > 0.5:
                    c = self.index[info["category_id"]]
                    self.counts[c, 0] += 1
                    self.iou[c] += iou
                    gt_matched.add(g)
                    pred_matched.add(p)
        crowd = {}
        for g, info in gt_segments.items():
            if g in gt_matched:
                continue
            if info.get("iscrowd", 0) == 1:
                crowd[info["category_id"]] = g          # the last crowd segment of a category in segments_info order
                continue
            self.counts[self.index[info["category_id"]], 2] += 1
        for p, cat in pred_segments.items():
            if p in pred_matched:
                continue
            inter = table[VOID, p]
            if cat in crowd:
                inter += table[row_of[crowd[cat]], p]
            if inter / pred_area[p] > 0.5:
                continue
            self.counts[self.index[cat], 1] += 1

    def average(self, categories, isthing):
        """pq_average over the JSON's categories (a list of {id, isthing}): categories with tp + fp + fn == 0 do not count.  With no
        category counted the averages are NaN (panopticapi divides by zero)."""
        pq = sq = rq = 0.0
        n = 0
        per_class = {}
        for cat in categories:
            if isthing is not None and (cat.get("isthing", 0) == 1) != isthing:
                continue
            i = self.index[cat["id"]]
            tp, fp, fn = (int(v) for v in self.counts[i])
            iou = float(self.iou[i])
            if tp + fp + fn == 0:
                per_class[cat["id"]] = {"pq": 0.0, "sq": 0.0, "rq": 0.0}
                continue
            n += 1
            pq_c = iou / (tp + 0.5 * fp + 0.5 * fn)
            sq_c = iou / tp if tp != 0 else 0
            rq_c = tp / (tp + 0.5 * fp + 0.5 * fn)
            per_class[cat["id"]] = {"pq": pq_c, "sq": sq_c, "rq": rq_c}
            pq, sq, rq = pq + pq_c, sq + sq_c, rq + rq_c
        nan = float("nan")
        return {"pq": pq / n if n else nan, "sq": sq / n if n else nan, "rq": rq / n if n else nan, "n": n}, per_class

    def results(self, categories):
        """COCOPanopticEvaluator.evaluate's dict (x 100) and panopticapi's per-class results of "All"."""
        avg = {}
        for name, isthing in (("All", None), ("Things", True), ("Stuff", False)):
            avg[name], per_class = self.average(categories, isthing)
            if name == "All":
                avg["per_class"] = per_class
        res = {}
        for key, name in (("", "All"), ("_th", "Things"), ("_st", "Stuff")):
            for m in ("pq", "sq", "rq"):
                res[m.upper() + key] = 100 * avg[name][m]
        return res, avg["per_class"]


# ---------------------------------------------------------------------------------------------------------------------------------
# host <-> device staging


def _distributed():
    return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


def _all_reduce(t):
    """Sum a tensor over the ranks (NCCL needs it on the device, gloo on the host); returns it on its original device."""
    if not _distributed():
        return t
    dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else torch.device("cpu")
    x = t.to(dev)
    dist.all_reduce(x)
    return x.to(t.device)


class _Inflight:
    """Pinned staging areas of the images still in flight on the current stream.  `acquire` hands out an arena; `release` records an
    event after the arena's copies and kernels were queued, with a callback that consumes its host views once the event has passed.
    Finished images are consumed on later calls without waiting; only when `depth` images are in flight does acquire wait for the
    oldest."""

    def __init__(self, depth=4, nbytes=8 << 20):
        self.depth, self.nbytes = depth, nbytes
        self.free, self.busy = [], collections.deque()

    def _retire(self, block):
        while self.busy and (block or self.busy[0][1].query()):
            arena, ev, done = self.busy.popleft()
            ev.synchronize()
            if done is not None:
                done()
            self.free.append(arena)
            block = block and len(self.busy) >= self.depth

    def acquire(self):
        self._retire(block=len(self.busy) >= self.depth)
        arena = self.free.pop() if self.free else PinnedArena(self.nbytes)
        arena.reset()
        return arena

    def release(self, arena, done=None):
        ev = torch.cuda.Event()
        ev.record()
        self.busy.append((arena, ev, done))

    def drain(self):
        while self.busy:
            self._retire(block=True)


def load_image_into_numpy_array(filename, dtype=None):
    """sem_seg_evaluation.py:20-27: PIL decode (8-bit PNG, 16-bit TIFF) into a numpy array."""
    from PIL import Image
    with open(filename, "rb") as f:
        return np.array(Image.open(f), dtype=dtype)


def read_panoptic_png(filename):
    """The RGB-coded panoptic GT PNG as (H, W, 3) uint8 (panopticapi decodes it with np.array(Image.open(...), dtype=np.uint32))."""
    from PIL import Image
    with open(filename, "rb") as f:
        a = np.array(Image.open(f).convert("RGB"), dtype=np.uint8)
    return a


# ---------------------------------------------------------------------------------------------------------------------------------
# evaluators


class SemSegEvaluator:
    """detectron2's SemSegEvaluator with the confusion matrix on the device.  records: the dataset's records (file_name ->
    sem_seg_file_name); class_names: C names (the IoU-<name> / ACC-<name> keys); ignore_label: 255, or 65535 for the 16-bit TIFF GT.
    process() decodes the GT on the host, copies it through pinned memory and launches hipie_semseg_confusion; nothing crosses back
    to the host until evaluate().  GT labels outside 0..C-1 other than ignore_label are counted on the device and raise in evaluate()."""

    def __init__(self, records, class_names, ignore_label, distributed=True):
        self.input_file_to_gt_file = {r["file_name"]: r["sem_seg_file_name"] for r in records}
        self._class_names = list(class_names)
        self._num_classes = len(self._class_names)
        self._ignore_label = int(ignore_label)
        self._distributed = distributed
        self._stage = _Inflight()
        self.reset()

    def reset(self):
        self._conf = None
        self._err = None
        self._images = 0

    def process(self, inputs, outputs):
        for inp, out in zip(inputs, outputs):
            sem = out["sem_seg"]
            if self._conf is None:
                self._conf = torch.zeros((self._num_classes + 1,) * 2, dtype=torch.int64, device=sem.device)
                self._err = torch.zeros(1, dtype=torch.int64, device=sem.device)
            if sem.shape[0] != self._num_classes:
                raise ValueError(f"SemSegEvaluator: sem_seg has {sem.shape[0]} classes, the dataset {self._num_classes}")
            gt = load_image_into_numpy_array(self.input_file_to_gt_file[inp["file_name"]], dtype=np.int32)
            if gt.shape != tuple(sem.shape[1:]):
                raise ValueError(f"SemSegEvaluator: GT of {inp['file_name']} is {gt.shape}, sem_seg {tuple(sem.shape[1:])}")
            arena = self._stage.acquire()
            gt_d = arena.to_device(np.ascontiguousarray(gt), sem.device)
            ops.semseg_confusion(sem.float(), gt_d, self._ignore_label, self._conf, self._err)
            self._stage.release(arena)
            self._images += 1

    def evaluate(self):
        self._stage.drain()
        C = self._num_classes
        conf = self._conf if self._conf is not None else torch.zeros((C + 1, C + 1), dtype=torch.int64)
        err = self._err if self._err is not None else torch.zeros(1, dtype=torch.int64)
        if self._distributed and _distributed():
            conf, err = _all_reduce(conf), _all_reduce(err)
            if dist.get_rank() != 0:
                return None
        if int(err.item()):
            raise ValueError(f"SemSegEvaluator: {int(err.item())} GT pixels carry a label outside 0..{C - 1} that is not the ignore "
                             f"label {self._ignore_label}")
        return {"sem_seg": semseg_metrics(conf.cpu().numpy(), self._class_names)}


class COCOPanopticEvaluator:
    """detectron2's COCOPanopticEvaluator + panopticapi's pq_compute with the pixel work on the device.  panoptic_json /
    panoptic_root: the dataset's GT JSON and PNG folder.  The model's contiguous category ids map to dataset ids through
    thing_dataset_id_to_contiguous_id or stuff_dataset_id_to_contiguous_id according to each segment's `isthing`
    (panoptic_evaluation.py:118-130); by default both are built from the JSON's category list as the reference's registrations build
    them from theirs (things: id -> position among all categories; stuff: every category).

    process() reads the GT PNG, launches hipie_panoptic_pairs and copies the pair table into pinned memory; the table is matched on the
    host (PQStat.add_image) once its copy has landed, on a later process() call or in evaluate().  Only processed images count."""

    def __init__(self, panoptic_json, panoptic_root, thing_dataset_id_to_contiguous_id=None, stuff_dataset_id_to_contiguous_id=None,
                 distributed=True):
        with open(panoptic_json, "r") as f:
            js = json.load(f)
        self.categories = js["categories"]
        self.gt_annotations = {a["image_id"]: a for a in js["annotations"]}
        self.panoptic_root = panoptic_root
        things, stuff = panoptic_category_maps(self.categories)
        things = things if thing_dataset_id_to_contiguous_id is None else thing_dataset_id_to_contiguous_id
        stuff = stuff if stuff_dataset_id_to_contiguous_id is None else stuff_dataset_id_to_contiguous_id
        self._thing_contiguous_id_to_dataset_id = {v: k for k, v in things.items()}
        self._stuff_contiguous_id_to_dataset_id = {v: k for k, v in stuff.items()}
        self._distributed = distributed
        self._stage = _Inflight()
        self.reset()

    def reset(self):
        self.stat = PQStat([c["id"] for c in self.categories])
        self._images = 0

    def _convert_category_id(self, info):
        isthing = info.get("isthing", None)
        if isthing is None:
            return info["category_id"]
        table = self._thing_contiguous_id_to_dataset_id if isthing else self._stuff_contiguous_id_to_dataset_id
        return table[info["category_id"]]

    def process(self, inputs, outputs):
        for inp, out in zip(inputs, outputs):
            pan, segments_info = out["panoptic_seg"]
            if segments_info is None:
                raise NotImplementedError("COCOPanopticEvaluator: category * label_divisor panoptic maps (segments_info None) are not "
                                          "produced by this engine")
            ann = self.gt_annotations[inp["image_id"]]
            gt_segments = {s["id"]: s for s in ann["segments_info"]}
            gt_ids = sorted(gt_segments)
            if gt_ids and gt_ids[0] <= 0:
                raise ValueError(f"COCOPanopticEvaluator: image {inp['image_id']} lists GT segment id {gt_ids[0]} (ids are positive)")
            pred_segments = {int(s["id"]): self._convert_category_id(s) for s in segments_info}
            S = max(pred_segments, default=0)
            rgb = read_panoptic_png(os.path.join(self.panoptic_root, ann["file_name"]))
            if rgb.shape[:2] != tuple(pan.shape):
                raise ValueError(f"COCOPanopticEvaluator: GT of image {inp['image_id']} is {rgb.shape[:2]}, the prediction "
                                 f"{tuple(pan.shape)}")
            arena = self._stage.acquire()
            rgb_d = arena.to_device(rgb, pan.device)
            ids_d = arena.to_device(np.asarray(gt_ids, dtype=np.int32), pan.device)
            err = torch.zeros(1, dtype=torch.int64, device=pan.device)
            table = ops.panoptic_pairs(pan.to(torch.int32), rgb_d, ids_d, S, err=err)
            table_h, err_h = arena.to_host(table), arena.to_host(err)
            image_id = inp["image_id"]

            def done(table_h=table_h, err_h=err_h, gt_ids=gt_ids, gt_segments=gt_segments, pred_segments=pred_segments, S=S,
                     image_id=image_id):
                if int(err_h[0]):
                    raise KeyError(f"In the image with ID {image_id} {int(err_h[0])} pixels carry a segment ID outside 0..{S}.")
                self.stat.add_image(table_h.numpy(), gt_ids, gt_segments, pred_segments, image_id)

            self._stage.release(arena, done)
            self._images += 1

    def evaluate(self):
        self._stage.drain()
        counts, iou = torch.from_numpy(self.stat.counts), torch.from_numpy(self.stat.iou)
        if self._distributed and _distributed():
            counts, iou = _all_reduce(counts), _all_reduce(iou)
            if dist.get_rank() != 0:
                return None
            self.stat.counts, self.stat.iou = counts.numpy(), iou.numpy()
        res, per_class = self.stat.results(self.categories)
        return {"panoptic_seg": res, "panoptic_seg_per_class": per_class}


class COCOInstanceEvaluator:
    """detectron2's COCOEvaluator / InstanceSegEvaluator (bbox and segm) with the mask overlaps on the device.  instances_json: the
    dataset's COCO instance annotations; thing_dataset_id_to_contiguous_id maps the model's classes back to dataset ids (a class outside
    it raises, as the reference's assert does); class_names: the AP-<name> keys, one per instance category (the reference asserts that
    count in _derive_coco_results).

    process() packs the predicted masks (ops.mask_pack), expands the image's GT runs (ops.rle_expand), launches ops.mask_overlaps and
    copies the (N, M) intersection table, the mask areas, boxes, scores and classes into pinned memory.  Once the copy has landed (a
    later process() call or evaluate()) COCOeval.evaluateImg runs for both tasks and only its compact per-image records are kept.
    evaluate() gathers the records to rank 0 and accumulates them in image-id order.  Only processed images count."""

    TASKS = ("bbox", "segm")

    def __init__(self, instances_json, thing_dataset_id_to_contiguous_id, class_names, distributed=True):
        with open(instances_json, "r") as f:
            js = json.load(f)
        self.cat_ids = sorted(c["id"] for c in js["categories"])
        self.class_names = list(class_names)
        if len(self.class_names) != len(self.cat_ids):
            raise ValueError(f"COCOInstanceEvaluator: {len(self.class_names)} thing classes for the {len(self.cat_ids)} categories of "
                             f"{instances_json}")
        self.images = {im["id"]: im for im in js["images"]}
        self._by_stem = {os.path.splitext(os.path.basename(im["file_name"]))[0]: im["id"] for im in js["images"]}
        self.anns = collections.defaultdict(list)
        for a in js["annotations"]:
            self.anns[a["image_id"]].append(a)
        self._dataset_id = {v: k for k, v in thing_dataset_id_to_contiguous_id.items()}
        self._distributed = distributed
        self._stage = _Inflight()
        self.reset()

    def reset(self):
        self._records = []                 # (image id, {task: image_records})
        self._any_predictions = False

    def _image_id(self, inp):
        if inp["image_id"] in self.images:
            return inp["image_id"]
        stem = os.path.splitext(os.path.basename(inp.get("file_name", "")))[0]
        if stem in self._by_stem:
            return self._by_stem[stem]
        raise KeyError(f"COCOInstanceEvaluator: image {inp['image_id']} is not in the instance annotations")

    def process(self, inputs, outputs):
        for inp, out in zip(inputs, outputs):
            inst = out["instances"]
            img_id = self._image_id(inp)
            H, W = self.images[img_id]["height"], self.images[img_id]["width"]
            masks = inst.pred_masks
            if masks.dim() != 3 or tuple(masks.shape[1:]) != (H, W):
                raise ValueError(f"COCOInstanceEvaluator: masks of image {inp['image_id']} are {tuple(masks.shape)}, the image {H} x {W}")
            anns = self.anns.get(img_id, [])
            runs = [cocoeval.ann_to_runs(a, H, W) for a in anns]
            gts = [{"id": a["id"], "category_id": a["category_id"], "iscrowd": a.get("iscrowd", 0), "area": a["area"]} for a in anns]
            gt_pixels = [cocoeval.runs_area(r) for r in runs]
            gt_boxes = [a["bbox"] for a in anns]
            N, M = masks.shape[0], len(runs)
            dev = masks.device
            arena = self._stage.acquire()
            err = torch.zeros(1, dtype=torch.int64, device=dev)
            pbits, parea = ops.mask_pack(masks)
            if N and M:
                ends, offsets = ops.rle_ends(runs, H, W)
                gbits = ops.rle_expand(arena.to_device(ends, dev), arena.to_device(offsets, dev), H, W, err=err)
            else:
                gbits = torch.zeros((M, ops.mask_words(H, W)), dtype=torch.int32, device=dev)
            inter = ops.mask_overlaps(pbits, gbits, H, W)
            host = [arena.to_host(t) for t in (inter, parea, inst.pred_boxes.tensor.float(), inst.scores.float(),
                                               inst.pred_classes.to(torch.int64), err)]
            image_id = inp["image_id"]

            def done(host=host, gts=gts, gt_pixels=gt_pixels, gt_boxes=gt_boxes, img_id=img_id, image_id=image_id):
                inter_h, area_h, boxes_h, scores_h, classes_h, err_h = (t.numpy() for t in host)
                if int(err_h[0]):
                    raise ValueError(f"COCOInstanceEvaluator: GT run lists of image {image_id} do not cover the image")
                self._add_image(img_id, inter_h, area_h, boxes_h, scores_h, classes_h, gts, gt_pixels, gt_boxes)

            self._stage.release(arena, done)

    def _add_image(self, img_id, inter, area, boxes, scores, classes, gts, gt_pixels, gt_boxes):
        """instances_to_coco_json + COCOeval.evaluateImg of one image: XYXY -> XYWH in float32 (BoxMode.convert), then Python floats."""
        for c in classes.tolist():
            if c not in self._dataset_id:
                raise ValueError(f"A prediction has class={c}, but the dataset only has class ids in "
                                 f"{sorted(self._dataset_id)} (thing_dataset_id_to_contiguous_id).")
        xywh = boxes.astype(np.float32).copy()
        xywh[:, 2] -= xywh[:, 0]
        xywh[:, 3] -= xywh[:, 1]
        xywh = xywh.tolist()
        scores = scores.tolist()
        cats = [self._dataset_id[c] for c in classes.tolist()]
        crowd = [g["iscrowd"] for g in gts]
        recs = {}
        for task in self.TASKS:
            if task == "segm":
                dts = [{"category_id": c, "score": s, "area": int(a)} for c, s, a in zip(cats, scores, area.tolist())]
                ious = cocoeval.mask_iou(inter, area, gt_pixels, crowd)
            else:
                dts = [{"category_id": c, "score": s, "area": b[2] * b[3]} for c, s, b in zip(cats, scores, xywh)]
                ious = cocoeval.bbox_iou(xywh, gt_boxes, crowd)
            recs[task] = cocoeval.image_records(self.cat_ids, gts, dts, ious)
        self._records.append((img_id, recs))
        self._any_predictions = self._any_predictions or len(scores) > 0

    def evaluate(self):
        self._stage.drain()
        records, any_pred = self._records, self._any_predictions
        if self._distributed and _distributed():
            parts = [None] * dist.get_world_size() if dist.get_rank() == 0 else None
            dist.gather_object((records, any_pred), parts, dst=0)
            if dist.get_rank() != 0:
                return None
            records = [r for p in parts for r in p[0]]
            any_pred = any(p[1] for p in parts)
        res = collections.OrderedDict()
        for task in self.TASKS:
            res[task] = cocoeval.evaluate_records([(i, r[task]) for i, r in records], self.cat_ids, self.class_names, any_pred)
        return res


# ---------------------------------------------------------------------------------------------------------------------------------
# datasets


def panoptic_category_maps(categories):
    """(thing_dataset_id_to_contiguous_id, stuff_dataset_id_to_contiguous_id) of a panoptic category list, as
    register_ade20k_panoptic.get_metadata / register_coco_panoptic_annos_semseg.get_metadata build them: position i in the list is the
    contiguous id; things map only the isthing categories, stuff maps every category."""
    things = {c["id"]: i for i, c in enumerate(categories) if c.get("isthing", 0)}
    stuff = {c["id"]: i for i, c in enumerate(categories)}
    return things, stuff


# name -> layout under the data root (the reference's registrations: register_ade20k_panoptic.py, register_coco_panoptic_annos_semseg.py
# with detectron2's coco_2017_val image root, register_ade_20k_full.py, register_pascal.py)
PRESETS = {
    "ade20k_panoptic_val": dict(
        kind="panoptic", vocabulary="ade20k_150", ignore_label=255, image_root="ade/ADEChallengeData2016/images/validation",
        panoptic_root="ade/ADEChallengeData2016/ade20k_panoptic_val", panoptic_json="ade/ADEChallengeData2016/ade20k_panoptic_val.json",
        sem_seg_root="ade/ADEChallengeData2016/annotations_detectron2/validation",
        instances_json="ade/ADEChallengeData2016/ade20k_instance_val.json"),
    "coco_2017_val_panoptic_with_sem_seg": dict(
        kind="panoptic", vocabulary="coco_panoptic", ignore_label=255, image_root="coco/val2017", panoptic_root="coco/panoptic_val2017",
        panoptic_json="coco/annotations/panoptic_val2017.json", sem_seg_root="coco/panoptic_semseg_val2017",
        instances_json="coco/annotations/instances_val2017.json"),
    "ade20k_full_sem_seg_val": dict(
        kind="sem_seg", vocabulary="ade20k_847", ignore_label=65535, num_classes=847,
        image_root="ade/ADE20K_2021_17_01/images_detectron2/validation", sem_seg_root="ade/ADE20K_2021_17_01/annotations_detectron2/validation",
        image_ext="jpg", gt_ext="tif"),
    "ctx59_sem_seg_val": dict(
        kind="sem_seg", vocabulary="pascal_context_59", ignore_label=255, num_classes=59, image_root="pascal_ctx_d2/images/validation",
        sem_seg_root="pascal_ctx_d2/annotations_ctx59/validation", image_ext="jpg", gt_ext="png"),
    "ctx459_sem_seg_val": dict(
        kind="sem_seg", vocabulary="pascal_context_459", ignore_label=65535, num_classes=459, image_root="pascal_ctx_d2/images/validation",
        sem_seg_root="pascal_ctx_d2/annotations_ctx459/validation", image_ext="jpg", gt_ext="tif"),
    "pascal21_sem_seg_val": dict(
        kind="sem_seg", vocabulary="pascal_voc_21", ignore_label=255, num_classes=21, image_root="pascal_voc_d2/images/validation",
        sem_seg_root="pascal_voc_d2/annotations_pascal21/validation", image_ext="jpg", gt_ext="png"),
}


def preset(name):
    if name not in PRESETS:
        raise KeyError(f"unknown dataset preset {name!r}; known: {sorted(PRESETS)}")
    return PRESETS[name]


def data_root(root=None):
    """--data-root, else $DETECTRON2_DATASETS, else `datasets` (the reference's convention)."""
    return root or os.getenv("DETECTRON2_DATASETS", "datasets")


def _paths(name, root):
    p = preset(name)
    return {k: os.path.join(root, v) for k, v in p.items() if k.endswith(("_root", "_json"))}


def load_sem_seg(gt_root, image_root, gt_ext="png", image_ext="jpg"):
    """detectron2's load_sem_seg: the files of image_root / gt_root with the extension (one directory level), matched by path relative to
    their root without extension; when the counts differ, the intersection of the base names.  image_id = that relative stem."""
    for d in (gt_root, image_root):
        if not os.path.isdir(d):
            raise FileNotFoundError(f"load_sem_seg: directory {d} does not exist")

    def stem(root, f):
        return os.path.splitext(os.path.normpath(os.path.relpath(f, start=root)))[0]

    inputs = sorted((os.path.join(image_root, f) for f in os.listdir(image_root) if f.endswith(image_ext)), key=lambda f: stem(image_root, f))
    gts = sorted((os.path.join(gt_root, f) for f in os.listdir(gt_root) if f.endswith(gt_ext)), key=lambda f: stem(gt_root, f))
    if not gts:
        raise FileNotFoundError(f"No annotations found in {gt_root}.")
    if len(inputs) != len(gts):
        common = sorted({os.path.basename(f)[:-len(image_ext)] for f in inputs} & {os.path.basename(f)[:-len(gt_ext)] for f in gts})
        inputs = [os.path.join(image_root, f + image_ext) for f in common]
        gts = [os.path.join(gt_root, f + gt_ext) for f in common]
    return [{"file_name": i, "image_id": stem(image_root, i), "sem_seg_file_name": g} for i, g in zip(inputs, gts)]


def load_panoptic_json(json_file, image_dir, gt_dir, semseg_dir):
    """load_ade20k_panoptic_json / load_coco_panoptic_json: one record per annotation, image <gt stem>.jpg, segment categories converted
    to contiguous ids (stuff map for every category, the thing map first) with `isthing` set."""
    if not os.path.isfile(json_file):
        raise FileNotFoundError(f"panoptic JSON {json_file} does not exist")
    with open(json_file, "r") as f:
        js = json.load(f)
    things, stuff = panoptic_category_maps(js["categories"])
    ret = []
    for ann in js["annotations"]:
        segs = []
        for s in ann["segments_info"]:
            s = dict(s)
            isthing = s["category_id"] in things
            s["category_id"] = things[s["category_id"]] if isthing else stuff[s["category_id"]]
            s["isthing"] = isthing
            segs.append(s)
        ret.append({"file_name": os.path.join(image_dir, os.path.splitext(ann["file_name"])[0] + ".jpg"), "image_id": ann["image_id"],
                    "pan_seg_file_name": os.path.join(gt_dir, ann["file_name"]),
                    "sem_seg_file_name": os.path.join(semseg_dir, ann["file_name"]), "segments_info": segs})
    if not ret:
        raise FileNotFoundError(f"No images found in {json_file}!")
    for k in ("file_name", "pan_seg_file_name", "sem_seg_file_name"):
        if not os.path.isfile(ret[0][k]):
            raise FileNotFoundError(ret[0][k])
    return ret, js["categories"]


def load_records(name, root=None):
    """-> (records, metadata) of a preset under the data root.  metadata: ignore_label, class_names, num_classes, vocabulary, and for
    panoptic presets panoptic_json / panoptic_root / categories / the contiguous-id maps / instances_json (the COCO instance
    annotations, which may be absent)."""
    p = preset(name)
    paths = _paths(name, data_root(root))
    meta = {"name": name, "ignore_label": p["ignore_label"], "vocabulary": p["vocabulary"]}
    if p["kind"] == "panoptic":
        records, cats = load_panoptic_json(paths["panoptic_json"], paths["image_root"], paths["panoptic_root"], paths["sem_seg_root"])
        things, stuff = panoptic_category_maps(cats)
        meta.update(panoptic_json=paths["panoptic_json"], panoptic_root=paths["panoptic_root"], categories=cats,
                    thing_dataset_id_to_contiguous_id=things, stuff_dataset_id_to_contiguous_id=stuff,
                    class_names=[c["name"] for c in cats], num_classes=len(cats))
        if "instances_json" in paths:
            meta["instances_json"] = paths["instances_json"]
    else:
        records = load_sem_seg(paths["sem_seg_root"], paths["image_root"], gt_ext=p["gt_ext"], image_ext=p["image_ext"])
        meta.update(thing_dataset_id_to_contiguous_id={}, num_classes=p["num_classes"], class_names=None)
    return records, meta


def preset_vocabulary(name, tokenizer, labels_root=None, thing_contiguous_ids=()):
    """The test mapper's vocabulary of a preset (coco_dataset_mapper_uni.py:196-215, 296-301, 556-566): expressions and
    positive_map_label_to_token from the openseg label file, is_thing[k] = (k - 1 is a thing contiguous id) over cat2ind's keys with
    is_thing[0] = False, open_seg_labels = the prompt-engineered labels."""
    vocab = preset(name)["vocabulary"]
    cats = get_openseg_labels(vocab, root=labels_root)
    expressions, pos_map = create_queries_and_maps(cats, tokenizer)
    things = set(thing_contiguous_ids)
    ind_to_class = cat2ind([{"name": c["name"]} for c in cats])       # the openseg reader already dropped invalid_class_id entries
    is_thing = {k: (k - 1) in things for k in ind_to_class}
    is_thing[0] = False
    return dict(dataset_name=vocab, expressions=expressions, positive_map_label_to_token=pos_map, is_thing=is_thing,
                open_seg_labels=get_openseg_labels(vocab, prompt_engineered=True, root=labels_root))


def default_evaluators(meta, records, labels_root=None):
    """SemSegEvaluator (every preset), COCOPanopticEvaluator (panoptic presets) and COCOInstanceEvaluator (panoptic presets whose
    instance JSON exists), as the reference's build_evaluator picks them.  A missing instance JSON leaves the other two as they are and
    says so in one line on stderr."""
    names = meta["class_names"]
    if names is None:
        names = [c["name"] for c in get_openseg_labels(meta["vocabulary"], root=labels_root)]
        if len(names) != meta["num_classes"]:
            raise ValueError(f"{meta['name']}: {len(names)} labels in the {meta['vocabulary']} label file for {meta['num_classes']} classes")
    evs = [SemSegEvaluator(records, names, meta["ignore_label"])]
    if "panoptic_json" in meta:
        evs.insert(0, COCOPanopticEvaluator(meta["panoptic_json"], meta["panoptic_root"], meta["thing_dataset_id_to_contiguous_id"],
                                            meta["stuff_dataset_id_to_contiguous_id"]))
    inst = meta.get("instances_json")
    if inst is not None:
        if os.path.isfile(inst):
            things = [c["name"] for c in meta["categories"] if c.get("isthing", 0)]
            evs.insert(0, COCOInstanceEvaluator(inst, meta["thing_dataset_id_to_contiguous_id"], things))
        else:
            print(f"{meta['name']}: instance annotations {inst} not found; AP_bbox / AP_segm are not evaluated", file=sys.stderr)
    return evs


# ---------------------------------------------------------------------------------------------------------------------------------
# driver


def read_image(file_name, format="BGR"):
    """detectron2.data.detection_utils.read_image: PIL decode, EXIF orientation applied, converted to `format` (RGB / BGR)."""
    from PIL import Image, ImageOps
    with open(file_name, "rb") as f:
        image = ImageOps.exif_transpose(Image.open(f))
        image = np.asarray(image.convert("RGB"))
    return image[:, :, ::-1] if format == "BGR" else image


def build_input(record, vocabulary, min_size, max_size, input_format):
    """The test loader's input dict for one record: image read and resized with ResizeShortestEdge(min_size, max_size), height / width
    of the original image (so outputs come back at GT resolution), the record's ids and the preset's vocabulary."""
    image = read_image(record["file_name"], input_format)
    height, width = image.shape[:2]
    aug = ResizeShortestEdge([min_size, min_size], max_size)
    resized = aug.apply_image(np.ascontiguousarray(image))
    x = {"image": torch.as_tensor(np.ascontiguousarray(resized.transpose(2, 0, 1))).float(), "height": height, "width": width,
         "file_name": record["file_name"], "image_id": record["image_id"], "task": "detection"}
    x.update(vocabulary)
    return x


@torch.no_grad()
def evaluate_dataset(model, dataset, data_root=None, evaluators=None, max_images=None, tokenizer=None, labels_root=None, min_size=None,
                     max_size=None, input_format=None):
    """Run `model` (HIPIE_IMG) over a dataset preset one image per step, feed the evaluators and return their merged results on rank 0
    (None on other ranks).  min_size / max_size / input_format default to the model's cfg.INPUT (MIN_SIZE_TEST, MAX_SIZE_TEST, FORMAT)
    or 800 / 1333 / BGR.  Under torchrun the first max_images records are sharded over the ranks (parallel.shard_indices); a host
    thread reads and resizes the next image while the device runs the current one."""
    records, meta = load_records(dataset, data_root)
    if max_images is not None:
        records = records[:int(max_images)]
    if tokenizer is None:
        tokenizer = getattr(model, "tokenizer", None)
        if tokenizer is None:
            from .data import load_tokenizer
            tokenizer = load_tokenizer()
    if getattr(model, "tokenizer", None) is None:
        model.tokenizer = tokenizer
    thing_ids = meta["thing_dataset_id_to_contiguous_id"].values()
    vocab = preset_vocabulary(dataset, tokenizer, labels_root, thing_ids)
    cfg = getattr(model, "cfg", None)
    inp_cfg = getattr(cfg, "INPUT", None)
    min_size = min_size or (inp_cfg.MIN_SIZE_TEST if inp_cfg is not None else 800)
    max_size = max_size or (inp_cfg.MAX_SIZE_TEST if inp_cfg is not None else 1333)
    input_format = input_format or (inp_cfg.FORMAT if inp_cfg is not None else "BGR")
    if evaluators is None:
        evaluators = default_evaluators(meta, records, labels_root)
    for ev in evaluators:
        ev.reset()
    if _distributed():
        records = [records[i] for i in shard_indices(len(records), dist.get_world_size(), dist.get_rank())]
    model.eval()
    with ThreadPoolExecutor(max_workers=1) as pool:
        nxt = pool.submit(build_input, records[0], vocab, min_size, max_size, input_format) if records else None
        for i in range(len(records)):
            x = nxt.result()
            nxt = pool.submit(build_input, records[i + 1], vocab, min_size, max_size, input_format) if i + 1 < len(records) else None
            outputs = model([x])
            for ev in evaluators:
                ev.process([x], outputs)
    results = collections.OrderedDict()
    for ev in evaluators:
        r = ev.evaluate()
        if r is not None:
            results.update(r)
    if _distributed() and dist.get_rank() != 0:
        return None
    return results


def _json_safe(o):
    if isinstance(o, dict):
        return {str(k): _json_safe(v) for k, v in o.items()}
    if isinstance(o, (float, np.floating)):
        return None if np.isnan(o) else float(o)
    if isinstance(o, np.integer):
        return int(o)
    return o


def main(argv=None):
    ap = argparse.ArgumentParser(description="Evaluate HIPIE on a segmentation benchmark (mIoU; PQ, and AP_bbox / AP_segm when the "
                                             "instance JSON is present, on panoptic presets).")
    ap.add_argument("--config-file", required=True)
    ap.add_argument("--dataset", required=True, choices=sorted(PRESETS))
    ap.add_argument("--data-root", default=None)
    ap.add_argument("--max-images", type=int, default=None)
    ap.add_argument("--output", default=None, help="also write the results as JSON to this file")
    ap.add_argument("--clip-weights", default=None, help="open_clip state_dict for configs with MODEL.CLIP.ENABLED")
    ap.add_argument("--labels-root", default=None, help="directory of the openseg label files")
    ap.add_argument("--bert-dir", default=None, help="bert-base-uncased directory (vocab.txt)")
    ap.add_argument("opts", nargs=argparse.REMAINDER, help="KEY VALUE pairs merged into the config")
    args = ap.parse_args(argv)
    from .config import setup_cfg
    from .data import load_tokenizer
    from .registry import DetectionCheckpointer, build_model
    cfg = setup_cfg(args.config_file, args.opts)
    if cfg.MODEL.CLIP.ENABLED and not args.clip_weights:
        ap.error("the config sets MODEL.CLIP.ENABLED: pass --clip-weights (an open_clip state_dict), or set MODEL.CLIP.ENABLED False")
    if cfg.MODEL.CLIP.ENABLED_TRAIN:
        ap.error("MODEL.CLIP.ENABLED_TRAIN rewrites the test vocabulary's token map; evaluation supports it off only")
    if "LOCAL_RANK" in os.environ and not dist.is_initialized():
        torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
        dist.init_process_group("nccl")
    model = build_model(cfg)
    model.eval()
    if getattr(cfg.MODEL, "WEIGHTS", ""):
        DetectionCheckpointer(model).load(cfg.MODEL.WEIGHTS)
    model.cfg = cfg
    if cfg.MODEL.CLIP.ENABLED:
        try:
            from open_clip import tokenize
        except ImportError:
            tokenize = None
        sd = torch.load(args.clip_weights, map_location="cpu", weights_only=True)
        model.attach_clip(sd, get_openseg_labels("coco_panoptic", prompt_engineered=True, root=args.labels_root), tokenize=tokenize)
    tok = load_tokenizer(args.bert_dir)
    res = evaluate_dataset(model, args.dataset, args.data_root, max_images=args.max_images, tokenizer=tok, labels_root=args.labels_root)
    if res is not None:
        line = json.dumps(_json_safe(res))
        print(line)
        if args.output:
            with open(args.output, "w") as f:
                f.write(line + "\n")
    if dist.is_initialized():
        dist.destroy_process_group()
    return res


if __name__ == "__main__":
    main()
