"""Golden fixture of COCO AP from the REAL reference (needs the reference tree that oracle/ref_import.py mounts):

    python oracle/gen_golden_coco_eval.py      # writes tests/golden/ref_coco_eval.pt

  ref_coco_eval.pt   detectron2/evaluation/refcocoeval.py executed unmodified: Params, evaluateImg, accumulate and summarize (pycocotools'
                     COCOeval logic verbatim); detectron2/evaluation/coco_evaluation.py's _derive_coco_results and instances_to_coco_json
                     (with the real BoxMode of detectron2/structures/boxes.py).

What is stubbed or restated:
  * pycocotools.mask is absent and stubbed.  The IoUs are planted: each (image, category) gets integer intersection counts and mask
    areas, and coco_eval.ious is set from them with maskApi.c rleIou's formula (i / (da + ga - i), i / da for a crowd GT, 0 where
    i = 0).  The fixture stores the counts, so the test feeds the same integers to hipie_b200.cocoeval.
  * pycocotools' COCOeval.evaluate() loop over categories, area ranges and images is commented out in refcocoeval.py; it is restated
    here (evalImgs in category-major, area, image order; _paramsEval a deep copy of params).  _prepare runs unmodified on a minimal
    in-memory COCO (getAnnIds / loadAnns / getImgIds / getCatIds of pycocotools' coco.py, loadRes's detection ids 1..N and areas).
  * numpy 2 removed np.float, which accumulate uses; it is set to float.  tabulate / create_small_table only format log lines and
    return "".

Planted cases: score ties within one image and across images; a crowd GT that matches two detections; GT areas exactly 32^2 and 96^2;
IoUs exactly 0.5, 0.75 and 0.95; an image with more than 100 detections and ones with fewer than 10; a category with detections but no
GT and one with GT but no detections; an image with neither; a GT with id 0 is not planted (its matches read as unmatched).
"""
import copy
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_import  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden")
REF = ref_import.REF_ROOT


class MiniCOCO:
    """pycocotools COCO's index (createIndex) and the accessors _prepare calls."""

    def __init__(self, images, anns, cats):
        self.imgs = {i: {"id": i} for i in images}
        self.anns = {a["id"]: a for a in anns}
        self.cats = {c: {"id": c} for c in cats}
        self.imgToAnns = {}
        for a in anns:
            self.imgToAnns.setdefault(a["image_id"], []).append(a)

    def getImgIds(self):
        return list(self.imgs)

    def getCatIds(self):
        return list(self.cats)

    def getAnnIds(self, imgIds=(), catIds=()):
        lists = [self.imgToAnns[i] for i in imgIds if i in self.imgToAnns]
        anns = [a for ls in lists for a in ls]
        return [a["id"] for a in anns if a["category_id"] in catIds]

    def loadAnns(self, ids):
        return [self.anns[i] for i in ids]

    def annToRLE(self, ann):
        return ann["segmentation"]


def rle_iou(inter, da, ga, crowd):
    inter = np.asarray(inter, dtype=np.int64)
    o = np.zeros(inter.shape)
    for d in range(inter.shape[0]):
        for g in range(inter.shape[1]):
            i = int(inter[d, g])
            u = 1 if i == 0 else (int(da[d]) if crowd[g] else int(da[d]) + int(ga[g]) - i)
            o[d, g] = i / u
    return o


def plant(seed=0):
    """-> images: list of dicts (id, gts: [{id, category_id, iscrowd, area, pixels}], dts: [{category_id, score, area}], inter (D, G))."""
    rng = np.random.RandomState(seed)
    cats = [1, 3, 4, 7]                     # 4: detections but no GT; 7: GT but no detections
    images = []

    def img(iid, gts, dts, inter):
        images.append(dict(id=iid, gts=gts, dts=dts, inter=np.asarray(inter, dtype=np.int64).reshape(len(dts), len(gts))))

    # image 5: thresholds hit exactly, area-range edges, a crowd matching two detections, score ties inside the image
    gts = [dict(id=11, category_id=1, iscrowd=0, area=32 * 32, pixels=100), dict(id=12, category_id=1, iscrowd=0, area=96 * 96, pixels=100),
           dict(id=13, category_id=1, iscrowd=1, area=5000, pixels=400), dict(id=14, category_id=3, iscrowd=0, area=2000.5, pixels=80),
           dict(id=15, category_id=7, iscrowd=0, area=300, pixels=300)]
    dts = [dict(category_id=1, score=0.9, area=100), dict(category_id=1, score=0.8, area=100), dict(category_id=1, score=0.8, area=60),
           dict(category_id=1, score=0.7, area=40), dict(category_id=3, score=0.6, area=80), dict(category_id=4, score=0.95, area=50),
           dict(category_id=1, score=0.5, area=9216)]
    inter = np.zeros((7, 5), np.int64)
    inter[0, 0] = 100                       # IoU 1
    inter[1, 1] = 100 * 2 // 3              # IoU 66/134
    inter[1, 0] = 50                        # 50 / 150
    inter[2, 1] = 64                        # 64 / 96 = 0.666..
    inter[1, 2] = 60                        # crowd: 60 / 100 = 0.6
    inter[2, 2] = 30                        # crowd: 30 / 60 = 0.5 exactly
    inter[3, 2] = 30                        # crowd: 30 / 40 = 0.75 exactly
    inter[4, 3] = 76                        # 76 / 84 = 0.9047..
    inter[6, 1] = 95                        # 95 / 9221
    img(5, gts, dts, inter)

    # image 2: IoU exactly 0.95 and 0.5 on plain GTs, fewer than 10 detections, a tie with image 5's 0.8
    gts = [dict(id=21, category_id=1, iscrowd=0, area=1023, pixels=200), dict(id=22, category_id=3, iscrowd=0, area=9217, pixels=100)]
    dts = [dict(category_id=1, score=0.8, area=190), dict(category_id=3, score=0.8, area=100), dict(category_id=3, score=0.3, area=100)]
    inter = np.zeros((3, 2), np.int64)
    inter[0, 0] = 190                       # 190 / 200 = 0.95
    inter[1, 1] = 200 // 3                  # 66 / 134
    inter[2, 1] = 200 // 3
    img(2, gts, dts, inter)

    # image 9: neither GT nor detections
    img(9, [], [], np.zeros((0, 0)))

    # image 7: 130 detections of category 1 (computeIoU keeps the best 100), scores quantised so that many tie, 12 GTs
    G, D = 12, 130
    gts = [dict(id=700 + j, category_id=1, iscrowd=int(j == 11), area=float(rng.choice([500, 1024, 3000, 9216, 12000])), pixels=200)
           for j in range(G)]
    dts = [dict(category_id=1, score=float(rng.randint(0, 20)) / 20, area=int(rng.randint(50, 250))) for _ in range(D)]
    inter = np.zeros((D, G), np.int64)
    for d in range(D):
        for g in rng.choice(G, 2, replace=False):
            inter[d, g] = rng.randint(0, min(dts[d]["area"], 200) + 1)
    for d in range(0, 40, 4):               # a few exact 0.5 / 0.75 ratios on plain GTs (pixels 200)
        dts[d]["area"] = 200
        inter[d, d // 4] = [134, 172][d % 8 // 4] if d // 4 < 11 else 0
    img(7, gts, dts, inter)

    # image 3: only detections (category 1 and 4), fewer than 10
    dts = [dict(category_id=1, score=0.4, area=30), dict(category_id=4, score=0.4, area=30)]
    img(3, [], dts, np.zeros((2, 0)))
    return cats, images


def run_reference(cats, images):
    ref_import.install()
    rc = ref_import._load_file("detectron2.evaluation.refcocoeval", f"{REF}/detectron2/evaluation/refcocoeval.py")
    np.float = float
    gt_anns, dt_anns = [], []
    for im in images:
        for g in im["gts"]:
            gt_anns.append(dict(id=g["id"], image_id=im["id"], category_id=g["category_id"], iscrowd=g["iscrowd"], area=g["area"],
                                segmentation=None))
        for d in im["dts"]:
            dt_anns.append(dict(id=len(dt_anns) + 1, image_id=im["id"], category_id=d["category_id"], score=d["score"], area=d["area"],
                                iscrowd=0, segmentation=None))            # loadRes: ids 1..N in result order
    coco_gt = MiniCOCO([im["id"] for im in images], gt_anns, cats)
    coco_dt = MiniCOCO([im["id"] for im in images], dt_anns, cats)
    ev = rc.RefCOCOeval(coco_gt, coco_dt, "segm")
    p = ev.params
    p.imgIds = list(np.unique(p.imgIds))                                  # pycocotools COCOeval.evaluate()
    p.catIds = list(np.unique(p.catIds))
    p.maxDets = sorted(p.maxDets)
    ev.params = p
    ev._prepare()
    by_id = {im["id"]: im for im in images}
    ev.ious = {}
    for i in p.imgIds:
        im = by_id[int(i)]
        for c in p.catIds:
            gi = [j for j, g in enumerate(im["gts"]) if g["category_id"] == c]
            di = [k for k, d in enumerate(im["dts"]) if d["category_id"] == c]
            if not gi and not di:
                ev.ious[i, c] = []
                continue
            di = [di[k] for k in np.argsort([-im["dts"][k]["score"] for k in di], kind="mergesort")][:p.maxDets[-1]]
            if not gi or not di:
                ev.ious[i, c] = []
                continue
            ev.ious[i, c] = rle_iou(im["inter"][np.ix_(di, gi)], [im["dts"][k]["area"] for k in di], [im["gts"][j]["pixels"] for j in gi],
                                    [im["gts"][j]["iscrowd"] for j in gi])
    ev.evalImgs = [ev.evaluateImg(imgId, catId, areaRng, p.maxDets[-1]) for catId in p.catIds for areaRng in p.areaRng for imgId in p.imgIds]
    ev._paramsEval = copy.deepcopy(ev.params)
    ev.accumulate()
    ev.summarize()
    return ev


def derive(ev, class_names):
    ref_import.install()
    boxes_mod = ref_import._load_file("detectron2.structures.boxes", f"{REF}/detectron2/structures/boxes.py")
    import detectron2.structures as d2s                                   # the stub package
    d2s.BoxMode = boxes_mod.BoxMode
    ce = ref_import._load_file("detectron2.evaluation.coco_evaluation", f"{REF}/detectron2/evaluation/coco_evaluation.py")
    ce.create_small_table = ce.tabulate = lambda *a, **k: ""              # logging only (tabulate is absent)
    me = types.SimpleNamespace(_logger=types.SimpleNamespace(info=lambda *a: None, warn=lambda *a: None, warning=lambda *a: None))
    res = ce.COCOEvaluator._derive_coco_results(me, ev, "segm", class_names=class_names)
    none = ce.COCOEvaluator._derive_coco_results(me, None, "segm", class_names=class_names)
    one = ce.COCOEvaluator._derive_coco_results(me, ev, "segm", class_names=["only"])
    # instances_to_coco_json on boxes whose float32 XYXY -> XYWH rounds
    g = torch.Generator().manual_seed(1)
    xyxy = torch.rand(6, 4, generator=g) * 1000
    xyxy[:, 2:] += xyxy[:, :2]
    xyxy[0] = torch.tensor([0.1, 0.2, 1000.3, 700.7])

    class Inst:
        pred_boxes = types.SimpleNamespace(tensor=xyxy)
        scores = torch.rand(6, generator=g)
        pred_classes = torch.arange(6)

        def __len__(self):
            return 6

        def has(self, k):
            return False
    js = ce.instances_to_coco_json(Inst(), 42)
    return res, none, one, dict(xyxy=xyxy, scores=Inst.scores, json=js)


def main():
    cats, images = plant()
    ev = run_reference(cats, images)
    names = ["dog", "cat", "kite", "boat"]
    res, none, one, boxes = derive(ev, names)
    out = dict(cats=cats, images=[dict(im, inter=torch.from_numpy(im["inter"])) for im in images], class_names=names,
               precision=torch.from_numpy(ev.eval["precision"]), recall=torch.from_numpy(ev.eval["recall"]),
               stats=torch.from_numpy(np.asarray(ev.stats)), results=res,
               results_no_predictions=none, results_one_name=one, boxes=boxes)
    path = os.path.join(OUT, "ref_coco_eval.pt")
    torch.save(out, path)
    print(f"wrote {path}: stats {np.round(ev.stats, 4).tolist()}")


if __name__ == "__main__":
    main()
