"""GPU: the instance-overlap kernels and the instance evaluator end to end.

* hipie_mask_pack / hipie_rle_expand / hipie_mask_overlaps equal numpy bit for bit: H * W not a multiple of 32 or 256, odd W,
  N, M in {0, 1, 100}, all-zero and all-one masks, run lists starting with a foreground run; a run list that does not cover the image
  raises.
* evaluate_dataset on a synthetic ADE-style tree with the vit_tiny random-weight HIPIE_IMG, the instance JSON built from a first
  forward's own predictions (copies, eroded copies near the IoU thresholds, a crowd; compressed-string, uncompressed and polygon GTs):
  bbox and segm equal the host oracle (numpy intersections + hipie_b200.cocoeval) on the recorded outputs, with --max-images and the
  command line too.
* With FG-mode scoring a stuff class can enter the top 100 only with score exactly 0; such a detection is refused, as the reference's
  assert refuses it.
"""
import json
import os

import numpy as np
import pytest
import torch

from test_instance_eval_host import _dense, rle_to_string

pytestmark = pytest.mark.gpu


def _pack_np(masks):
    N, H, W = masks.shape
    K = H * W
    flat = masks.reshape(N, K).astype(bool)
    KW = (K + 255) // 256 * 8
    pad = np.zeros((N, KW * 32), bool)
    pad[:, :K] = flat
    return np.packbits(pad, axis=1, bitorder="little").view("<u4").view(np.int32).reshape(N, KW)


def _runs_of(mask):
    """Column-major COCO counts of a (H, W) bool mask, background first."""
    flat = mask.T.reshape(-1).astype(np.int8)
    change = np.flatnonzero(np.diff(flat)) + 1
    bounds = np.concatenate([[0], change, [flat.size]])
    counts = np.diff(bounds).tolist()
    if flat.size and flat[0]:
        counts = [0] + counts
    return counts


def _masks(rng, N, H, W):
    m = rng.rand(N, H, W) < rng.rand(N, 1, 1)
    if N > 2:
        m[0] = False
        m[1] = True
    return m


@pytest.mark.parametrize("H,W", [(1, 1), (7, 9), (33, 31), (16, 16), (97, 131), (512, 683)])
@pytest.mark.parametrize("N,M", [(0, 1), (1, 0), (1, 1), (100, 100)])
def test_pack_expand_overlaps_match_numpy(cuda, H, W, N, M):
    from hipie_b200 import ops
    rng = np.random.RandomState(H * 7 + N + M)
    if H * W > 100000 and N * M > 1:
        N, M = 100, 20
    pm = _masks(rng, N, H, W)
    gm = _masks(rng, M, H, W)
    bits, area = ops.mask_pack(torch.from_numpy(pm.astype(np.uint8)).cuda())
    assert np.array_equal(bits.cpu().numpy(), _pack_np(pm)) and np.array_equal(area.cpu().numpy(), pm.reshape(N, H * W).sum(1))
    runs = [_runs_of(g) for g in gm]
    assert all(_dense(r, H, W).tolist() == g.tolist() for r, g in zip(runs, gm))
    ends, off = ops.rle_ends(runs, H, W)
    gbits = ops.rle_expand(torch.from_numpy(ends).cuda(), torch.from_numpy(off).cuda(), H, W)
    assert np.array_equal(gbits.cpu().numpy(), _pack_np(gm))
    inter = ops.mask_overlaps(bits, gbits, H, W)
    want = pm.reshape(N, H * W).astype(np.int64) @ gm.reshape(M, H * W).astype(np.int64).T
    assert inter.shape == (N, M) and np.array_equal(inter.cpu().numpy(), want)


def test_rle_expand_foreground_first_and_refusal(cuda):
    from hipie_b200 import ops
    H, W = 5, 13
    runs = [[0, 65], [0, 3, 62], [65], [0, 1, 1, 1, 1, 61]]
    ends, off = ops.rle_ends(runs, H, W)
    g = ops.rle_expand(torch.from_numpy(ends).cuda(), torch.from_numpy(off).cuda(), H, W)
    assert np.array_equal(g.cpu().numpy(), _pack_np(np.stack([_dense(r, H, W) for r in runs])))
    bad = torch.tensor([3, 60], dtype=torch.int32, device="cuda")                 # ends at 60 of 65 pixels
    with pytest.raises(ValueError, match="do not sum"):
        ops.rle_expand(bad, torch.tensor([0, 2], dtype=torch.int64, device="cuda"), H, W)


# ------------------------------------------------------------------------------------------------------------------- end to end

WORDS = ["wall", "person", "sky"]


def _tree(tmp_path, all_things=True):
    from test_evaluation_gpu import _tree as pan_tree
    cats, images = pan_tree(tmp_path)
    js_path = tmp_path / "data" / "ade" / "ADEChallengeData2016" / "ade20k_panoptic_val.json"
    if all_things:
        js = json.loads(js_path.read_text())
        for c in js["categories"]:
            c["isthing"] = 1
        js_path.write_text(json.dumps(js))
        cats = js["categories"]
    return cats, images


class _Recorder:
    def __init__(self, model):
        self.model, self.calls = model, []
        self.tokenizer = model.tokenizer

    def eval(self):
        return self

    def __call__(self, inputs):
        out = self.model(inputs)
        inst = out[0]["instances"]
        self.calls.append((inputs[0], inst.pred_masks.cpu().numpy().astype(bool), inst.pred_boxes.tensor.cpu().numpy(),
                           inst.scores.cpu().numpy(), inst.pred_classes.cpu().numpy()))
        return out


def _erode(m):
    e = m.copy()
    e[1:] &= m[:-1]
    e[:-1] &= m[1:]
    e[:, 1:] &= m[:, :-1]
    e[:, :-1] &= m[:, 1:]
    return e


def _instance_json(path, calls, cat_ids):
    """GT from the predictions of a first forward: the best masks copied, eroded copies, a crowd, the three segmentation formats."""
    rng = np.random.RandomState(0)
    images, anns = [], []
    for i, (x, masks, boxes, scores, classes) in enumerate(calls):
        H, W = masks.shape[1:]
        images.append({"id": 10 + i, "file_name": os.path.basename(x["file_name"]), "height": int(H), "width": int(W)})
        order = np.argsort(-scores, kind="stable")[:6]
        for j, k in enumerate(order):
            m = masks[k] if j % 2 == 0 else _erode(masks[k])
            if not m.any():
                continue
            runs = _runs_of(m)
            fmt = j % 3
            seg = ({"size": [int(H), int(W)], "counts": rle_to_string(runs)} if fmt == 0 else
                   {"size": [int(H), int(W)], "counts": [int(c) for c in runs]})
            ys, xs = np.nonzero(m)
            anns.append({"id": len(anns) + 1, "image_id": 10 + i, "category_id": cat_ids[int(classes[k])], "iscrowd": int(j == 5),
                         "area": int(m.sum()), "bbox": [float(xs.min()), float(ys.min()), float(xs.max() - xs.min() + 1),
                                                        float(ys.max() - ys.min() + 1)], "segmentation": seg})
        x0, y0 = rng.randint(0, W // 2), rng.randint(0, H // 2)           # a polygon GT
        anns.append({"id": len(anns) + 1, "image_id": 10 + i, "category_id": cat_ids[int(classes[order[0]])] if len(order) else cat_ids[0],
                     "iscrowd": 0, "area": float((W // 3) * (H // 3)), "bbox": [x0, y0, W // 3, H // 3],
                     "segmentation": [[x0, y0, x0 + W // 3, y0, x0 + W // 3, y0 + H // 3, x0, y0 + H // 3]]})
    js = {"images": images, "annotations": anns, "categories": [{"id": c, "name": f"c{c}"} for c in cat_ids]}
    with open(path, "w") as f:
        json.dump(js, f)
    return js


def _oracle(calls, js, cat_ids, names):
    """Host oracle: numpy intersections of the recorded masks with the decoded GTs, then hipie_b200.cocoeval."""
    from hipie_b200 import cocoeval as ce
    by_name = {im["file_name"]: im for im in js["images"]}
    per = {"bbox": [], "segm": []}
    anyp = False
    for x, masks, boxes, scores, classes in calls:
        im = by_name[os.path.basename(x["file_name"])]
        H, W = im["height"], im["width"]
        anns = [a for a in js["annotations"] if a["image_id"] == im["id"]]
        gm = np.stack([_dense(ce.ann_to_runs(a, H, W), H, W) for a in anns]) if anns else np.zeros((0, H, W), bool)
        inter = masks.reshape(len(masks), -1).astype(np.int64) @ gm.reshape(len(gm), -1).astype(np.int64).T
        gts = [{"id": a["id"], "category_id": a["category_id"], "iscrowd": a["iscrowd"], "area": a["area"]} for a in anns]
        crowd = [a["iscrowd"] for a in anns]
        xywh = boxes.astype(np.float32).copy()
        xywh[:, 2] -= xywh[:, 0]
        xywh[:, 3] -= xywh[:, 1]
        xywh = xywh.tolist()
        cats = [cat_ids[int(c)] for c in classes]
        sc = scores.tolist()
        area = masks.reshape(len(masks), -1).sum(1)
        dts = [{"category_id": c, "score": s, "area": int(a)} for c, s, a in zip(cats, sc, area)]
        per["segm"].append((im["id"], ce.image_records(sorted(cat_ids), gts, dts, ce.mask_iou(inter, area, gm.reshape(len(gm), -1).sum(1), crowd))))
        dts = [{"category_id": c, "score": s, "area": b[2] * b[3]} for c, s, b in zip(cats, sc, xywh)]
        per["bbox"].append((im["id"], ce.image_records(sorted(cat_ids), gts, dts, ce.bbox_iou(xywh, [a["bbox"] for a in anns], crowd))))
        anyp = anyp or len(sc) > 0
    return {t: ce.evaluate_records(per[t], sorted(cat_ids), names, anyp) for t in ("bbox", "segm")}


def _same(got, want):
    assert list(got) == list(want)
    np.testing.assert_array_equal(np.array([np.nan if v is None else v for v in got.values()], dtype=float),
                                  np.array(list(want.values()), dtype=float))


def test_evaluate_dataset_instances_match_host_oracle(cuda, tmp_path):
    from test_evaluation_gpu import _tiny_model
    from hipie_b200.data import load_tokenizer
    from hipie_b200.evaluation import evaluate_dataset
    cats, images = _tree(tmp_path)
    tok = load_tokenizer(str(tmp_path))
    model = _tiny_model()
    model.tokenizer = tok
    kw = dict(tokenizer=tok, labels_root=str(tmp_path / "labels"), min_size=96, max_size=128, input_format="RGB")
    first = _Recorder(model)
    res0 = evaluate_dataset(first, "ade20k_panoptic_val", str(tmp_path / "data"), **kw)
    assert "bbox" not in res0 and "panoptic_seg" in res0                # no instance JSON yet: today's output
    cat_ids = [c["id"] for c in cats]
    names = [c["name"] for c in cats]
    inst_path = tmp_path / "data" / "ade" / "ADEChallengeData2016" / "ade20k_instance_val.json"
    js = _instance_json(inst_path, first.calls, cat_ids)
    assert sum(len(c[3]) for c in first.calls) > 0 and len(js["annotations"]) > 8

    rec = _Recorder(model)
    res = evaluate_dataset(rec, "ade20k_panoptic_val", str(tmp_path / "data"), **kw)
    want = _oracle(rec.calls, js, cat_ids, names)
    for t in ("bbox", "segm"):
        _same(res[t], want[t])
    assert res["segm"]["AP50"] > 0 and "AP-person" in res["segm"]
    assert "panoptic_seg" in res and "sem_seg" in res

    rec2 = _Recorder(model)
    res2 = evaluate_dataset(rec2, "ade20k_panoptic_val", str(tmp_path / "data"), max_images=2, **kw)
    assert len(rec2.calls) == 2
    want2 = _oracle(rec2.calls, js, cat_ids, names)
    for t in ("bbox", "segm"):
        _same(res2[t], want2[t])

    from hipie_b200 import evaluation, registry
    cfg_file = os.path.join(os.path.dirname(__file__), "golden", "hipie_configs", "projects", "HIPIE", "configs", "eval",
                            "image_joint_r50_pan_maskdino_ade_test.yaml")
    orig = registry.build_model
    rec3 = _Recorder(model)
    registry.build_model = lambda cfg: rec3
    try:
        out = tmp_path / "res.json"
        evaluation.main(["--config-file", cfg_file, "--dataset", "ade20k_panoptic_val", "--data-root", str(tmp_path / "data"),
                         "--labels-root", str(tmp_path / "labels"), "--bert-dir", str(tmp_path), "--output", str(out),
                         "MODEL.WEIGHTS", "", "MODEL.CLIP.ENABLED", "False", "INPUT.MIN_SIZE_TEST", "96", "INPUT.MAX_SIZE_TEST", "128",
                         "INPUT.FORMAT", "RGB"])
    finally:
        registry.build_model = orig
    got = json.loads(out.read_text())
    want3 = _oracle(rec3.calls, js, cat_ids, names)
    for t in ("bbox", "segm"):
        _same(got[t], want3[t])


def test_stuff_classes_enter_the_top100_only_at_score_zero(cuda, tmp_path):
    """The 3-word vocabulary with one thing class: FG-mode scoring masks the two stuff classes to -9999, so their probability is
    exactly 0 and they fill the top 100 only behind every thing entry.  The instance evaluator refuses them, as the reference does."""
    from test_evaluation_gpu import _tiny_model
    from hipie_b200.data import load_tokenizer
    from hipie_b200.evaluation import COCOInstanceEvaluator, evaluate_dataset
    cats, images = _tree(tmp_path, all_things=False)
    tok = load_tokenizer(str(tmp_path))
    model = _tiny_model()
    model.tokenizer = tok
    rec = _Recorder(model)
    evaluate_dataset(rec, "ade20k_panoptic_val", str(tmp_path / "data"), tokenizer=tok, labels_root=str(tmp_path / "labels"),
                     min_size=96, max_size=128, input_format="RGB")
    things = {i for i, c in enumerate(cats) if c["isthing"]}
    stuff_seen = False
    for _, masks, boxes, scores, classes in rec.calls:
        is_stuff = np.array([int(c) not in things for c in classes], bool)
        assert (scores[is_stuff] == 0).all()
        if is_stuff.any():
            assert scores[~is_stuff].min() > 0 and np.flatnonzero(~is_stuff).max() < np.flatnonzero(is_stuff).min()
        stuff_seen = stuff_seen or is_stuff.any()
    if stuff_seen:
        path = tmp_path / "i.json"
        x, masks, boxes, scores, classes = rec.calls[0]
        path.write_text(json.dumps({"images": [{"id": 10, "file_name": "a.jpg", "height": masks.shape[1], "width": masks.shape[2]}],
                                    "annotations": [], "categories": [{"id": 1, "name": "person"}]}))
        ev = COCOInstanceEvaluator(str(path), {1: 1}, ["person"], distributed=False)
        with pytest.raises(ValueError, match="class="):
            ev._add_image(10, np.zeros((len(scores), 0), np.int32), masks.reshape(len(masks), -1).sum(1), boxes, scores, classes, [], [], [])
