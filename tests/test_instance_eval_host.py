"""CPU: COCO instance evaluation on the host (hipie_b200.cocoeval) and the instance evaluator's wiring.

* The matcher equals the reference's COCOeval (refcocoeval.py evaluateImg / accumulate / summarize, run unmodified into
  tests/golden/ref_coco_eval.pt) on planted intersection tables: precision, recall and stats exactly, _derive_coco_results within
  rtol 1e-12, and instances_to_coco_json's float32 XYWH boxes.
* rle_from_string on hand-encoded strings (negative deltas, the first three counts taken as they are) and a round trip through a
  test-side restatement of maskApi.c rleToString.
* polygon_runs on hand-stepped cases (a rectangle, a triangle, a polygon crossing the image edge, two polygons of one annotation) and
  invariants (vertex-start rotation, union).
* The readers and refusals, and a 2-rank gloo gather equal to the single-process result.
"""
import json
import os
import socket

import numpy as np
import pytest
import torch

from hipie_b200 import cocoeval as ce

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_coco_eval.pt")


def _records(fx):
    per_image = []
    for im in fx["images"]:
        inter = im["inter"].numpy()
        gts = [dict(g) for g in im["gts"]]
        dts = [dict(d) for d in im["dts"]]
        ious = ce.mask_iou(inter, [d["area"] for d in dts], [g["pixels"] for g in gts], [g["iscrowd"] for g in gts])
        per_image.append((im["id"], ce.image_records(fx["cats"], gts, dts, ious)))
    return per_image


def test_matcher_equals_reference_cocoeval():
    fx = torch.load(GOLDEN, weights_only=False)
    per_image = _records(fx)
    precision, recall, _ = ce.accumulate(per_image[::-1], len(fx["cats"]))       # input order does not matter: image-id order
    np.testing.assert_array_equal(precision, fx["precision"].numpy())
    np.testing.assert_array_equal(recall, fx["recall"].numpy())
    stats = ce.summarize(precision, recall)
    np.testing.assert_array_equal(stats, fx["stats"].numpy())
    res = ce.derive_results(stats, precision, fx["class_names"])
    want = fx["results"]
    assert list(res) == list(want)
    np.testing.assert_allclose([res[k] for k in want], [want[k] for k in want], rtol=1e-12, equal_nan=True)
    got_none = ce.evaluate_records(per_image, fx["cats"], fx["class_names"], any_predictions=False)
    assert list(got_none) == list(fx["results_no_predictions"]) and all(np.isnan(v) for v in got_none.values())
    assert ce.derive_results(stats, precision, ["only"]) == pytest.approx(fx["results_one_name"], rel=1e-12, nan_ok=True)
    with pytest.raises(ValueError):
        ce.derive_results(stats, precision, ["a", "b"])


def test_planted_cases_are_exercised():
    """The fixture's planted cases reach the branches they are meant for."""
    fx = torch.load(GOLDEN, weights_only=False)
    recs = dict(_records(fx))
    scores, matched, ignored, npig = recs[5][(0, 0)]                # image 5, category 1, area all
    # detections sorted by -score with a stable sort: the two 0.8 keep their order
    assert scores.tolist() == [0.9, 0.8, 0.8, 0.7, 0.5]
    # the crowd GT (ignored) matches two detections at 0.5 (IoU 0.6 and 0.75 = i / da), and the second one still at exactly 0.75;
    # detection 2 prefers the plain GT at 0.667 and stays unmatched from 0.7 on
    t50, t70, t75 = 0, 4, 5
    assert ignored[t50, 1] and ignored[t50, 3] and ignored[t75, 3] and not ignored[t75, 1]
    assert matched[t50, 2] and not ignored[t50, 2] and not matched[t70, 2]
    assert npig == 2
    assert recs[5][(0, 1)][3] == 1                                  # area exactly 32^2 is small (inclusive bounds) ...
    assert recs[5][(0, 2)][3] == 2 and recs[5][(0, 3)][3] == 1      # ... and medium; 96^2 is medium and large
    assert recs[7][(0, 0)][0].shape == (100,)                       # 130 detections cut at 100
    assert 9 not in [i for i, r in _records(fx) if r]               # the empty image has no records
    prec = fx["precision"].numpy()
    assert (prec[:, :, 2] == -1).all()                             # category 4: detections, no GT
    assert (prec[:, :, 3, 0] == 0).all() and (fx["recall"].numpy()[:, 3, 0] == 0).all()    # category 7: GT, no detections


def test_instances_to_coco_json_boxes():
    fx = torch.load(GOLDEN, weights_only=False)
    b = fx["boxes"]
    xywh = b["xyxy"].numpy().astype(np.float32).copy()
    xywh[:, 2] -= xywh[:, 0]
    xywh[:, 3] -= xywh[:, 1]
    assert xywh.tolist() == [r["bbox"] for r in b["json"]]
    assert b["scores"].tolist() == [r["score"] for r in b["json"]]


def test_bbox_iou_cases():
    dt = [[0, 0, 10, 10], [5, 5, 10, 10], [20, 20, 1, 1], [0, 0, 0, 0]]
    gt = [[0, 0, 10, 10], [5, 0, 10, 10]]
    o = ce.bbox_iou(dt, gt, [0, 1])
    assert o[0, 0] == 1.0 and o[1, 0] == 25 / 175 and o[0, 1] == 50 / 100 and o[1, 1] == 50 / 100
    assert (o[2] == 0).all() and (o[3] == 0).all()
    m = ce.mask_iou([[10, 0], [0, 0]], [20, 0], [15, 0], [0, 1])
    assert m[0, 0] == 10 / 25 and m[0, 1] == 0 and m[1, 1] == 0


# ------------------------------------------------------------------------------------------------------------------- run lists


def rle_to_string(cnts):
    """maskApi.c rleToString, restated on the test side."""
    out = []
    for i, c in enumerate(cnts):
        x = int(c)
        if i > 2:
            x -= int(cnts[i - 2])
        more = True
        while more:
            ch = x & 0x1f
            x >>= 5
            more = (x != -1) if (ch & 0x10) else (x != 0)
            if more:
                ch |= 0x20
            out.append(chr(ch + 48))
    return "".join(out)


def test_rle_string_hand_encoded():
    # "0" -> 0; ";" = 11; "1" -> 1; count 3: delta +2 on cnts[1]; count 4: delta -5 on cnts[2] ('K' = 75 - 48 = 27 = 0x1b: sign bit,
    # value 0x1b - 32 = -5)
    assert ce.rle_from_string("0;1", 2, 6).tolist() == [0, 11, 1]
    got = ce.rle_from_string("0;12K", 4, 4).tolist()
    assert got[:4] == [0, 11, 1, 13] and got[4] == (1 - 5) & 0xffffffff
    # two-character values: 100 = 0b11_00100 -> 'T' (0x24 | 0x20 continuation -> 4 + 32 + 48 = 84) then '3' (3 + 48)
    assert ce.rle_from_string("T3", 1, 100).tolist() == [100]
    assert rle_to_string([100]) == "T3"
    # m <= 2 takes values as they are, even when a later delta would be negative
    assert ce.rle_from_string(rle_to_string([7, 3, 9, 1, 30]), 1, 50).tolist() == [7, 3, 9, 1, 30]


@pytest.mark.parametrize("seed", range(4))
def test_rle_string_round_trip(seed):
    rng = np.random.RandomState(seed)
    cnts = rng.randint(0, 5000, rng.randint(1, 60)).tolist()
    cnts[0] = int(rng.randint(0, 2)) * cnts[0]
    assert ce.rle_from_string(rle_to_string(cnts)).tolist() == cnts


def _dense(counts, h, w):
    flat = np.zeros(h * w, bool)
    pos = 0
    for i, c in enumerate(np.asarray(counts, dtype=np.int64)):
        if i % 2:
            flat[pos:pos + c] = True
        pos += c
    assert pos == h * w
    return flat.reshape(w, h).T                   # column-major


def test_polygon_rectangle_and_triangle():
    # a rectangle with vertices on pixel centres covers the pixels between them inclusive of the left/top, as rleFrPoly rasterises
    m = _dense(ce.polygon_runs([1, 1, 4, 1, 4, 3, 1, 3], 6, 7), 6, 7)
    want = np.zeros((6, 7), bool)
    want[1:3, 1:4] = True
    np.testing.assert_array_equal(m, want)
    # a right triangle (0,0) (4,0) (0,4), stepped by hand through rleFrPoly: x5 the hypotenuse runs u = 20 - t, v = t; column x is
    # sampled where (u + .5) / 5 - .5 = x, i.e. u = 5x + 2, with yd = ceil((v_prev + .5) / 5 - .5) = 3 - x; the top edge gives yd = 0
    t = _dense(ce.polygon_runs([0, 0, 4, 0, 0, 4], 5, 5), 5, 5)
    want = np.zeros((5, 5), bool)
    for x, n in enumerate([3, 2, 1, 0]):
        want[:n, x] = True
    np.testing.assert_array_equal(t, want)
    assert ce.runs_area(ce.polygon_runs([0, 0, 4, 0, 0, 4], 5, 5)) == 6


def test_polygon_crossing_the_edge_and_union():
    # a box hanging over the left and bottom edges is clipped to the image
    c = _dense(ce.polygon_runs([-3, 2, 3, 2, 3, 9, -3, 9], 6, 5), 6, 5)
    want = np.zeros((6, 5), bool)
    want[2:6, 0:3] = True
    np.testing.assert_array_equal(c, want)
    # two polygons of one annotation: the union of their masks
    a, b = [0, 0, 2, 0, 2, 2, 0, 2], [1, 1, 4, 1, 4, 4, 1, 4]
    ann = {"id": 1, "segmentation": [a, b]}
    u = _dense(ce.ann_to_runs(ann, 6, 6), 6, 6)
    np.testing.assert_array_equal(u, _dense(ce.polygon_runs(a, 6, 6), 6, 6) | _dense(ce.polygon_runs(b, 6, 6), 6, 6))


@pytest.mark.parametrize("seed", range(3))
def test_polygon_invariants(seed):
    rng = np.random.RandomState(seed)
    h, w = 40, 37
    ang = np.sort(rng.rand(7)) * 2 * np.pi
    r = 5 + rng.rand(7) * 12
    poly = np.stack([18 + r * np.cos(ang), 20 + r * np.sin(ang)], 1).ravel().tolist()
    base = _dense(ce.polygon_runs(poly, h, w), h, w)
    for k in range(1, 7):                                       # starting at another vertex gives the same mask
        rot = poly[2 * k:] + poly[:2 * k]
        np.testing.assert_array_equal(_dense(ce.polygon_runs(rot, h, w), h, w), base)
    assert 0 < base.sum() < h * w
    other = (np.asarray(poly) + 3).tolist()
    u = _dense(ce.merge_runs([ce.polygon_runs(poly, h, w), ce.polygon_runs(other, h, w)], h * w), h, w)
    np.testing.assert_array_equal(u, base | _dense(ce.polygon_runs(other, h, w), h, w))


def test_ann_to_runs_forms_and_refusals():
    cnts = [3, 4, 5, 2, 10]                                     # 24 = 4 x 6
    assert ce.ann_to_runs({"segmentation": {"size": [4, 6], "counts": cnts}}, 4, 6).tolist() == cnts
    assert ce.ann_to_runs({"segmentation": {"size": [4, 6], "counts": rle_to_string(cnts)}}, 4, 6).tolist() == cnts
    with pytest.raises(ValueError):
        ce.ann_to_runs({"id": 3, "segmentation": {"size": [6, 4], "counts": cnts}}, 4, 6)
    box = ce.ann_to_runs({"segmentation": [[1, 1, 2, 2]]}, 6, 6)         # 4 numbers: frBbox
    np.testing.assert_array_equal(_dense(box, 6, 6), _dense(ce.polygon_runs([1, 1, 1, 3, 3, 3, 3, 1], 6, 6), 6, 6))


def test_rle_ends_refusals():
    from hipie_b200 import ops
    ends, off = ops.rle_ends([[3, 4, 5], [0, 12]], 3, 4)
    assert ends.tolist() == [3, 7, 12, 0, 12] and off.tolist() == [0, 3, 5]
    with pytest.raises(ValueError, match="sums to"):
        ops.rle_ends([[3, 4, 4]], 3, 4)
    with pytest.raises(ValueError):
        ops.rle_ends([[13, -1]], 3, 4)


def test_limits_refused_in_the_library():
    import ctypes
    from hipie_b200 import _lib, build
    build.build()
    lib = _lib.load()
    fake = ctypes.c_void_p(16)
    assert lib.hipie_mask_pack(fake, 1025, 4, 4, fake, fake, None) == -1 and b"1024" in lib.hipie_last_error()
    assert lib.hipie_mask_pack(None, 3, 4, 4, fake, fake, None) == -1 and b"null" in lib.hipie_last_error()
    assert lib.hipie_mask_pack(fake, 3, 46341, 46341, fake, fake, None) == -1 and b"2^31" in lib.hipie_last_error()
    assert lib.hipie_mask_pack(None, 0, 4, 4, None, None, None) == 0
    assert lib.hipie_rle_expand(fake, fake, 4097, 4, 4, fake, fake, None) == -1 and b"4096" in lib.hipie_last_error()
    assert lib.hipie_rle_expand(fake, None, 2, 4, 4, fake, fake, None) == -1 and b"null" in lib.hipie_last_error()
    assert lib.hipie_rle_expand(None, None, 0, 4, 4, None, None, None) == 0
    assert lib.hipie_mask_overlaps(fake, 1025, fake, 1, 4, 4, fake, None) == -1
    assert lib.hipie_mask_overlaps(fake, 1, fake, 4097, 4, 4, fake, None) == -1
    assert lib.hipie_mask_overlaps(fake, 1, None, 1, 4, 4, fake, None) == -1 and b"null" in lib.hipie_last_error()
    assert lib.hipie_mask_overlaps(fake, 1, fake, 1, 0, 4, fake, None) == -1
    assert lib.hipie_mask_overlaps(None, 0, None, 5, 4, 4, None, None) == 0
    assert lib.hipie_mask_words(3, 100) == 16 and lib.hipie_mask_words(16, 16) == 8


def test_ops_refuse_without_launch():
    from hipie_b200 import ops
    with pytest.raises(ValueError):
        ops.mask_pack(torch.zeros(1025, 2, 2, dtype=torch.uint8))
    with pytest.raises(ValueError):
        ops.mask_overlaps(torch.zeros(1, 8, dtype=torch.int32), torch.zeros(4097, 8, dtype=torch.int32), 4, 4)
    with pytest.raises(ValueError):
        ops.mask_overlaps(torch.zeros(1, 7, dtype=torch.int32), torch.zeros(1, 8, dtype=torch.int32), 4, 4)
    bits, area = ops.mask_pack(torch.zeros(0, 5, 7, dtype=torch.uint8))
    assert bits.shape == (0, 8) and area.shape == (0,)
    assert ops.mask_overlaps(bits, torch.zeros(3, 8, dtype=torch.int32), 5, 7).shape == (0, 3)
    assert ops.rle_expand(torch.zeros(0, dtype=torch.int32), torch.zeros(1, dtype=torch.int64), 5, 7).shape == (0, 8)


# ------------------------------------------------------------------------------------------------------------------- evaluator


def test_presets_and_missing_instance_json(tmp_path, capsys):
    from test_evaluation_host import write_ade_panoptic_tree
    from hipie_b200.evaluation import PRESETS, COCOPanopticEvaluator, SemSegEvaluator, default_evaluators, load_records
    assert PRESETS["ade20k_panoptic_val"]["instances_json"] == "ade/ADEChallengeData2016/ade20k_instance_val.json"
    assert PRESETS["coco_2017_val_panoptic_with_sem_seg"]["instances_json"] == "coco/annotations/instances_val2017.json"
    write_ade_panoptic_tree(str(tmp_path), [(np.zeros((2, 2, 3), np.uint8), np.zeros((2, 2), np.int64), [], np.zeros((2, 2)))])
    recs, meta = load_records("ade20k_panoptic_val", str(tmp_path))
    evs = default_evaluators(meta, recs, labels_root=None)
    assert [type(e) for e in evs] == [COCOPanopticEvaluator, SemSegEvaluator]
    assert "not found" in capsys.readouterr().err
    js = {"images": [{"id": 1, "file_name": "ADE_val_00000000.jpg", "height": 2, "width": 2}], "annotations": [],
          "categories": [{"id": 1, "name": "person"}]}
    with open(meta["instances_json"], "w") as f:
        json.dump(js, f)
    evs = default_evaluators(meta, recs, labels_root=None)
    assert type(evs[0]).__name__ == "COCOInstanceEvaluator" and evs[0].class_names == ["person"]
    js["categories"].append({"id": 2, "name": "car"})
    with open(meta["instances_json"], "w") as f:
        json.dump(js, f)
    with pytest.raises(ValueError, match="thing classes"):
        default_evaluators(meta, recs, labels_root=None)


def _instance_json(path):
    js = {"images": [{"id": i, "file_name": f"im{i}.jpg", "height": 8, "width": 8} for i in (3, 1, 2)],
          "categories": [{"id": 4, "name": "a"}, {"id": 9, "name": "b"}],
          "annotations": [{"id": 1, "image_id": 1, "category_id": 4, "iscrowd": 0, "area": 16, "bbox": [0, 0, 4, 4],
                           "segmentation": [[0, 0, 4, 0, 4, 4, 0, 4]]},
                          {"id": 2, "image_id": 2, "category_id": 9, "iscrowd": 0, "area": 12, "bbox": [2, 2, 4, 3],
                           "segmentation": {"size": [8, 8], "counts": [18, 3, 5, 3, 5, 3, 5, 3, 19]}},
                          {"id": 3, "image_id": 3, "category_id": 4, "iscrowd": 1, "area": 64, "bbox": [0, 0, 8, 8],
                           "segmentation": {"size": [8, 8], "counts": [0, 64]}}]}
    with open(path, "w") as f:
        json.dump(js, f)
    return js


def _fake_image(ev, img_id, seed):
    """Feed _add_image as the device copy would: random predictions on an 8 x 8 image, intersections counted with numpy."""
    rng = np.random.RandomState(seed)
    anns = ev.anns.get(img_id, [])
    runs = [ce.ann_to_runs(a, 8, 8) for a in anns]
    gm = np.stack([_dense(r, 8, 8).ravel() for r in runs]) if runs else np.zeros((0, 64), bool)
    N = rng.randint(0, 5)
    pm = rng.rand(N, 64) < 0.4
    inter = (pm[:, None, :] & gm[None]).sum(-1).astype(np.int32)
    boxes = np.sort(rng.rand(N, 2, 2) * 8, axis=1).reshape(N, 4)[:, [0, 2, 1, 3]].astype(np.float32)
    ev._add_image(img_id, inter, pm.sum(1).astype(np.int32), boxes, rng.rand(N).astype(np.float32), rng.randint(0, 2, N) * 2 + 1,
                  [{"id": a["id"], "category_id": a["category_id"], "iscrowd": a["iscrowd"], "area": a["area"]} for a in anns],
                  [ce.runs_area(r) for r in runs], [a["bbox"] for a in anns])


def test_evaluator_refuses_unknown_class(tmp_path):
    from hipie_b200.evaluation import COCOInstanceEvaluator
    _instance_json(tmp_path / "i.json")
    ev = COCOInstanceEvaluator(str(tmp_path / "i.json"), {4: 1, 9: 3}, ["a", "b"], distributed=False)
    with pytest.raises(ValueError, match="class=2"):
        ev._add_image(1, np.zeros((1, 1), np.int32), np.ones(1, np.int32), np.zeros((1, 4), np.float32), np.ones(1, np.float32),
                      np.array([2]), [{"id": 1, "category_id": 4, "iscrowd": 0, "area": 16}], [16], [[0, 0, 4, 4]])
    ev.reset()
    res = ev.evaluate()
    assert set(res) == {"bbox", "segm"} and all(np.isnan(v) for v in res["segm"].values())


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _gloo_worker(rank, world, port, path, q):
    import torch.distributed as dist
    from hipie_b200.evaluation import COCOInstanceEvaluator
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ev = COCOInstanceEvaluator(path, {4: 1, 9: 3}, ["a", "b"])
    for img_id, seed in [(3, 0), (1, 1), (2, 2)][rank::world]:         # rank 0 gets images 3 and 2, rank 1 image 1
        _fake_image(ev, img_id, seed)
    q.put((rank, ev.evaluate()))
    dist.destroy_process_group()


def test_two_rank_gather_equals_single_process(tmp_path):
    import torch.multiprocessing as mp
    from hipie_b200.evaluation import COCOInstanceEvaluator
    path = str(tmp_path / "i.json")
    _instance_json(path)
    ev = COCOInstanceEvaluator(path, {4: 1, 9: 3}, ["a", "b"], distributed=False)
    for img_id, seed in [(3, 0), (1, 1), (2, 2)]:
        _fake_image(ev, img_id, seed)
    want = ev.evaluate()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, path, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=120) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
    assert res[1] is None
    for task in ("bbox", "segm"):
        assert list(res[0][task]) == list(want[task])
        np.testing.assert_array_equal(np.array(list(res[0][task].values())), np.array(list(want[task].values())))
