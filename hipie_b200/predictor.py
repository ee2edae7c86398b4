"""HIPIEPredictor on the CUDA engine: same constructor and call signature as the reference's demo / evaluation predictor
(/root/reference/projects/HIPIE/predictor.py:245-372): takes one BGR uint8 image (cv2 layout), converts it per cfg.INPUT.FORMAT,
applies ResizeShortestEdge(MIN_SIZE_TEST, MAX_SIZE_TEST), builds the caption and the label -> token map for the requested
vocabulary (detection) or takes the referring expression (grounding), and runs `model([inputs])[0]`.
"""
import numpy as np
import torch

from .data import ResizeShortestEdge, create_queries_and_maps, get_openseg_labels, load_tokenizer
from .registry import DetectionCheckpointer, build_model


def cat2ind(categories):
    """hipie/data/coco_dataset_mapper_uni.py:30-40"""
    ind_to_class = {0: "__background__"}
    index = 1
    for x in categories:
        isthing = x["isthing"] if "isthing" in x else 1
        if isthing == 1:
            ind_to_class[index] = x["name"]
            index += 1
    return ind_to_class


class HIPIEPredictor:
    def __init__(self, cfg, test_categories=None, tokenizer=None, model=None, labels_root=None):
        """`tokenizer` / `model` / `labels_root` are additions for offline use (a tokenizer object, an already built HIPIE_IMG, the
        directory of the reference's openseg label files); with the defaults the behaviour is the reference's: model from cfg,
        weights from cfg.MODEL.WEIGHTS, tokenizer from projects/HIPIE/bert-base-uncased."""
        self.cfg = cfg.clone() if hasattr(cfg, "clone") else cfg
        self.model = model if model is not None else build_model(self.cfg)
        self.model.eval()
        if model is None and getattr(cfg.MODEL, "WEIGHTS", ""):
            DetectionCheckpointer(self.model).load(cfg.MODEL.WEIGHTS)
        self.aug = ResizeShortestEdge([cfg.INPUT.MIN_SIZE_TEST, cfg.INPUT.MIN_SIZE_TEST], cfg.INPUT.MAX_SIZE_TEST)
        self.input_format = cfg.INPUT.FORMAT
        assert self.input_format in ["RGB", "BGR"], self.input_format
        self.tokenizer = tokenizer if tokenizer is not None else load_tokenizer()
        if getattr(self.model, "tokenizer", None) is None:
            self.model.tokenizer = self.tokenizer
        self.labels_root = labels_root
        self.prompt_test_dict, self.positive_map_label_to_token_dict, self.is_thing = {}, {}, {}
        if test_categories is not None:
            prompt_test, pos_map = create_queries_and_maps(test_categories, self.tokenizer)
            self.prompt_test_dict["custom"] = prompt_test
            self.positive_map_label_to_token_dict["custom"] = pos_map
            self.is_thing["custom"] = {i + 1: bool(c.get("isthing", 1)) for i, c in enumerate(test_categories)}
        else:
            for dataset_name in ("coco_panoptic", "ade20k_150", "coco"):
                try:
                    cats = get_openseg_labels(dataset_name, root=labels_root)
                except FileNotFoundError:
                    continue
                prompt_test, pos_map = create_queries_and_maps(cats, self.tokenizer)
                self.prompt_test_dict[dataset_name] = prompt_test
                self.positive_map_label_to_token_dict[dataset_name] = pos_map
                self.is_thing.setdefault(dataset_name, {k: True for k in pos_map})

    def _vocabulary(self, dataset_name, test_categories, test_is_thing):
        if test_categories is not None:
            expressions, pos_map = create_queries_and_maps(test_categories, self.tokenizer)
            is_thing = test_is_thing if test_is_thing is not None else {i + 1: bool(c.get("isthing", 1)) for i, c in enumerate(test_categories)}
            return expressions, pos_map, is_thing
        if dataset_name not in self.prompt_test_dict and "custom" in self.prompt_test_dict:
            dataset_name = "custom"
        expressions = self.prompt_test_dict[dataset_name]
        pos_map = self.positive_map_label_to_token_dict[dataset_name]
        is_thing = self.is_thing.get(dataset_name, self.is_thing.get("coco", {k: True for k in pos_map}))
        return expressions, pos_map, is_thing

    def __call__(self, original_image, task, expressions=None, test_categories=None, open_seg_labels=None, test_is_thing=None,
                 dataset_name="coco"):
        with torch.no_grad():
            if self.input_format == "RGB":
                original_image = original_image[:, :, ::-1]      # the model expects RGB, the caller hands BGR
            height, width = original_image.shape[:2]
            image = self.aug.apply_image(np.ascontiguousarray(original_image))
            image = torch.as_tensor(image.astype("float32").transpose(2, 0, 1))
            if task == "detection":
                expressions, pos_map, is_thing = self._vocabulary(dataset_name, test_categories, test_is_thing)
                inputs = {"image": image, "height": height, "width": width, "task": task, "expressions": expressions, "is_thing": is_thing,
                          "positive_map_label_to_token": pos_map, "open_seg_labels": open_seg_labels}
            elif task == "grounding":
                assert expressions is not None
                inputs = {"image": image, "height": height, "width": width, "task": task, "expressions": expressions, "is_thing": {1: True}}
            else:
                raise ValueError("""Unsupported task. task must be in ["detection", "grounding", "sot"]""")
            return self.model([inputs])[0]
