"""HIPIE_IMG meta-architecture on the CUDA engine — drop-in for the reference's
`META_ARCH_REGISTRY.get("HIPIE_IMG")(cfg)` (/root/reference/projects/HIPIE/hipie/hipie_img.py:45-420):
same constructor argument (a cfg node), same `forward(batched_inputs, do_postprocess=True)` contract, same
state_dict key names (modeling/params.py), same output dictionaries.

The forward path has no CPU fallback: the CUDA extension must be built and a CUDA device present.
"""
from collections import OrderedDict

import os

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from ..structures import Boxes, ImageList, Instances
from . import params as P
from .engine import Engine, inverse_sigmoid


def box_cxcywh_to_xyxy(x):
    x_c, y_c, w, h = x.unbind(-1)
    return torch.stack([(x_c - 0.5 * w), (y_c - 0.5 * h), (x_c + 0.5 * w), (y_c + 0.5 * h)], dim=-1)


def hp_from_cfg(cfg):
    """Translate the detectron2-style cfg (config.py: add_hipie_config + the MaskDINO yaml) into engine hyper-parameters."""
    m = cfg.MODEL
    hp = dict(hidden_dim=m.DDETRS.HIDDEN_DIM, enc_layers=m.DDETRS.ENC_LAYERS, dec_layers=m.DDETRS.DEC_LAYERS,
              dim_ff=m.DDETRS.DIM_FEEDFORWARD, num_queries=m.DDETRS.TWO_STAGE_NUM_PROPOSALS,
              num_bg=m.DDETRS.TWO_STAGE_NUM_BG_PROPOSALS, vl_hidden=m.DDETRS.VL_HIDDEN_DIM, lang_dim=m.LANGUAGE_BACKBONE.LANG_DIM,
              max_query_len=m.LANGUAGE_BACKBONE.MAX_QUERY_LEN, max_pool=bool(cfg.TEST.MAX_POOL),
              bg_cls_agnostic=bool(cfg.TEST.BG_CLS_AGNOSTIC),
              bert=dict(vocab=30522, hidden=768, layers=12, heads=12, inter=3072, max_pos=512))
    if m.BACKBONE.NAME == "D2ViT":
        dims = {"ViT-Base": (768, 12, 12), "ViT-Large": (1024, 24, 16), "ViT-huge": (1280, 32, 16)}[m.VIT.NAME]
        hp["backbone"] = "vit"
        hp["vit"] = dict(embed_dim=dims[0], depth=dims[1], num_heads=dims[2], window_size=14,
                         window_block_indexes=(0, 1, 3, 4, 6, 7, 9, 10), img_size=1024, patch_size=16, pretrain_img_size=224)
    else:
        hp["backbone"] = "r50"
    # inference settings (reference: hipie_img.py:56-133 reads the same keys); the engine implements the configuration every shipped
    # yaml uses and refuses the others instead of silently computing something else
    unsupported = []
    if not m.OTA:
        unsupported.append("MODEL.OTA=False (the non-NMS selection path)")
    if not m.PANO_TRANSFORM_EVAL:
        unsupported.append("MODEL.PANO_TRANSFORM_EVAL=False")
    if m.DDETRS.MASK_STRIDE != 4:
        unsupported.append(f"MODEL.DDETRS.MASK_STRIDE={m.DDETRS.MASK_STRIDE} (kernels are written for stride 4)")
    if not (m.DDETRS.USE_DINO and m.DDETRS.TWO_STAGE):
        unsupported.append("MODEL.DDETRS.USE_DINO / TWO_STAGE must be on")
    if m.DDETRS.NEW_MASK_HEAD or m.DDETRS.USE_RAFT or not m.DDETRS.USE_REL_COORD:
        unsupported.append("MODEL.DDETRS.NEW_MASK_HEAD / USE_RAFT / USE_REL_COORD=False")
    if getattr(m, "MODE_FREE_MATCHING_INFERENCE", False):
        unsupported.append("MODEL.MODE_FREE_MATCHING_INFERENCE")
    if getattr(cfg.TEST, "USE_BG_FOR_PANO_ON", False):
        unsupported.append("TEST.USE_BG_FOR_PANO_ON")
    if unsupported:
        raise NotImplementedError("hipie_b200.HIPIE_IMG does not implement: " + "; ".join(unsupported))
    hp.update(mask_stride=m.DDETRS.MASK_STRIDE, mask_thres=float(m.DDETRS.MASK_THRES), pano_temp=float(m.PANO_TEMPERATURE),
              object_mask_threshold=float(m.OBJECT_MASK_THRESHOLD), overlap_threshold=float(m.OVERLAP_THRESHOLD),
              pad_max=bool(m.LANGUAGE_BACKBONE.PAD_MAX), clip_enabled=bool(getattr(getattr(m, "CLIP", None), "ENABLED", False)))
    if hp["clip_enabled"]:               # hipie_img.py:249-262
        cl = m.CLIP
        hp.update(clip_name=str(cl.NAME), clip_alpha=float(cl.ALPHA), clip_beta=float(cl.BETA), clip_fg_a=float(cl.FG_IOU_A),
                  clip_fg_b=float(cl.FG_IOU_B), clip_agg_mode=str(cl.AGG_MODE), pano_temp_fg=float(m.PANO_TEMPERATURE_CLIP_FG))
    md = getattr(cfg, "_maskdino_cfg", None)
    if md is not None:
        hp.update(md_queries=md.MODEL.MaskDINO.NUM_OBJECT_QUERIES, md_dec_layers=md.MODEL.MaskDINO.DEC_LAYERS,
                  md_enc_layers=md.MODEL.SEM_SEG_HEAD.TRANSFORMER_ENC_LAYERS, md_dim_ff=md.MODEL.MaskDINO.DIM_FEEDFORWARD)
    else:
        hp.update(md_queries=300, md_dec_layers=9, md_enc_layers=6, md_dim_ff=2048)
    return hp


class HIPIE_IMG(nn.Module):
    """Unified open-vocabulary detection / segmentation / grounding model, inference only."""

    def __init__(self, cfg=None, hp=None, state_dict=None, device=None):
        super().__init__()
        if hp is None:
            hp = hp_from_cfg(cfg)
        self.cfg = cfg
        self.hp = hp
        self.device_ = torch.device(device or (cfg.MODEL.DEVICE if cfg is not None else "cuda"))
        if self.device_.type != "cuda":
            raise RuntimeError("hipie_b200.HIPIE_IMG runs on a CUDA (sm_90a) device only; there is no CPU path")
        self.demo_only = False
        self.num_bg, self.num_fg = hp.get("num_bg", 10), hp.get("num_queries", 900)
        self.mask_stride, self.mask_thres = hp.get("mask_stride", 4), hp.get("mask_thres", 0.5)
        self.pano_temp, self.object_mask_threshold = hp.get("pano_temp", 0.06), hp.get("object_mask_threshold", 0.25)
        self.overlap_threshold = hp.get("overlap_threshold", 0.8)
        self.tokenizer = None              # attached by the predictor, or loaded lazily from projects/HIPIE/bert-base-uncased
        self.fused_postprocess = True      # semantic/panoptic tensor work in one kernel (ops.seg_postprocess)
        self.use_cuda_graphs = False       # see enable_cuda_graphs()
        self.overlap_branches = os.environ.get("HIPIE_OVERLAP_BRANCHES", "1") != "0"   # DETR and MaskDINO branches on two streams (coco_inference)
        self._side_stream = None
        self._text_stream = None
        self.overlap_text = os.environ.get("HIPIE_OVERLAP_TEXT", "1") != "0"          # text encoder beside the backbone (forward_text_async)
        self._graphs = {}
        self.max_pool, self.bg_cls_agnostic, self.use_bg_for_pano = hp.get("max_pool", False), hp.get("bg_cls_agnostic", False), False
        # MaskCLIP re-scoring (MODEL.CLIP.ENABLED; hipie_img.py:249-262).  CLIP weights are never part of the HIPIE checkpoint
        # (open_vocab/clip.py:125-126): attach them with attach_clip(); until then an enabled config refuses to run.
        self.enable_clip = bool(hp.get("clip_enabled", False))
        self.clip, self.train_labels, self.clip_tokenize = None, None, None
        self.clip_alpha, self.clip_beta = hp.get("clip_alpha", 0.35), hp.get("clip_beta", 0.7)
        self.clip_fg_a, self.clip_fg_b = hp.get("clip_fg_a", 0.3), hp.get("clip_fg_b", 1.7)
        self.clip_agg_mode, self.pano_temp_fg = hp.get("clip_agg_mode", "MUL"), hp.get("pano_temp_fg", 0.06)
        self._sd = OrderedDict()
        self.engine = None
        if state_dict is None:
            state_dict = P.random_state_dict(hp, seed=0)
        self.load_state_dict(state_dict)

    @property
    def device(self):
        return self.device_

    # ---- checkpoint interface (reference key names)
    def state_dict(self, *a, **k):
        return OrderedDict(self._sd)

    def load_state_dict(self, sd, strict=True):
        spec = P.build_spec(self.hp)
        new = OrderedDict()
        for k, v in sd.items():
            c = P.canonical_name(k, self.hp)
            if c in spec.shapes:
                if tuple(v.shape) != spec.shapes[c]:
                    raise RuntimeError(f"size mismatch for {c}: {tuple(v.shape)} vs {spec.shapes[c]}")
                new.setdefault(c, v.detach().float().cpu())
        missing = [k for k in spec.shapes if k not in new]
        # keys the engine does not consume: aliases of shared modules are expected (decoder.bbox_embed.* == bbox_embed.* ...);
        # anything else is reported so a checkpoint of a different architecture does not load silently
        self.unexpected_keys = [k for k in sd if P.canonical_name(k, self.hp) not in spec.shapes]
        if strict and missing:
            raise RuntimeError(f"missing keys in state_dict: {missing[:8]} ... ({len(missing)})")
        if strict and self.unexpected_keys:
            raise RuntimeError(f"unexpected keys in state_dict: {self.unexpected_keys[:8]} ... ({len(self.unexpected_keys)})")
        self._sd = new
        self.engine = Engine(new, self.hp, self.device_)
        return missing

    # ---- stages
    def preprocess_image(self, batched_inputs):
        """hipie_img.py:880-898 + util/misc.py:288-316: the (x-mean)/std normalisation is fused into the patch kernel for the
        ViT path, so this only pads raw pixels; padded pixels must equal `mean` so that they normalise to 0."""
        imgs = [x["image"].to(self.device_, non_blocking=True).float() for x in batched_inputs]
        sizes = [tuple(i.shape[-2:]) for i in imgs]
        div = 32 if self.hp["backbone"] == "vit" else 0
        H, Wd = max(s[0] for s in sizes), max(s[1] for s in sizes)
        if div > 1:
            H, Wd = (H + div - 1) // div * div, (Wd + div - 1) // div * div
        mean = torch.tensor([123.675, 116.280, 103.530], device=self.device_).view(3, 1, 1)
        if all(s == (H, Wd) for s in sizes):
            tensor = torch.stack(imgs)
        else:
            tensor = mean.expand(3, H, Wd).unsqueeze(0).repeat(len(imgs), 1, 1, 1).contiguous()
            for i, im in enumerate(imgs):
                tensor[i, :, :im.shape[1], :im.shape[2]] = im
        mask = torch.ones(len(imgs), H, Wd, dtype=torch.bool, device=self.device_)
        for i, s in enumerate(sizes):
            mask[i, :s[0], :s[1]] = False
        return tensor, mask, sizes

    @torch.no_grad()
    def coco_inference(self, tensor, pad_mask, image_sizes, lang, task="detection", forced=None):
        """DDETRSegmUniDN.coco_inference (H/models/ddetrs_dn.py:801-978)."""
        forced = forced or {}
        eng, hp = self.engine, self.hp
        B = tensor.shape[0]
        feats = eng.vit(tensor) if hp["backbone"] == "vit" else eng.resnet50(tensor)
        if callable(lang):                 # text encoder launched on its own stream (forward_text_async): join here, after the backbone
            lang = lang()
        if task == "grounding":
            lm = lang["masks"].float()
            lang_feat_pool = ((lang["hidden"] * lm.unsqueeze(-1)).sum(1) / lm.sum(-1, keepdim=True)).unsqueeze(1)   # pre-fusion (:809-811)
        any_pad = any(tuple(s) != tuple(tensor.shape[-2:]) for s in image_sizes)      # host-side: no device sync
        # The MaskDINO branch (pixel decoder + 9 decoder layers + mask-embed) and the DETR branch (VL fusion, encoder, decoder, heads,
        # CondInst) only share the backbone features: they run on two streams, so the many small launches of the two decoders fill
        # each other's gaps (inside a CUDA-graph capture the fork / join becomes graph dependencies).
        if self.overlap_branches:
            cur = torch.cuda.current_stream(self.device_)
            if self._side_stream is None:
                self._side_stream = torch.cuda.Stream(device=self.device_)
            side = self._side_stream
            side.wait_stream(cur)
            with torch.cuda.stream(side):
                md = eng.maskdino(feats, B, forced_topk=forced.get("topk_md"))
            di = eng.detr_inputs(feats, pad_mask, B, any_pad=any_pad)
            tr = eng.detr_transformer(di, lang, B, forced_topk=forced.get("topk_fg"))
        else:
            di = eng.detr_inputs(feats, pad_mask, B, any_pad=any_pad)
            tr = eng.detr_transformer(di, lang, B, forced_topk=forced.get("topk_fg"))
            md = eng.maskdino(feats, B, forced_topk=forced.get("topk_md"))
        nd = hp.get("dec_layers", 6)
        lvl = nd - 1
        hs, hs_s = tr["hs"][lvl]
        Q = hs.shape[1]
        lang_for_cls = lang_feat_pool if task == "grounding" else tr["lang_hidden"]
        out = {}
        out["pred_logits"] = eng.vl_align(f"detr.detr.class_embed.{lvl}", hs_s.view(B * Q, 256), lang_for_cls, B, Q)
        out["pred_boxes"] = tr["refs"][lvl]          # == sigmoid(bbox_embed[lvl](hs[lvl]) + inverse_sigmoid(refs[lvl-1])) (:900-920)
        wi, bi = eng.W.lin(f"detr.detr.iou_head.{lvl}")
        out["pred_boxious"] = ops.gemm(hs_s.view(B * Q, 256), wi, bias=bi)[0].view(B, Q, 1)
        masks, mh_feats, params, ref_px = eng.condinst(tr["memory"], tr, di, image_sizes, B)
        out["pred_masks"] = masks.unsqueeze(2)
        if self.overlap_branches:
            torch.cuda.current_stream(self.device_).wait_stream(self._side_stream)      # join: everything below reads the MaskDINO outputs
        nqm = md["pred_logits_emb"].shape[1]
        ncls = hp.get("md_dec_layers", 9) + 2
        out["pred_logits_maskdino"] = eng.vl_align(f"detr.mask_dino_cls_embed.{ncls - 1}", md["pred_logits_emb_s"], lang_for_cls, B, nqm)
        out["pred_masks_maskdino"] = md["pred_masks"]
        out["pred_boxes_maskdino"] = md["pred_boxes"]
        out["aux"] = dict(enc_scores=tr["enc_scores"], topk=tr["topk"], md_enc_scores=md["enc_scores"], md_topk=md["topk"],
                          memory=tr["memory"], hs=[h[0] for h in tr["hs"]], refs=tr["refs"], mask_head_feats=mh_feats,
                          lang_hidden_fused=tr["lang_hidden"], feats={k: v[0] for k, v in feats.items()},
                          mask_bits=md["mask_bits"])
        return out

    def capture_hot_path(self, tensor, pad_mask, image_sizes, input_ids, attention_mask, task="detection", warmup=2, same_rows=None,
                         chunk_plan=None):
        """CUDA-graph the hot path (text encoder + coco_inference) for fixed-shape serving: ~2000 kernel launches per
        batch become one graph launch, which removes the host launch overhead.
        Returns `replay() -> out` whose tensors are static buffers; refill `tensor` / `input_ids` in place between replays."""
        from .. import _lib
        ids, am = input_ids.to(self.device_), attention_mask.to(self.device_)
        # whether all rows hold one prompt is part of the captured launch sequence (BERT on 1 row vs B rows): decided once,
        # before the capture, and baked in -- replaying with prompts of the other kind needs its own graph (see forward)
        if same_rows is None:
            same_rows = self.engine.rows_equal(input_ids, attention_mask)

        # prompts longer than 512 tokens: the cut positions are host logic on the token ids (bert_model.py:48-120), fixed before
        # the capture; replays refill chunk_plan.rows_d / masks_d in place (forward keys its graphs on the plan's signature)
        if chunk_plan is None:
            chunk_plan = self.engine.text_chunk_plan(input_ids, attention_mask, same_rows)

        def step():
            lang = self.forward_text_async(ids, am, same_rows=same_rows, chunk_plan=chunk_plan)
            return self.coco_inference(tensor, pad_mask, image_sizes, lang, task=task)

        side = torch.cuda.Stream(device=self.device_)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):          # populate weight / tensor-map / row-map caches outside the capture
                step()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        n0 = _lib.launch_count()
        with torch.cuda.graph(graph):
            out = step()
        launches = _lib.launch_count() - n0

        def replay():
            graph.replay()
            return out

        replay.launches_per_replay = launches
        replay.graph = graph
        replay.chunk_plan = chunk_plan
        return replay

    def enable_cuda_graphs(self, on=True):
        """Serving mode: `forward` replays one CUDA graph per (batch shape, image sizes, task) instead of ~2000 launches."""
        self.use_cuda_graphs = bool(on)
        if not on:
            self._graphs.clear()
        return self

    def _graphed_hot_path(self, tensor, pad_mask, image_sizes, ids, am, task, same_rows):
        plan = self.engine.text_chunk_plan(ids, am, same_rows)        # None unless the prompt exceeds 512 tokens
        key = (tuple(tensor.shape), tuple(ids.shape), task, bool(same_rows), tuple(tuple(int(v) for v in s) for s in image_sizes),
               None if plan is None else plan.signature)
        ent = self._graphs.get(key)
        if ent is None:
            if len(self._graphs) >= 4:           # static buffers are large; keep a handful of shapes
                self._graphs.pop(next(iter(self._graphs)))
            st = dict(tensor=tensor.clone(), pad=pad_mask.clone(), ids=ids.to(self.device_).clone(), am=am.to(self.device_).clone())
            st["replay"] = self.capture_hot_path(st["tensor"], st["pad"], image_sizes, st["ids"], st["am"], task=task, same_rows=same_rows,
                                                 chunk_plan=plan)
            self._graphs[key] = ent = st
        elif plan is not None:                   # same cut positions, possibly other tokens: refill the captured plan's buffers
            ent["replay"].chunk_plan.rows_d.copy_(plan.rows, non_blocking=True)
            ent["replay"].chunk_plan.masks_d.copy_(plan.masks, non_blocking=True)
        ent["tensor"].copy_(tensor)
        ent["pad"].copy_(pad_mask)
        ent["ids"].copy_(ids, non_blocking=True)
        ent["am"].copy_(am, non_blocking=True)
        return ent["replay"]()

    # ---- post-processing (hipie_img.py:537-766, 473-535, 870-878, 1025-1052); device-side torch glue for now ("next" tier, SURVEY §8f)
    def _pool_tables(self, positive_map, num_classes, Lt, is_thing, device):
        """Token->class pooling tables, built once per vocabulary (hipie_img.py:1025-1052 loops over the classes with host index
        tensors): a padded (C, maxlen) int32 token table + token counts (0 = class absent from the positive map -> score 0, as in
        the reference's zero-initialised `scores`) and the two -9999 masks (mode FG masks stuff classes, mode BG masks things)."""
        key = (tuple((k, tuple(v)) for k, v in sorted(positive_map.items())), num_classes, Lt, tuple(sorted(is_thing.items())))
        cache = self.__dict__.setdefault("_pool_cache", {})
        if key not in cache:
            if len(cache) > 8:
                cache.clear()
            maxlen = max(len(v) for v in positive_map.values())
            tok = torch.zeros(num_classes, maxlen, dtype=torch.int32)
            cnt = torch.zeros(num_classes, dtype=torch.int32)
            fg = torch.zeros(num_classes, dtype=torch.int8)
            bg = torch.zeros(num_classes, dtype=torch.int8)
            for label_j, toks in positive_map.items():
                if max(toks) >= Lt or min(toks) < 0:
                    raise ValueError(f"positive map token {toks} of class {label_j} outside the {Lt} text positions")
                tok[label_j - 1, :len(toks)] = torch.tensor(toks, dtype=torch.int32)
                tok[label_j - 1, len(toks):] = toks[0]
                cnt[label_j - 1] = len(toks)
                thing = bool(is_thing.get(label_j, True))
                fg[label_j - 1] = 0 if thing else 1
                bg[label_j - 1] = 1 if thing else 0
            cache[key] = (tok.to(device), cnt.to(device), fg.to(device), bg.to(device))
        return cache[key]

    # ---- MaskCLIP re-scoring (SURVEY a22 / f2; hipie_img.py:592-609, 735-747, 811-868; open_vocab/clip.py:243-383)
    def attach_clip(self, clip, train_labels, tokenize=None):
        """clip: a hipie_b200.modeling.maskclip.MaskCLIP or an open_clip state_dict; train_labels: the COCO-panoptic prompt-engineered
        label list the reference reads at hipie_img.py:72 (data.load_openseg_labels); tokenize: callable(list[str]) -> (N, ctx) int64
        CLIP token ids (open_clip.tokenize), needed unless the inputs carry `clip_prompt_ids`."""
        from .maskclip import MaskCLIP
        self.clip = clip if isinstance(clip, MaskCLIP) else MaskCLIP(clip, device=self.device_)
        self.train_labels, self.clip_tokenize = train_labels, tokenize
        self.enable_clip = True
        return self

    def _clip_tables(self, x):
        """prompt embeddings, prompt offsets per class and seen-class flags of one input's `open_seg_labels` (cached per label set)."""
        from .maskclip import class_tables
        if self.clip is None:
            raise RuntimeError("MODEL.CLIP.ENABLED is set but no CLIP weights are attached: call model.attach_clip(state_dict, train_labels)")
        test_labels = x.get("open_seg_labels")
        if test_labels is None:
            raise ValueError("MaskCLIP re-scoring needs `open_seg_labels` (list of {id, name}) in every input (hipie_img.py:347)")
        key = str(test_labels)
        prompts, seg, overlap = class_tables(test_labels, self.train_labels, self.device_)
        flat = [t for ls in prompts for t in ls]
        if key not in self.clip.cache_text:
            ids = x.get("clip_prompt_ids")
            if ids is None:
                if self.clip_tokenize is None:
                    raise RuntimeError("no CLIP tokenizer: pass tokenize= to attach_clip or put `clip_prompt_ids` into the inputs")
                ids = self.clip_tokenize(flat)
            if ids.shape[0] != len(flat):
                raise ValueError(f"clip_prompt_ids has {ids.shape[0]} rows for {len(flat)} prompts")
        else:
            ids = None
        text_unit, _ = self.clip.build_text_embed(ids, cache_key=key)
        return text_unit, seg, overlap

    def _clip_scores(self, x, masks, scores, temp, mode, iou=None, up=1, crop=None):
        """get_clip_logits (hipie_img.py:811-868) for one image: masks (Q, h, w) logits, scores (Q, C) class scores."""
        text_unit, seg, overlap = self._clip_tables(x)
        image01 = (x["image"].to(self.device_, torch.float32) / 255.0).contiguous()            # hipie_img.py:350-352
        emb = self.clip.get_mask_embed(image01, masks, up=up, crop=crop)
        raw = self.clip.raw_logits(emb, text_unit)
        return ops.clip_fuse(raw, emb, self.clip.logit_scale, seg, scores, temp, overlap, self.clip_alpha, self.clip_beta,
                             self.clip_agg_mode == "ADD", mode, iou=iou, fg_a=self.clip_fg_a, fg_b=self.clip_fg_b)

    def convert_grounding_to_od_logits(self, logits, num_classes, positive_map, is_thing, mode=None, max_pool=False, iou=None):
        """logits (bs, Q, Lt) -> scores (bs, Q, C): per-class mean (or max) over its token span, -9999 for masked classes; one kernel
        (ops.class_scores).  With `iou` (bs, Q, 1) also returns prob = sqrt(sigmoid(score) * sigmoid(iou)), its row max and argmax."""
        tok, cnt, fg, bg = self._pool_tables(positive_map, num_classes, logits.shape[-1], is_thing, logits.device)
        masked = fg if mode == "FG" else (bg if mode == "BG" else None)
        bs, Q, Lt = logits.shape
        sc, prob, rmax, rarg = ops.class_scores(logits.reshape(bs * Q, Lt), tok, cnt, masked=masked,
                                                iou=None if iou is None else iou.reshape(bs * Q), max_pool=max_pool, want_prob=iou is not None)
        if iou is None:
            return sc.view(bs, Q, num_classes)
        return sc.view(bs, Q, num_classes), prob.view(bs, Q, num_classes), rmax.view(bs, Q), rarg.view(bs, Q)

    def semantic_inference(self, mask_cls, mask_pred):
        return torch.einsum("qc,qhw->chw", mask_cls, mask_pred.sigmoid())

    def panoptic_inference(self, mask_cls, mask_pred, is_thing):
        scores, labels = mask_cls.max(-1)
        mask_pred = mask_pred.sigmoid()
        keep = scores > self.object_mask_threshold
        cur_scores, cur_classes, cur_masks = scores[keep], labels[keep], mask_pred[keep]
        cur_prob_masks = cur_scores.view(-1, 1, 1) * cur_masks
        h, w = cur_masks.shape[-2:]
        panoptic_seg = torch.zeros((h, w), dtype=torch.int32, device=cur_masks.device)
        segments_info = []
        current_segment_id = 0
        if cur_masks.shape[0] == 0:
            return panoptic_seg, segments_info
        cur_mask_ids = cur_prob_masks.argmax(0)
        K = cur_classes.shape[0]
        ids = torch.arange(K, device=cur_masks.device).view(K, 1, 1)
        own = cur_mask_ids.unsqueeze(0) == ids
        mask_area = own.flatten(1).sum(1)
        original_area = (cur_masks >= 0.5).flatten(1).sum(1)
        inter = (own & (cur_masks >= 0.5))
        inter_area = inter.flatten(1).sum(1)
        mask_area_c, original_area_c, inter_area_c, classes_c = mask_area.tolist(), original_area.tolist(), inter_area.tolist(), cur_classes.tolist()
        stuff_memory_list = {}
        for k in range(K):
            pred_class = classes_c[k]
            isthing = is_thing.get(int(pred_class + 1), True)
            if mask_area_c[k] > 0 and original_area_c[k] > 0 and inter_area_c[k] > 0:
                if mask_area_c[k] / original_area_c[k] < self.overlap_threshold:
                    continue
                if not isthing:
                    if int(pred_class) in stuff_memory_list:
                        panoptic_seg[inter[k]] = stuff_memory_list[int(pred_class)]
                        continue
                    stuff_memory_list[int(pred_class)] = current_segment_id + 1
                current_segment_id += 1
                panoptic_seg[inter[k]] = current_segment_id
                segments_info.append({"id": current_segment_id, "isthing": bool(isthing), "category_id": int(pred_class)})
        return panoptic_seg, segments_info

    def fused_sem_pano_launch(self, mask_cls, mask_low, image_size):
        """semantic_inference + the tensor part of panoptic_inference (hipie_img.py:880-1023) from the 1/4-resolution logits in
        one kernel (ops.seg_postprocess).  Returns the device-side handles; the segment merge (a short host loop over the kept
        queries) is finished by fused_sem_pano_finish once every image of the batch has been queued, so the device never idles
        on a per-image host round trip."""
        Hc, Wc = int(image_size[0]), int(image_size[1])
        sem, ids, areas, scores, labels = ops.seg_postprocess(mask_low, mask_cls, self.object_mask_threshold, Hc, Wc,
                                                              stride=self.mask_stride)
        host_d = torch.cat([areas, labels.to(torch.int32).unsqueeze(0), (scores > self.object_mask_threshold).to(torch.int32).unsqueeze(0)])
        return dict(sem=sem, ids=ids, host_d=host_d, Q=mask_cls.shape[0])

    def fused_sem_pano_finish(self, pend, host, is_thing):
        mask_area, original_area, inter_area, classes, keep = host.tolist()
        Q, ids = pend["Q"], pend["ids"]
        lut = [0] * (2 * Q + 1)           # ids+1 -> segment id (odd entries = argmax winner with sigmoid >= .5)
        segments_info, stuff_memory_list, current_segment_id = [], {}, 0
        for k in range(Q):
            if not keep[k]:
                continue
            pred_class = classes[k]
            isthing = is_thing.get(int(pred_class + 1), True)
            if mask_area[k] > 0 and original_area[k] > 0 and inter_area[k] > 0:
                if mask_area[k] / original_area[k] < self.overlap_threshold:
                    continue
                if not isthing:
                    if int(pred_class) in stuff_memory_list:
                        lut[2 * k + 2] = stuff_memory_list[int(pred_class)]
                        continue
                    stuff_memory_list[int(pred_class)] = current_segment_id + 1
                current_segment_id += 1
                lut[2 * k + 2] = current_segment_id
                segments_info.append({"id": current_segment_id, "isthing": bool(isthing), "category_id": int(pred_class)})
        lut_d = torch.tensor(lut, dtype=torch.int32, device=ids.device)
        panoptic_seg = lut_d[(ids + 1).long()]
        return pend["sem"], (panoptic_seg, segments_info)

    @torch.no_grad()
    def inference(self, out, image_sizes, positive_map, num_classes, task, is_thing, sizes, batched_inputs=None):
        """HIPIE_IMG.inference (hipie_img.py:537-766, OTA path): class pooling, sqrt(cls x iou), class-aware NMS and the flat
        top-100 run as kernels for the whole batch (ops.class_scores / batched_nms / topk); one device->host read of the kept
        counts sizes the per-image tensors."""
        max_num_inst = 100 if task == "detection" else 1
        fg = self.num_bg
        box_cls, box_pred = out["pred_logits"][:, fg:], out["pred_boxes"][:, fg:]
        mask_pred, iou_pred = out["pred_masks"][:, fg:], out["pred_boxious"][:, fg:]
        box_cls_bg = out["pred_logits_maskdino"]
        mask_pred_bg = out["pred_masks_maskdino"].unsqueeze(2)
        nimg = len(image_sizes)
        Qfg = box_cls.shape[1]
        # class scores / probabilities / NMS keys; images may carry different is_thing tables -> one launch per distinct table
        logits_fg, prob_all, nms_scores, idxs = [None] * nimg, [None] * nimg, [None] * nimg, [None] * nimg
        same_tables = all(is_thing[i] == is_thing[0] for i in range(nimg))
        groups = [list(range(nimg))] if same_tables else [[i] for i in range(nimg)]
        for grp in groups:
            has_thing = any(is_thing[grp[0]].values())
            sc, pr, rm, ra = self.convert_grounding_to_od_logits(box_cls[grp[0]:grp[-1] + 1], num_classes, positive_map, is_thing[grp[0]],
                                                                 mode="FG" if has_thing else None, max_pool=self.max_pool,
                                                                 iou=iou_pred[grp[0]:grp[-1] + 1])
            for j, i in enumerate(grp):
                logits_fg[i], prob_all[i], nms_scores[i], idxs[i] = sc[j], pr[j], rm[j], ra[j]
                if self.enable_clip:
                    # hipie_img.py:592-609: the foreground scores become sqrt(sigmoid(fused)^a * sigmoid(iou)^b) on thing classes, fused =
                    # MaskCLIP's class probabilities of the 1/4-resolution masks ensembled with softmax(sigmoid(score) / T_fg)
                    temp = self.pano_temp_fg if num_classes > 1 else 0.0
                    prob_all[i], nms_scores[i], idxs[i] = self._clip_scores(batched_inputs[i], mask_pred[i][:, 0], sc[j], temp, 1,
                                                                            iou=iou_pred[i].reshape(-1))
        keep_all, nkeep = ops.batched_nms(box_pred, torch.stack(nms_scores), torch.stack(idxs), 0.7)
        nk_host = nkeep.tolist()                       # the one host read of the selection stage
        results = []
        for i in range(nimg):
            image_size = image_sizes[i]
            logits_per_image = logits_fg[i]
            keep_indices = keep_all[i, :nk_host[i]].long()
            prob = prob_all[i][keep_indices]
            num_inst = min(max_num_inst, prob.numel())
            box_k, mask_k = box_pred[i][keep_indices], mask_pred[i][keep_indices]
            topk_values, topk_indexes = ops.topk(prob.view(1, -1), num_inst)
            topk_values, topk_indexes = topk_values[0], topk_indexes[0].long()
            topk_boxes = torch.div(topk_indexes, logits_per_image.shape[1], rounding_mode="floor")
            labels = topk_indexes % logits_per_image.shape[1]
            box_k, mask_i = box_k[topk_boxes], mask_k[topk_boxes]
            result = Instances(image_size)
            result.pred_boxes = Boxes(box_cxcywh_to_xyxy(box_k))
            result.pred_boxes.scale(scale_x=image_size[1], scale_y=image_size[0])
            N, C, H, Wd = mask_i.shape
            if self.fused_postprocess and self.mask_stride == 4:
                result.pred_masks = ops.upsample_threshold(mask_i[:, 0], self.mask_thres, int(image_size[0]), int(image_size[1])).unsqueeze(1)
            else:
                m = F.interpolate(mask_i, size=(H * self.mask_stride, Wd * self.mask_stride), mode="bilinear", align_corners=False)
                result.pred_masks = (m.sigmoid() > self.mask_thres)[:, :, :image_size[0], :image_size[1]]
            result.scores = topk_values
            result.pred_classes = labels
            sem = None
            pano = (None, None)
            if task == "detection":
                mode = None if (self.use_bg_for_pano or self.bg_cls_agnostic) else "BG"
                logits_bg = self.convert_grounding_to_od_logits(box_cls_bg[i].unsqueeze(0), num_classes, positive_map, is_thing[i],
                                                                mode=mode, max_pool=self.max_pool)[0]
                logits_all = torch.cat([logits_per_image[keep_indices], logits_bg], dim=0)
                mask_all = torch.cat([mask_pred[i][keep_indices], mask_pred_bg[i]], dim=0)
                N, C, H, Wd = mask_all.shape
                if self.enable_clip:
                    # hipie_img.py:735-747: class probabilities = softmax of the fused log-probabilities; MaskCLIP sees the x4-upsampled,
                    # cropped masks (evaluated on the fly by the patch-mask kernel)
                    logits_all = self._clip_scores(batched_inputs[i], mask_all[:, 0], logits_all, self.pano_temp, 2, up=self.mask_stride,
                                                   crop=image_size)
                else:
                    logits_all = F.softmax(logits_all.sigmoid() / self.pano_temp, dim=-1)
                if (self.fused_postprocess and self.mask_stride == 4 and N <= 8192 and tuple(sizes[i]) == tuple(image_size)):
                    pend = self.fused_sem_pano_launch(logits_all, mask_all[:, 0], image_size)
                    results.append(dict(instances=result, panoptic_seg=None, sem_seg=None, _pending=pend))
                    continue
                mask_all = F.interpolate(mask_all, size=(H * self.mask_stride, Wd * self.mask_stride), mode="bilinear", align_corners=False)
                mask_all = mask_all[:, :, :image_size[0], :image_size[1]]
                if tuple(mask_all.shape[-2:]) == tuple(sizes[i]):
                    mask_up = mask_all[:, 0]          # same size: the bilinear resize is the identity
                else:
                    mask_up = F.interpolate(mask_all, size=sizes[i], mode="bilinear", align_corners=False)[:, 0]
                sem = self.semantic_inference(logits_all, mask_up)
                pano = self.panoptic_inference(logits_all, mask_up, is_thing[i])
            results.append(dict(instances=result, panoptic_seg=pano, sem_seg=sem))
        pending = [(i, r.pop("_pending")) for i, r in enumerate(results) if "_pending" in r]
        if pending:
            # one device->host copy of all images' area counters / labels (pinned, after every kernel has been queued)
            sizes_q = [p["host_d"].shape[1] for _, p in pending]
            host_all = torch.cat([p["host_d"] for _, p in pending], dim=1).cpu()
            off = 0
            for (i, p), nq in zip(pending, sizes_q):
                sem, pano = self.fused_sem_pano_finish(p, host_all[:, off:off + nq], is_thing[i])
                off += nq
                results[i]["sem_seg"], results[i]["panoptic_seg"] = sem, pano
        return results

    @staticmethod
    def segmentation_postprocess(results, output_height, output_width):
        """H/models/ddetrs.py:1029-1076"""
        sx, sy = output_width / results.image_size[1], output_height / results.image_size[0]
        out = Instances((output_height, output_width))
        boxes = Boxes(results.pred_boxes.tensor.clone())
        boxes.scale(sx, sy)
        boxes.clip((output_height, output_width))
        keep = boxes.nonempty()
        out.pred_boxes = Boxes(boxes.tensor[keep])
        if tuple(results.pred_masks.shape[-2:]) == (output_height, output_width):
            m0 = results.pred_masks[:, 0]                                # nearest resize to the same size is the identity;
            masks = m0.view(torch.uint8) if m0.dtype == torch.bool and m0.is_contiguous() else m0.to(torch.uint8)   # bool bytes ARE uint8 0/1
        else:
            masks = F.interpolate(results.pred_masks.float(), size=(output_height, output_width), mode="nearest")[:, 0].to(torch.uint8)
        out.pred_masks = masks[keep]
        out.scores = results.scores[keep]
        out.pred_classes = results.pred_classes[keep]
        return out

    def forward_text_async(self, input_ids, attention_mask, same_rows=None, chunk_plan=None):
        """The text encoder does not depend on the image: launch it on a second stream so that its ~100 small kernels run beside the
        backbone, and hand back a join() that makes the current stream wait for it and returns the features (coco_inference calls
        it after the backbone).  With overlap_branches off this is the plain synchronous call."""
        if same_rows is None:
            same_rows = self.engine.rows_equal(input_ids, attention_mask)
        ids, am = input_ids.to(self.device_), attention_mask.to(self.device_)
        if not (self.overlap_branches and self.overlap_text):
            return self.engine.forward_text(ids, am, same_rows=same_rows, chunk_plan=chunk_plan)
        cur = torch.cuda.current_stream(self.device_)
        if self._text_stream is None:
            self._text_stream = torch.cuda.Stream(device=self.device_)
        side = self._text_stream
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            lang = self.engine.forward_text(ids, am, same_rows=same_rows, chunk_plan=chunk_plan)

        def join():
            torch.cuda.current_stream(self.device_).wait_stream(side)
            return lang
        return join

    def forward_text(self, input_ids, attention_mask, same_rows=None):
        if same_rows is None:
            same_rows = self.engine.rows_equal(input_ids, attention_mask)     # host tensors: compared on the host
        return self.engine.forward_text(input_ids.to(self.device_), attention_mask.to(self.device_), same_rows=same_rows)

    @torch.no_grad()
    def forward(self, batched_inputs, do_postprocess=True, forced=None, return_raw=False):
        """batched_inputs: list[dict] with image (3,H,W) 0..255, height, width, task, is_thing, positive_map_label_to_token and
        either `expressions` (str; needs a tokenizer attached via `self.tokenizer`) or pre-tokenised `input_ids`/`attention_mask`."""
        task_list = [x["task"] for x in batched_inputs]
        assert len(set(task_list)) == 1
        task = task_list[0]
        if task not in ("detection", "grounding"):
            raise ValueError("task must be detection or grounding")
        tensor, pad_mask, image_sizes = self.preprocess_image(batched_inputs)
        positive_map = {1: [0]} if task == "grounding" else batched_inputs[0]["positive_map_label_to_token"]
        num_classes = len(positive_map)
        if "input_ids" in batched_inputs[0]:
            ids = torch.stack([x["input_ids"] for x in batched_inputs])
            am = torch.stack([x["attention_mask"] for x in batched_inputs])
        else:
            if self.tokenizer is None:      # hipie_img.py:153: AutoTokenizer.from_pretrained('projects/HIPIE/bert-base-uncased')
                from ..data import load_tokenizer
                self.tokenizer = load_tokenizer()          # raises with the searched paths when the vocabulary is absent
            from ..data import tokenize_captions
            ids, am, _ = tokenize_captions(self.tokenizer, [x["expressions"] for x in batched_inputs], self.hp["max_query_len"],
                                           pad_max=self.hp.get("pad_max", True))
        same_rows = self.engine.rows_equal(ids, am)      # one prompt for the whole batch? (decided on the values, every call)
        if self.use_cuda_graphs and forced is None:
            out = self._graphed_hot_path(tensor, pad_mask, image_sizes, ids, am, task, same_rows)
        else:
            lang = self.forward_text_async(ids, am, same_rows=same_rows)
            out = self.coco_inference(tensor, pad_mask, image_sizes, lang, task=task, forced=forced)
        is_thing = [x["is_thing"] for x in batched_inputs]
        sizes = [(x.get("height", s[0]), x.get("width", s[1])) for x, s in zip(batched_inputs, image_sizes)]
        if self.enable_clip and self.clip is None:
            raise RuntimeError("MODEL.CLIP.ENABLED is set but no CLIP weights are attached: call model.attach_clip(state_dict, train_labels)")
        results = self.inference(out, image_sizes, positive_map, num_classes, task, is_thing, sizes, batched_inputs=batched_inputs)
        if do_postprocess:
            for r, x, s in zip(results, batched_inputs, image_sizes):
                r["instances"] = self.segmentation_postprocess(r["instances"], x.get("height", s[0]), x.get("width", s[1]))
        return (results, out) if return_raw else results
