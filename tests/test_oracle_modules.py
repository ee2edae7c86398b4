"""CPU: the oracle's module-level restatements against outputs of the REAL reference modules
(oracle/gen_golden_modules.py ran the unmodified files of /root/reference in the build container; see its docstring and
tests/golden/MANIFEST.md for what each fixture pins).  Weights are re-created by name with hipie_oracle.synth.fill_by_name_,
so every test also checks that the oracle module exposes exactly the reference's parameter names and shapes."""
import copy
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

from hipie_oracle import detr, maskdino, vit
from hipie_oracle.synth import fill_by_name_


def _unpack(v):
    """Fixtures keep 0/1 masks as packed bits ({"packed_bits_of_shape", "dtype", "bits"}): restored to the stored tensor."""
    if isinstance(v, dict) and "packed_bits_of_shape" in v:
        shape = v["packed_bits_of_shape"]
        n = 1
        for d in shape:
            n *= d
        bits = torch.from_numpy(np.unpackbits(v["bits"].numpy())[:n].copy())
        return bits.reshape(shape).to(getattr(torch, v["dtype"]))
    if isinstance(v, dict):
        return {k: _unpack(x) for k, x in v.items()}
    if isinstance(v, list):
        return [_unpack(x) for x in v]
    if isinstance(v, tuple):
        return tuple(_unpack(x) for x in v)
    return v


def _load(golden_dir, name):
    p = os.path.join(golden_dir, name)
    if not os.path.exists(p):
        pytest.skip(f"{name} not generated")
    return _unpack(torch.load(p))


def _close(actual, ref, atol):
    """allclose against a stored reference tensor, or against a fixed seeded sample of its elements ({"sample_of_shape", "idx",
    "values"}: large outputs are stored that way to keep the fixtures small)."""
    if isinstance(ref, dict):
        assert tuple(actual.shape) == tuple(ref["sample_of_shape"]), (actual.shape, ref["sample_of_shape"])
        actual, ref = actual.reshape(-1)[ref["idx"].long()], ref["values"]
    err = (actual - ref).abs().max()
    assert torch.allclose(actual, ref, atol=atol), err


def _same_keys(module, keys):
    mine = sorted(module.state_dict().keys())
    assert mine == sorted(keys), (sorted(set(mine) ^ set(keys))[:10])


def test_vit_forward_matches_reference(golden_dir):
    """backbone/vit.py ViT.forward: patch embed + bicubic abs-pos + windowed/global blocks with decomposed rel-pos + FPN"""
    g = _load(golden_dir, "ref_vit.pt")
    m = vit.ViT(**g["kw"]).eval()
    _same_keys(m, g["keys"])
    fill_by_name_(m, g["seed"])
    with torch.no_grad():
        out = m(g["x"])
    for k in ("res3", "res4", "res5"):
        ref = g["out"][k]          # fp32 rounding only: 1e-5 of the feature range
        assert (out[k] - ref).abs().max() < 1e-5 * ref.abs().max() + 1e-5, (k, (out[k] - ref).abs().max(), ref.abs().max())


def _oracle_transformer(kw):
    tr = detr.DeformableTransformerVLDINO(**kw)
    d, nd = kw["d_model"], kw["num_decoder_layers"]
    class_embed = detr.VL_Align(kw["lang_dim"], d)
    bbox_embed = detr.MLP(d, d, 4, 3)
    tr.decoder.class_embed = nn.ModuleList([copy.deepcopy(class_embed) for _ in range(nd + 1)])
    tr.decoder.bbox_embed = nn.ModuleList([copy.deepcopy(bbox_embed) for _ in range(nd + 1)])
    tr.decoder.class_embed[-1] = detr.Still_Classifier(d)
    return tr


def test_transformer_forward_matches_reference(golden_dir):
    """deformable_transformer_dino.py DeformableTransformerVLDINO.forward with padded inputs: VL fusion, 2 encoder layers
    (MSDeformAttn.forward), two-stage proposals + top-k, bg queries, 2 decoder layers, intermediate reference points"""
    g = _load(golden_dir, "ref_transformer.pt")
    tr = _oracle_transformer(g["kw"]).eval()
    _same_keys(tr, g["keys"])
    fill_by_name_(tr, g["seed"])
    lang = {k: v.clone() for k, v in g["lang"].items()}
    with torch.no_grad():
        hs, memory, init_ref, inter_refs, lang_out, aux = tr(g["srcs"], g["masks"], g["poses"], lang)
    _close(memory, g["memory"], 2e-5)
    assert torch.allclose(lang_out["hidden"], g["lang_hidden"], atol=2e-5)
    assert torch.allclose(aux["enc_scores"], g["enc_cls"][..., 0], atol=2e-5)
    assert torch.allclose(init_ref, g["init_ref"], atol=1e-5)
    assert torch.allclose(hs, g["hs"], atol=5e-5), (hs - g["hs"]).abs().max()
    assert torch.allclose(inter_refs, g["inter_refs"], atol=1e-5)


def test_heads_match_reference(golden_dir):
    """deformable_detr.py VL_Align.forward (normalise, /2, projection, per-token bias, exp(log_scale), clamp) and MLP"""
    g = _load(golden_dir, "ref_heads.pt")
    va = fill_by_name_(detr.VL_Align(768, 256), g["va_seed"]).eval()
    with torch.no_grad():
        va.log_scale.fill_(0.3)
        assert torch.allclose(va(g["q"], g["emb"]), g["va_out"], atol=1e-5)
        mlp = fill_by_name_(detr.MLP(256, 256, 4, 3), g["mlp_seed"]).eval()
        assert torch.allclose(mlp(g["q"]), g["mlp_out"], atol=1e-5)


def test_maskdino_encoder_decoder_match_reference(golden_dir):
    """maskdino_encoder.py MaskDINOEncoder.forward_features (input_proj + GN, 2 MSDeformAttn encoder layers, FPN level on res3,
    mask_features head) and maskdino_decoder.py MaskDINODecoder.forward (coarse->fine re-flattening, two-stage top-k, 3 DINO decoder
    layers, double decoder_norm, mask-embed einsum, box refinement)"""
    g = _load(golden_dir, "ref_maskdino.pt")
    enc = maskdino.MaskDINOEncoder(g["in_channels"], conv_dim=256, mask_dim=256, enc_layers=2, dim_ff=48, nheads=8).eval()
    _same_keys(enc, g["enc_keys"])
    fill_by_name_(enc, g["enc_seed"])
    with torch.no_grad():
        mf, out0, ms = enc.forward_features(g["feats"])
    _close(mf, g["mask_features"], 2e-5)
    assert len(ms) == len(g["multi_scale"])
    for a, b in zip(ms, g["multi_scale"]):
        _close(a, b, 2e-5)
    dec = maskdino.MaskDINODecoder(hidden_dim=256, num_queries=7, nheads=8, dim_feedforward=48, dec_layers=3, mask_dim=256, num_classes=256).eval()
    _same_keys(dec, g["dec_keys"])
    fill_by_name_(dec, g["dec_seed"])
    with torch.no_grad():
        out = dec(ms, mf)          # the encoder outputs just checked against the reference's (the fixture keeps a sample of them)
    assert torch.allclose(out["pred_logits"], g["pred_logits"], atol=5e-5)
    assert torch.allclose(out["pred_boxes"], g["pred_boxes"], atol=1e-5)
    assert torch.allclose(out["interm_masks"], g["interm_masks"], atol=1e-4)
    ref = g["pred_masks"]
    assert (out["pred_masks"] - ref).abs().max() < 1e-5 * ref.abs().max() + 1e-4, (out["pred_masks"] - ref).abs().max()


def test_condinst_matches_reference(golden_dir):
    """ddetrs_dn.py MaskHeadSmallConv.forward, DDETRSegmUniDN.dynamic_mask_with_coords (+ mask_heads_forward, parse_dynamic_params),
    compute_locations, aligned_bilinear"""
    from hipie_oracle import condinst
    from hipie_oracle.model import MaskHeadSmallConv
    g = _load(golden_dir, "ref_condinst.pt")
    head = MaskHeadSmallConv(256).eval()
    _same_keys(head, g["head_keys"])
    fill_by_name_(head, g["head_seed"])
    with torch.no_grad():
        decod = head(g["enc"])
        assert torch.allclose(decod, g["decod"], atol=1e-5)
        logits = condinst.dynamic_mask_with_coords(g["decod"], g["ref_px"], g["params"], stride=8)
    ref = g["logits"]
    assert (logits - ref).abs().max() < 1e-5 * ref.abs().max() + 1e-5, ((logits - ref).abs().max(), ref.abs().max())
    assert torch.equal(condinst.aligned_bilinear(g["ab_in"], 2), g["ab_out"])
    assert torch.equal(condinst.compute_locations(3, 4, stride=8), g["locations"])


def test_bert_encoder_chunk_path_matches_reference(golden_dir):
    """bert_model.py BertEncoder.forward: <= 512 tokens straight through HF BertModel; 1305 tokens through the chunking at
    '.' / EOS boundaries with [CLS] re-insertion and scatter back (:68-135)"""
    from hipie_oracle.model import BertEncoder
    g = _load(golden_dir, "ref_bert_chunk.pt")
    enc = BertEncoder({"bert": g["bert"]}).eval()
    mine = sorted(k for k in enc.state_dict().keys())
    assert mine == sorted(g["keys"]), sorted(set(mine) ^ set(g["keys"]))[:10]
    fill_by_name_(enc, g["seed"])
    with torch.no_grad():
        long = enc({"input_ids": g["ids"], "attention_mask": g["am"]}, sep=1012)
        short = enc({"input_ids": g["ids2"], "attention_mask": g["am2"]}, sep=1012)
    assert torch.allclose(short["hidden"], g["hidden_short"], atol=1e-5)
    _close(long["hidden"], g["hidden_long"], 1e-5)


def test_postprocessing_matches_reference_inference(golden_dir):
    """hipie_img.py HIPIE_IMG.inference (class pooling mean / max, FG / BG masking, sqrt(cls x iou), batched NMS 0.7, flat top-100,
    x4 bilinear upsample + sigmoid > 0.5, softmax(sigmoid / 0.06), second resize, semantic einsum, panoptic merge incl. stuff merging)
    and ddetrs.py segmentation_postprocess, both variants of the shipped yamls"""
    import types
    from hipie_oracle.model import HipieOracle
    g = _load(golden_dir, "ref_postproc.pt")
    pool = g["pool"]
    assert torch.equal(HipieOracle.convert_grounding_to_od_logits(pool["logits"], g["num_classes"], g["pos_map"], g["is_thing"], mode="FG"), pool["mean_fg"])
    assert torch.equal(HipieOracle.convert_grounding_to_od_logits(pool["logits"], g["num_classes"], g["pos_map"], g["is_thing"], mode="BG", max_pool=True),
                       pool["max_bg"])
    for tag, v in g["variants"].items():
        fake = types.SimpleNamespace(num_bg=g["nbg"], num_fg=g["nfg"], mask_stride=4, mask_thres=0.5, pano_temp=0.06, object_mask_threshold=0.25,
                                     overlap_threshold=0.8, max_pool=v["max_pool"], use_bg_for_pano=False, bg_cls_agnostic=v["bg_cls_agnostic"], clip=None)
        fake.convert_grounding_to_od_logits = HipieOracle.convert_grounding_to_od_logits
        fake.semantic_inference = lambda *a, f=fake: HipieOracle.semantic_inference(f, *a)
        fake.panoptic_inference = lambda *a, f=fake: HipieOracle.panoptic_inference(f, *a)
        res = HipieOracle.inference(fake, {k: t.clone() for k, t in g["out"].items()}, g["image_sizes"], g["pos_map"], g["num_classes"], "detection",
                                    [g["is_thing"], g["is_thing"]], g["sizes"])
        for r, ref, isz, (oh, ow) in zip(res, v["results"], g["image_sizes"], g["sizes"]):
            inst = r["instances"]
            assert torch.equal(inst["pred_classes"], ref["pred_classes"]), tag
            assert torch.allclose(inst["scores"], ref["scores"], atol=1e-6)
            assert torch.allclose(inst["pred_boxes"], ref["pred_boxes"], atol=1e-4)
            assert torch.equal(inst["pred_masks"], ref["pred_masks"])
            post = HipieOracle.segmentation_postprocess(inst, isz, oh, ow)
            assert torch.allclose(post["pred_boxes"], ref["post_boxes"], atol=1e-4)
            assert torch.equal(post["pred_masks"], ref["post_masks"]) and torch.equal(post["pred_classes"], ref["post_classes"])
            _close(r["sem_seg"], ref["sem_seg"], 1e-5)
            assert torch.equal(r["panoptic_seg"][0], ref["panoptic_seg"])
            assert r["panoptic_seg"][1] == ref["segments_info"] and len(ref["segments_info"]) > 0


def test_resnet50_matches_reference(golden_dir):
    """detectron2 ResNet-50 (BasicStem, 16 BottleneckBlocks with FrozenBatchNorm2d, stride in the 3x3) on a 96x72 input"""
    from hipie_oracle.resnet import ResNet50
    g = _load(golden_dir, "ref_r50.pt")
    m = ResNet50().eval()
    _same_keys(m, g["keys"])
    fill_by_name_(m, g["seed"])
    with torch.no_grad():
        out = m(g["x"])
    for k in ("res3", "res4", "res5"):
        ref = g["out"][k]
        got = out[k][:, ::8]
        assert (got - ref).abs().max() < 1e-5 * ref.abs().max() + 1e-5, (k, (got - ref).abs().max())


def test_maskclip_matches_reference(golden_dir):
    """open_vocab/clip.py MaskCLIP + ClipAdapter._encode_text and hipie_img.py get_clip_logits, run unmodified on the restated
    open_clip model (tiny configuration), against hipie_oracle.clip: mask embeddings, per-class logits (max over synonyms,
    clamped logit scale) and the fused log-probabilities in both aggregation modes."""
    from hipie_oracle import clip as oc
    g = _load(golden_dir, "ref_maskclip.pt")
    mc = oc.MaskCLIPOracle(oc.init_clip_(oc.CLIP(g["cfg"]), g["seed"]))
    assert abs(float(mc.logit_scale) - g["logit_scale"]) < 1e-6
    with torch.no_grad():
        te = mc.build_text_embed(g["ids"])
        out = mc(g["image"], g["mask"], te, g["labels"])
    tol = lambda ref: 2e-5 * float(ref.abs().max()) + 2e-6
    assert (te - g["text_embed"]).abs().max() < tol(g["text_embed"])
    assert (out["mask_embed"] - g["mask_embed"]).abs().max() < tol(g["mask_embed"])
    assert (out["mask_pred_open_logits"] - g["logits"]).abs().max() < tol(g["logits"])
    assert torch.equal(oc.synth_clip_tokenize([t for ls in g["labels"] for t in ls], g["cfg"]["text_ctx"], g["cfg"]["vocab"]), g["ids"])
    assert oc.prompt_labels([x["name"].split(",") for x in g["test_labels"]], "photo") == g["labels"]
    assert oc.category_overlapping_mask(g["test_labels"], g["train_labels"]).tolist() == [1, 0, 0, 1, 1]
    for mode, ref in g["fused"].items():
        with torch.no_grad():
            got = oc.get_clip_logits(mc, g["test_labels"], g["train_labels"], g["mask"], g["image"], g["pred_open_prob"], te, 0.35, 0.7, mode)
        assert (got - ref).abs().max() < 2e-5 * float(ref.abs().max()) + 1e-5, mode
    with torch.no_grad():
        single = mc.pred_logits(out["mask_embed"], te[:1], [g["labels"][0][:1]])
    assert (single - g["single_logits"]).abs().max() < tol(g["single_logits"])
    # the attention mask the oracle builds is the reference's layout: nobody attends to mask tokens, CLS always visible
    import torch.nn.functional as F
    m336 = F.interpolate(g["mask"], size=(g["cfg"]["image_size"],) * 2, mode="bilinear", align_corners=False)
    a = mc.attention_mask(m336)
    Q = g["mask"].shape[1]
    assert a.shape == (1, Q + 17, Q + 17) and bool(a[:, :, :Q].all()) and not bool(a[:, :, Q].any()) and not bool(a[:, Q:, Q:].any())
    assert 0 < int(a[:, :Q, Q + 1:].sum()) < Q * 16
