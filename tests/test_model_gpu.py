"""GPU: whole-model parity of the CUDA engine against the CPU oracle on the tiny ViT configuration
(same code paths as ViT-H: windowed + global blocks with rel-pos interpolation, 4 levels, VL fusion, two-stage
top-k, bg queries, MaskDINO branch, CondInst), same seeded weights and inputs.

The discontinuous selections (top-k proposals, NMS) are compared as sets on their scores and then pinned to the
oracle's indices for the tensor comparisons (SURVEY.md §7 "hard parts").  Tolerances (bf16x3 parity mode):
north-star says 1e-3 abs on mask logits; the random-weight CondInst logits are O(50..1000) (relative pixel
coordinates times unit-variance dynamic weights), so those are checked at 1e-3 relative to the max logit and
the MaskDINO mask logits (O(1)) at 1e-3 absolute.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def setup(cuda):
    from hipie_oracle import hparams, synth
    from hipie_oracle.model import HipieOracle
    from hipie_b200 import ops
    from hipie_b200.modeling.hipie_img import HIPIE_IMG
    torch.manual_seed(0)
    hp = hparams.get("vit_tiny")
    oracle = HipieOracle(hp).eval()
    synth.perturb_(oracle)
    inputs, ids, am = synth.make_batch(2, 256, 256, 5, hp["max_query_len"])
    with torch.no_grad():
        res_o, out_o = oracle(inputs, ids, am)
    ops.set_precision(3)
    model = HIPIE_IMG(hp=hp, state_dict=oracle.state_dict(), device="cuda:0")
    for x, i, a in zip(inputs, ids, am):
        x["input_ids"], x["attention_mask"] = i, a
    forced = {"topk_fg": out_o["aux"]["topk"].to(cuda), "topk_md": out_o["md"]["topk"].to(cuda)}
    res_g, out_g = model(inputs, forced=forced, return_raw=True)
    res_u, out_u = model(inputs, return_raw=True)
    return dict(oracle=oracle, model=model, res_o=res_o, out_o=out_o, res_g=res_g, out_g=out_g, out_u=out_u, inputs=inputs)


def _err(a, b):
    return (a.detach().float().cpu() - b.detach().float().cpu()).abs().max().item()


def test_backbone_features(setup):
    o, g = setup["out_o"]["features"], setup["out_g"]["aux"]["feats"]
    for k in ("res3", "res4", "res5"):
        ref = o[k].permute(0, 2, 3, 1)
        e = _err(g[k], ref)
        assert e < 1e-3 * max(1.0, ref.abs().max().item()), (k, e)


def test_text_and_fusion(setup):
    e = _err(setup["out_g"]["aux"]["lang_hidden_fused"], setup["out_o"]["lang_hidden_fused"])
    assert e < 1e-3, e
    e = _err(setup["out_g"]["aux"]["memory"], setup["out_o"]["memory"])
    assert e < 1e-3, e


def test_proposal_scores_and_topk_sets(setup):
    so, sg = setup["out_o"]["aux"]["enc_scores"], setup["out_u"]["aux"]["enc_scores"].cpu()
    assert (so - sg).abs().max() < 1e-3
    to, tg = setup["out_o"]["aux"]["topk"], setup["out_u"]["aux"]["topk"].cpu()
    for b in range(to.shape[0]):
        same = len(set(to[b].tolist()) & set(tg[b].tolist())) / to.shape[1]
        assert same >= 0.95, same       # near-ties at the cut-off may swap
    so, sg = setup["out_o"]["md"]["enc_scores"], setup["out_u"]["aux"]["md_enc_scores"].cpu()
    assert (so - sg).abs().max() < 1e-3


def test_decoder_states_boxes_logits(setup):
    o, g = setup["out_o"], setup["out_g"]
    for l in range(o["hs"].shape[0]):
        assert _err(g["aux"]["hs"][l], o["hs"][l]) < 2e-3, l
        assert _err(g["aux"]["refs"][l], o["inter_references"][l]) < 1e-4, l
    assert _err(g["pred_boxes"], o["pred_boxes"]) < 1e-4
    assert _err(g["pred_logits"], o["pred_logits"]) < 2e-3
    assert _err(g["pred_boxious"], o["pred_boxious"]) < 2e-3
    assert _err(g["pred_logits_maskdino"], o["pred_logits_maskdino"]) < 2e-3
    assert _err(g["pred_boxes_maskdino"], o["pred_boxes_maskdino"]) < 1e-4


def test_mask_logits(setup):
    o, g = setup["out_o"], setup["out_g"]
    e = _err(g["pred_masks_maskdino"], o["pred_masks_maskdino"])
    assert e < 1e-3, e                                           # north-star: 1e-3 abs on mask logits
    ref = o["pred_masks"]
    e = _err(g["pred_masks"], ref)
    assert e < 1e-3 * ref.abs().max().item(), (e, ref.abs().max().item())
    # fused sigmoid>0.5 bit-packed output of the mask-embed GEMM == sign of the logits
    bits = g["aux"]["mask_bits"].cpu()
    lg = g["pred_masks_maskdino"].cpu().flatten(2)
    B, Q, HW = lg.shape
    want = (lg > 0).view(B, Q, HW // 32, 32).long()
    want = (want << torch.arange(32)).sum(-1)
    want = torch.where(want >= 2 ** 31, want - 2 ** 32, want).int()
    assert torch.equal(bits.view(B, Q, HW // 32), want)


def test_final_outputs_identical_classes(setup):
    """identical argmax class assignments (pred_classes, sem_seg argmax, panoptic categories) with pinned selections"""
    for ro, rg in zip(setup["res_o"], setup["res_g"]):
        io, ig = ro["instances_post"], rg["instances"]
        assert torch.equal(io["pred_classes"], ig.pred_classes.cpu())
        assert (io["scores"] - ig.scores.cpu()).abs().max() < 1e-4
        assert (io["pred_boxes"] - ig.pred_boxes.tensor.cpu()).abs().max() < 1e-2
        agree = (io["pred_masks"] == ig.pred_masks.cpu()).float().mean()
        assert agree > 0.9999, agree
        so, sg = ro["sem_seg"], rg["sem_seg"].cpu()
        assert (so.argmax(0) == sg.argmax(0)).float().mean() > 0.9995
        assert (so - sg).abs().max() < 1e-3 * max(1.0, so.abs().max().item())
        po, pg = ro["panoptic_seg"], rg["panoptic_seg"]
        assert [s["category_id"] for s in po[1]] == [s["category_id"] for s in pg[1]]
        assert (po[0] == pg[0].cpu()).float().mean() > 0.9995


def test_fast_mode_runs_and_is_close(setup):
    """plain-bf16 mode (prec 1 + bf16 value map): same pipeline, looser agreement — reported, not a parity claim."""
    from hipie_b200 import ops
    model = setup["model"]
    ops.set_precision(1)
    try:
        forced = {"topk_fg": setup["out_o"]["aux"]["topk"].cuda(), "topk_md": setup["out_o"]["md"]["topk"].cuda()}
        _, out = model(setup["inputs"], forced=forced, return_raw=True)
    finally:
        ops.set_precision(3)
    ref = setup["out_o"]["pred_masks_maskdino"]
    rel = _err(out["pred_masks_maskdino"], ref) / ref.abs().max().item()
    assert rel < 0.25, rel


def test_cuda_graph_forward_matches_eager(setup):
    """enable_cuda_graphs(): forward() replays a captured graph; results equal the eager launch sequence (same kernels)."""
    model = setup["model"]
    eager = model(setup["inputs"])
    model.enable_cuda_graphs(True)
    try:
        first = model(setup["inputs"])       # captures
        again = model(setup["inputs"])       # replays
    finally:
        model.enable_cuda_graphs(False)
    for re_, r1, r2 in zip(eager, first, again):
        for r in (r1, r2):
            assert torch.equal(re_["instances"].pred_classes, r["instances"].pred_classes)
            assert (re_["instances"].scores - r["instances"].scores).abs().max() < 1e-6
            assert (re_["sem_seg"] - r["sem_seg"]).abs().max() < 1e-5
            assert torch.equal(re_["panoptic_seg"][0], r["panoptic_seg"][0])


def test_fused_postprocess_matches_op_chain(setup):
    """the fused semantic/panoptic kernel against the same model with the torch op chain (upsample -> sigmoid -> einsum / argmax)"""
    model = setup["model"]
    fused = model(setup["inputs"])
    model.fused_postprocess = False
    try:
        chain = model(setup["inputs"])
    finally:
        model.fused_postprocess = True
    for rf, rc in zip(fused, chain):
        assert (rf["sem_seg"] - rc["sem_seg"]).abs().max() < 1e-3 * max(1.0, rc["sem_seg"].abs().max().item())
        assert [s["category_id"] for s in rf["panoptic_seg"][1]] == [s["category_id"] for s in rc["panoptic_seg"][1]]
        assert (rf["panoptic_seg"][0] == rc["panoptic_seg"][0]).float().mean() > 0.9995


def _run_pair(cuda, inputs, ids, am, seed=0):
    from hipie_oracle import hparams, synth
    from hipie_oracle.model import HipieOracle
    from hipie_b200 import ops
    from hipie_b200.modeling.hipie_img import HIPIE_IMG
    torch.manual_seed(seed)
    hp = hparams.get("vit_tiny")
    oracle = HipieOracle(hp).eval()
    synth.perturb_(oracle, seed=seed + 1)
    with torch.no_grad():
        res_o, out_o = oracle(inputs, ids, am)
    ops.set_precision(3)
    model = HIPIE_IMG(hp=hp, state_dict=oracle.state_dict(), device="cuda:0")
    for x, i, a in zip(inputs, ids, am):
        x["input_ids"], x["attention_mask"] = i, a
    forced = {"topk_fg": out_o["aux"]["topk"].to(cuda), "topk_md": out_o["md"]["topk"].to(cuda)}
    res_g, out_g = model(inputs, forced=forced, return_raw=True)
    return res_o, out_o, res_g, out_g


def test_grounding_task_parity(cuda):
    """task == "grounding" (SURVEY §8 config #4 semantics): class logit from the PRE-fusion pooled sentence feature,
    positive_map {1: [0]}, top-1 instance, no semantic / panoptic branch."""
    from hipie_oracle import hparams, synth
    hp = hparams.get("vit_tiny")
    inputs, ids, am = synth.make_batch(2, 256, 256, 1, hp["max_query_len"], task="grounding", seed=4)
    res_o, out_o, res_g, out_g = _run_pair(cuda, inputs, ids, am, seed=2)
    assert _err(out_g["pred_logits"], out_o["pred_logits"]) < 2e-3
    assert _err(out_g["pred_boxes"], out_o["pred_boxes"]) < 1e-4
    ref = out_o["pred_masks"]
    assert _err(out_g["pred_masks"], ref) < 1e-3 * max(1.0, ref.abs().max().item())
    for ro, rg in zip(res_o, res_g):
        io, ig = ro["instances_post"], rg["instances"]
        assert len(ig) == 1 and torch.equal(io["pred_classes"], ig.pred_classes.cpu())
        assert (io["scores"] - ig.scores.cpu()).abs().max() < 1e-4
        assert (io["pred_boxes"] - ig.pred_boxes.tensor.cpu()).abs().max() < 1e-2
        assert (io["pred_masks"] == ig.pred_masks.cpu()).float().mean() > 0.9995
        assert rg["sem_seg"] is None and rg["panoptic_seg"][0] is None


def test_ragged_batch_padding_and_output_resize(cuda):
    """two images of different sizes (zero padding to the batch max rounded to 32, real padding masks, valid ratios < 1)
    and requested output sizes different from the input sizes (box rescale, nearest mask resize, second bilinear resize of
    the semantic / panoptic masks: the un-fused post-processing path)."""
    from hipie_oracle import hparams, synth
    hp = hparams.get("vit_tiny")
    _, ids, am = synth.make_batch(2, 256, 256, 5, hp["max_query_len"], seed=6)
    ii, aa, pos_map, is_thing = synth.make_text(5, hp["max_query_len"], 6)
    g = torch.Generator().manual_seed(9)
    sizes = [(224, 256), (256, 192)]
    outs = [(300, 343), (256, 192)]
    inputs = [dict(image=torch.rand(3, h, w, generator=g) * 255.0, height=oh, width=ow, task="detection", is_thing=is_thing,
                   positive_map_label_to_token=pos_map) for (h, w), (oh, ow) in zip(sizes, outs)]
    res_o, out_o, res_g, out_g = _run_pair(cuda, inputs, ids, am, seed=5)
    assert _err(out_g["pred_logits"], out_o["pred_logits"]) < 2e-3
    assert _err(out_g["pred_boxes"], out_o["pred_boxes"]) < 1e-4
    ref = out_o["pred_masks_maskdino"]
    assert _err(out_g["pred_masks_maskdino"], ref) < 1e-3 * max(1.0, ref.abs().max().item())
    for ro, rg, (oh, ow) in zip(res_o, res_g, outs):
        io, ig = ro["instances_post"], rg["instances"]
        assert tuple(ig.pred_masks.shape[-2:]) == (oh, ow)
        assert torch.equal(io["pred_classes"], ig.pred_classes.cpu())
        assert (io["pred_boxes"] - ig.pred_boxes.tensor.cpu()).abs().max() < 2e-2
        assert (io["pred_masks"] == ig.pred_masks.cpu()).float().mean() > 0.9995
        so, sg = ro["sem_seg"], rg["sem_seg"].cpu()
        assert tuple(sg.shape[-2:]) == (oh, ow)
        assert (so.argmax(0) == sg.argmax(0)).float().mean() > 0.9995
        assert (so - sg).abs().max() < 1e-3 * max(1.0, so.abs().max().item())
        assert (ro["panoptic_seg"][0] == rg["panoptic_seg"][0].cpu()).float().mean() > 0.9995


def test_wide_image_uses_tcgen05_attention(cuda):
    """128 x 1024 input -> 8 x 64 token grid: the global blocks take the wgmma flash-attention path (kw == 64, T % 128 == 0,
    V emitted transposed by the GEMM); rel-pos tables are interpolated 127 -> 15 along the height axis."""
    from hipie_oracle import hparams, synth
    from hipie_oracle.model import HipieOracle
    from hipie_b200 import ops
    from hipie_b200.modeling.hipie_img import HIPIE_IMG
    torch.manual_seed(1)
    hp = hparams.get("vit_tiny")
    hp["vit"] = dict(hp["vit"], img_size=1024, depth=3, window_block_indexes=(0,))
    oracle = HipieOracle(hp).eval()
    synth.perturb_(oracle, seed=3)
    inputs, ids, am = synth.make_batch(1, 128, 1024, 4, hp["max_query_len"], seed=5)
    with torch.no_grad():
        _, out_o = oracle(inputs, ids, am)
    ops.set_precision(3)
    model = HIPIE_IMG(hp=hp, state_dict=oracle.state_dict(), device="cuda:0")
    for x, i, a in zip(inputs, ids, am):
        x["input_ids"], x["attention_mask"] = i, a
    forced = {"topk_fg": out_o["aux"]["topk"].to(cuda), "topk_md": out_o["md"]["topk"].to(cuda)}
    ops.profiler.start()
    _, out_g = model(inputs, forced=forced, return_raw=True)
    prof = ops.profiler.stop()
    assert any(k.startswith("attention_tc") for k in prof), list(prof)
    for k in ("res3", "res4", "res5"):
        ref = out_o["features"][k].permute(0, 2, 3, 1)
        assert _err(out_g["aux"]["feats"][k], ref) < 1e-3 * max(1.0, ref.abs().max().item()), k
    assert _err(out_g["pred_masks_maskdino"], out_o["pred_masks_maskdino"]) < 1e-3
    assert _err(out_g["pred_logits"], out_o["pred_logits"]) < 2e-3


def _distinct_grounding_batch(hp, B, h, w, seed):
    """B images with B DIFFERENT referring expressions (different token ids per row)."""
    from hipie_oracle import synth
    imgs = synth.make_images(B, h, w, seed)
    rows_i, rows_a = [], []
    for b in range(B):
        g = torch.Generator().manual_seed(100 * seed + b)
        n = 4 + 2 * b
        toks = [101] + torch.randint(1996, 30000, (n,), generator=g).tolist() + [102]
        ii = torch.zeros(hp["max_query_len"], dtype=torch.long)
        ii[:len(toks)] = torch.tensor(toks)
        aa = torch.zeros(hp["max_query_len"], dtype=torch.long)
        aa[:len(toks)] = 1
        rows_i.append(ii)
        rows_a.append(aa)
    inputs = [dict(image=im, height=h, width=w, task="grounding", is_thing={1: True}, positive_map_label_to_token={1: [0]}) for im in imgs]
    return inputs, torch.stack(rows_i), torch.stack(rows_a)


def test_distinct_prompts_after_detection_batch(setup, cuda):
    """A detection batch (one prompt for every row) followed by a grounding batch with a different expression per row at the
    same (B, Lt): the text encoder must encode every row (round-1 bug: a pointer-keyed 'all rows equal' cache went stale when
    the allocator handed the new ids the old address).  Also through the CUDA-graph path, whose key carries the flag."""
    from hipie_oracle import hparams
    hp = hparams.get("vit_tiny")
    model, oracle = setup["model"], setup["oracle"]
    model(setup["inputs"])                                           # detection: same prompt in both rows
    inputs, ids, am = _distinct_grounding_batch(hp, 2, 256, 256, seed=7)
    assert not torch.equal(ids[0], ids[1])
    with torch.no_grad():
        res_o, out_o = oracle(inputs, ids, am)
    for x, i, a in zip(inputs, ids, am):
        x["input_ids"], x["attention_mask"] = i, a
    forced = {"topk_fg": out_o["aux"]["topk"].to(cuda), "topk_md": out_o["md"]["topk"].to(cuda)}
    _, out_g = model(inputs, forced=forced, return_raw=True)
    assert _err(out_g["aux"]["lang_hidden_fused"], out_o["lang_hidden_fused"]) < 1e-3
    assert _err(out_g["pred_logits"], out_o["pred_logits"]) < 2e-3
    assert _err(out_g["pred_boxes"], out_o["pred_boxes"]) < 1e-4
    # rows must differ from each other (a broadcast of row 0 would make them equal)
    assert (out_g["pred_logits"][0] - out_g["pred_logits"][1]).abs().max() > 1e-3
    eager = model(inputs)
    model.enable_cuda_graphs(True)
    try:
        model(setup["inputs"])                                       # captures the one-prompt graph
        g1 = model(inputs)                                           # must capture its own graph (flag is part of the key)
        g2 = model(inputs)
    finally:
        model.enable_cuda_graphs(False)
    for re_, r1, r2 in zip(eager, g1, g2):
        for r in (r1, r2):
            assert torch.equal(re_["instances"].pred_classes, r["instances"].pred_classes)
            assert (re_["instances"].scores - r["instances"].scores).abs().max() < 1e-6
            assert (re_["instances"].pred_boxes.tensor - r["instances"].pred_boxes.tensor).abs().max() < 1e-3


def test_bert_chunk_path_over_512_tokens(cuda):
    """MAX_QUERY_LEN 1024 with a ~700-token prompt: BertEncoder's chunking at '.'/EOS boundaries (bert_model.py:68-135) on both
    sides; the text features, the fused features and the class logits must agree; max-pooled scoring over 300 classes."""
    from hipie_oracle import hparams, synth
    from hipie_oracle.model import HipieOracle
    from hipie_b200 import ops
    from hipie_b200.modeling.hipie_img import HIPIE_IMG
    torch.manual_seed(11)
    hp = hparams.get("vit_tiny")
    hp.update(max_query_len=1024, max_pool=True, bg_cls_agnostic=True)
    oracle = HipieOracle(hp).eval()
    synth.perturb_(oracle, seed=12)
    inputs, ids, am = synth.make_batch(1, 256, 256, 230, 1024, seed=13)
    assert 512 < int(am[0].sum()) <= 1024
    with torch.no_grad():
        lang_o = oracle.forward_text(ids, am)
        res_o, out_o = oracle(inputs, ids, am)
    ops.set_precision(3)
    model = HIPIE_IMG(hp=hp, state_dict=oracle.state_dict(), device="cuda:0")
    lang_g = model.forward_text(ids, am)
    assert _err(lang_g["hidden"], lang_o["hidden"]) < 1e-3
    for x, i, a in zip(inputs, ids, am):
        x["input_ids"], x["attention_mask"] = i, a
    forced = {"topk_fg": out_o["aux"]["topk"].to(cuda), "topk_md": out_o["md"]["topk"].to(cuda)}
    res_g, out_g = model(inputs, forced=forced, return_raw=True)
    assert _err(out_g["aux"]["lang_hidden_fused"], out_o["lang_hidden_fused"]) < 1e-3
    assert _err(out_g["pred_logits"], out_o["pred_logits"]) < 2e-3
    assert _err(out_g["pred_masks_maskdino"], out_o["pred_masks_maskdino"]) < 1e-3
    for ro, rg in zip(res_o, res_g):
        assert torch.equal(ro["instances_post"]["pred_classes"], rg["instances"].pred_classes.cpu())
        so, sg = ro["sem_seg"], rg["sem_seg"].cpu()
        assert so.shape[0] == 230 and (so.argmax(0) == sg.argmax(0)).float().mean() > 0.9995
        assert [s["category_id"] for s in ro["panoptic_seg"][1]] == [s["category_id"] for s in rg["panoptic_seg"][1]]
    # serving mode: the cut positions are planned on the host before the capture (the capture itself may not read the ids back);
    # the replay with other tokens at the same cut positions refills the plan's buffers and must equal the eager result
    eager = model(inputs)
    ids2 = ids.clone()
    word = (am[0] == 1) & (ids[0] != 1012) & (ids[0] != 101) & (ids[0] != 102)
    ids2[0, word] = (ids[0, word] + 7) % 900 + 1100
    inputs2 = [dict(x, input_ids=i) for x, i in zip(inputs, ids2)]
    eager2 = model(inputs2)
    model.enable_cuda_graphs(True)
    try:
        cap = model(inputs)
        rep2 = model(inputs2)
        assert len(model._graphs) == 1                    # same plan signature: one graph, refilled
    finally:
        model.enable_cuda_graphs(False)
    for e, g in ((eager, cap), (eager2, rep2)):
        for re_, rg in zip(e, g):
            assert torch.equal(re_["instances"].pred_classes, rg["instances"].pred_classes)
            assert (re_["sem_seg"] - rg["sem_seg"]).abs().max() < 1e-5
    assert (eager[0]["sem_seg"] - eager2[0]["sem_seg"]).abs().max() > 1e-4          # the second prompt is a different prompt


def test_pybind_shim_through_reference_style_function(cuda):
    """hipie_b200.MultiScaleDeformableAttention installed under the pybind module's name and called the way the reference's
    MSDeformAttnFunction.forward does (ops/functions/ms_deform_attn_func.py:21-30: custom_fwd(cast_inputs=float32), positional
    (value, shapes, level_start, loc, weights, im2col_step)); result == ms_deform_attn_core_pytorch (the oracle restatement)."""
    import sys
    from torch.autograd import Function
    import hipie_b200.MultiScaleDeformableAttention as shim
    from hipie_oracle.msda import ms_deform_attn_core
    sys.modules["MultiScaleDeformableAttention"] = shim
    import MultiScaleDeformableAttention as MSDA

    class MSDeformAttnFunction(Function):
        @staticmethod
        @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
        def forward(ctx, value, shapes, lsi, loc, w, im2col_step):
            return MSDA.ms_deform_attn_forward(value, shapes, lsi, loc, w, im2col_step)

    g = torch.Generator().manual_seed(3)
    N, M, D, Lq, L, P = 2, 8, 32, 50, 4, 4
    shapes = torch.tensor([(16, 16), (8, 8), (4, 4), (2, 2)], dtype=torch.long)
    lsi = torch.cat((shapes.new_zeros((1,)), shapes.prod(1).cumsum(0)[:-1]))
    S = int(shapes.prod(1).sum())
    value = torch.rand(N, S, M, D, generator=g) * 0.01
    loc = torch.rand(N, Lq, M, L, P, 2, generator=g)
    w = torch.rand(N, Lq, M, L, P, generator=g) + 1e-5
    w = w / w.sum(-1, keepdim=True).sum(-2, keepdim=True)
    ref = ms_deform_attn_core(value, shapes, loc, w)
    out = MSDeformAttnFunction.apply(value.cuda(), shapes.cuda(), lsi.cuda(), loc.cuda(), w.cuda(), 64)
    assert (out.cpu() - ref).abs().max() < 1e-6
    with pytest.raises(RuntimeError, match="Not implemented on the CPU"):
        MSDA.ms_deform_attn_forward(value, shapes, lsi, loc, w, 64)
    with pytest.raises(RuntimeError):
        MSDA.ms_deform_attn_forward(value.cuda()[:, ::2], shapes.cuda(), lsi.cuda(), loc.cuda(), w.cuda(), 64)


def test_predictor_and_registry_components(setup, cuda, tmp_path):
    """HIPIEPredictor (predictor.py:245-372 contract) on a BGR uint8 image with a custom vocabulary and with a referring
    expression, through the tokenizer / prompt builder; D2ViT and MaskDINOHead from the registries reproduce the engine stages."""
    import numpy as np
    from hipie_oracle import hparams
    from hipie_b200 import registry
    from hipie_b200.config import add_hipie_config, get_cfg
    from hipie_b200.data import load_tokenizer
    from hipie_b200.predictor import HIPIEPredictor
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]", ".", "person", "traffic", "light", "dog", "sky", "wall", "the", "left", "hair", "dr", "##ier"]
    (tmp_path / "vocab.txt").write_text("\n".join(vocab) + "\n")
    tok = load_tokenizer(str(tmp_path))
    model = setup["model"]
    cfg = get_cfg()
    add_hipie_config(cfg)
    cfg.INPUT.MIN_SIZE_TEST, cfg.INPUT.MAX_SIZE_TEST, cfg.INPUT.FORMAT = 192, 256, "RGB"
    cats = [{"name": "person"}, {"name": "traffic light"}, {"name": "dog"}, {"name": "sky", "isthing": 0}, {"name": "hair drier"}]
    pred = HIPIEPredictor(cfg, test_categories=cats, tokenizer=tok, model=model)
    img = (np.random.RandomState(0).rand(120, 160, 3) * 255).astype(np.uint8)
    out = pred(img, "detection", dataset_name="custom")
    inst = out["instances"]
    assert inst.pred_masks.shape[-2:] == (120, 160) and len(inst) > 0 and int(inst.pred_classes.max()) < len(cats)
    assert out["sem_seg"].shape == (len(cats), 120, 160)
    # same image through the model API with the predictor's pre-processing done by hand -> identical results
    from hipie_b200.data import ResizeShortestEdge, create_queries_and_maps
    rgb = ResizeShortestEdge([192, 192], 256).apply_image(np.ascontiguousarray(img[:, :, ::-1]))
    q, pm = create_queries_and_maps(cats, tok)
    direct = model([dict(image=torch.as_tensor(rgb.astype("float32").transpose(2, 0, 1)), height=120, width=160, task="detection", expressions=q,
                         is_thing={1: True, 2: True, 3: True, 4: False, 5: True}, positive_map_label_to_token=pm)])[0]
    assert torch.equal(direct["instances"].pred_classes, inst.pred_classes) and torch.equal(direct["sem_seg"], out["sem_seg"])
    g = pred(img, "grounding", expressions="the dog left")
    assert len(g["instances"]) == 1 and g["sem_seg"] is None
    with pytest.raises(ValueError):
        pred(img, "sot")
    # registry components
    hp = hparams.get("vit_tiny")
    registry._register_defaults()
    sd = setup["oracle"].state_dict()
    vit_sd = {k[len("detr.detr.backbone.0.backbone."):]: v for k, v in sd.items() if k.startswith("detr.detr.backbone.0.backbone.")}
    bb = registry.BACKBONE_REGISTRY.get("D2ViT")(hp=hp, device="cuda:0", state_dict=vit_sd)
    assert bb.size_divisibility == 32 and bb.output_shape()["res4"].stride == 16
    x = torch.randn(1, 3, 128, 160)
    with torch.no_grad():
        ref = setup["oracle"].detr.detr.backbone[0].backbone(x)
    got = bb(x)
    for k in ("res3", "res4", "res5"):
        assert _err(got[k], ref[k]) < 1e-3 * max(1.0, ref[k].abs().max().item())
    md_sd = {k[len("detr.mask_dino."):]: v for k, v in sd.items() if k.startswith("detr.mask_dino.")}
    head = registry.SEM_SEG_HEADS_REGISTRY.get("MaskDINOHead")(hp=hp, device="cuda:0", state_dict=md_sd)
    with torch.no_grad():
        ref_md = setup["oracle"].detr.mask_dino(ref)
    out_md, _ = head(ref)
    assert _err(out_md["pred_masks"], ref_md["pred_masks"]) < 1e-3
    assert out_md["pred_masks"].shape == ref_md["pred_masks"].shape and out_md["pred_logits"].shape == ref_md["pred_logits"].shape


def test_pinned_arena_results_to_host(cuda):
    """hipie_b200.hostio.PinnedArena: async device->host copies into ONE persistent page-locked buffer (views valid after wait();
    dtype / shape / alignment preserved; a step that outgrows the arena spills to fresh pinned tensors and the arena grows at reset)."""
    from hipie_b200.hostio import PinnedArena
    arena = PinnedArena(1 << 16)
    g = torch.Generator(device="cuda").manual_seed(1)
    tensors = [torch.randn(100, 7, device=cuda, generator=g), torch.randint(0, 255, (33,), device=cuda, dtype=torch.uint8, generator=g),
               torch.randint(0, 9, (5, 11), device=cuda, generator=g), torch.randn(64, 64, device=cuda, generator=g) > 0]
    for step in range(3):
        arena.reset()
        host = [arena.to_host(t) for t in tensors]
        big = arena.to_host(torch.ones(1 << 15, device=cuda)) if step == 0 else None      # 128 KB > the 64 KB arena: spill, then growth
        arena.wait()
        for h, t in zip(host, tensors):
            assert h.is_pinned() and h.dtype == t.dtype and h.shape == t.shape and torch.equal(h, t.cpu())
            assert h.data_ptr() % 256 == 0 or big is not None
        if big is not None:
            assert big.is_pinned() and float(big.sum()) == float(1 << 15)
