"""GPU: whole-model parity at the BASELINE.json sizes, UNFORCED (no selection is pinned to the oracle's) and forced.

Every case builds the CPU oracle (oracle/hipie_oracle, the restatement of the reference eval forward) and the CUDA engine
from the same seeded weights, runs both on the same seeded inputs and compares

  * the continuous outputs stage by stage (ViT residual stream after blocks 8/16/32, FPN features, encoder memory, fused
    text features, decoder states, class logits, boxes, MaskDINO mask logits, CondInst logits) -- the table is written to
    gpurun_out/parity_<case>.json for profiles/ and printed,
  * the discrete results of the public API with NOTHING forced: pred_classes, sem_seg.argmax, panoptic categories.

Cases (SURVEY.md §8d):
  c1   configs[1] at B=1: ViT-H (32 blocks, d=1280, T=4096), 1024x1024, 80 classes, Lt=512, task detection
  c4   configs[3] path: ViT-H, 1280x1280 (80-wide token grid, rel-pos tables 127->159, 36 padded windows), task grounding
  c5   configs[4] path: ViT-H, 847-class vocabulary, Lt=4096 (> 512 tokens: BertEncoder chunk path, bert_model.py:68-135),
       max-pooled / class-agnostic-bg scoring of the ADE eval yaml, at 512x512 so the CPU oracle stays within the test budget

Tolerances (written here, north-star: 1e-3 abs on mask logits, identical argmax class assignments):
  MaskDINO mask logits 1e-3 ABS; class logits 2e-3 abs; boxes 1e-4 abs; CondInst logits are O(1e3) with seeded random
  weights (pixel-unit relative coordinates times unit-variance dynamic filters) -- fp32 itself moves them by > 1e-3 when the
  summation order changes, so they are asserted at 3e-4 RELATIVE to max|logit| and their absolute error is reported in
  the table (the thresholded masks, which are what the reference emits, must agree on > 99.99 % of the pixels).
"""
import json
import os
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_T0 = time.time()
BUDGET_S = 900.0          # the whole GPU suite has to stay well inside the driver's pytest limit


def _budget(need):
    if time.time() - _T0 + need > BUDGET_S:
        pytest.skip(f"time budget: {time.time() - _T0:.0f}s used, case needs ~{need:.0f}s")


def _err(a, b):
    return (a.detach().float().cpu() - b.detach().float().cpu()).abs().max().item()


def _run_case(name, hp, inputs, ids, am, seed, taps=(7, 15, 31)):
    from hipie_oracle import synth
    from hipie_oracle.model import HipieOracle
    from hipie_b200 import ops
    from hipie_b200.modeling.hipie_img import HIPIE_IMG
    torch.set_num_threads(min(32, os.cpu_count() or 8))
    torch.manual_seed(seed)
    t0 = time.time()
    oracle = HipieOracle(hp).eval()
    synth.perturb_(oracle, seed=seed + 1)
    blocks = getattr(oracle.detr.detr.backbone[0].backbone, "blocks", [])      # ViT only; the R50 case has no residual-stream taps
    taps = tuple(t for t in taps if t < len(blocks))
    otaps, hooks = {}, []
    for t in taps:
        hooks.append(blocks[t].register_forward_hook(lambda m, i, o, t=t: otaps.__setitem__(t, o.detach().clone())))
    with torch.no_grad():
        res_o, out_o = oracle(inputs, ids, am)
    for h in hooks:
        h.remove()
    t_oracle = time.time() - t0
    for x, i, a in zip(inputs, ids, am):
        x["input_ids"], x["attention_mask"] = i, a
    model = HIPIE_IMG(hp=hp, state_dict=oracle.state_dict(), device="cuda:0")
    forced = {"topk_fg": out_o["aux"]["topk"].cuda(), "topk_md": out_o["md"]["topk"].cuda()}
    table = {"case": name, "oracle_seconds": t_oracle, "cpu_threads": torch.get_num_threads(), "stages": {}}
    runs = {}
    for prec in (3, 1):
        ops.set_precision(prec)
        model.engine.bf16_value_map = False
        model.engine.taps = {"blocks": taps}
        try:
            res_f, out_f = model(inputs, forced=forced, return_raw=True)
            gt = dict(model.engine.taps)
            model.engine.taps = None
            res_u, out_u = (model(inputs, return_raw=True) if prec == 3 else (None, None))
        finally:
            ops.set_precision(3)
            model.engine.taps = None
        st = {}
        for t in taps:
            st[f"vit.block{t + 1}"] = (_err(gt[f"vit.block{t}"], otaps[t]), otaps[t].abs().max().item())
        for k in ("res3", "res4", "res5"):
            ref = out_o["features"][k].permute(0, 2, 3, 1)
            st[f"fpn.{k}"] = (_err(out_f["aux"]["feats"][k], ref), ref.abs().max().item())
        st["encoder.memory"] = (_err(out_f["aux"]["memory"], out_o["memory"]), out_o["memory"].abs().max().item())
        st["text.fused"] = (_err(out_f["aux"]["lang_hidden_fused"], out_o["lang_hidden_fused"]), out_o["lang_hidden_fused"].abs().max().item())
        st["decoder.hs_last"] = (_err(out_f["aux"]["hs"][-1], out_o["hs"][-1]), out_o["hs"][-1].abs().max().item())
        for k in ("pred_logits", "pred_boxes", "pred_boxious", "pred_logits_maskdino", "pred_boxes_maskdino", "pred_masks_maskdino", "pred_masks"):
            st[k] = (_err(out_f[k], out_o[k]), out_o[k].abs().max().item())
        table["stages"][f"prec{prec}"] = {k: {"max_abs_err": v[0], "ref_max_abs": v[1]} for k, v in st.items()}
        runs[prec] = (res_f, out_f, res_u, out_u)
    del model
    torch.cuda.empty_cache()
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", f"parity_{name}.json"), "w") as f:
        json.dump(table, f, indent=1)
    print(f"\n[{name}] oracle {t_oracle:.0f}s on {table['cpu_threads']} threads")
    for k in table["stages"]["prec3"]:
        a, b = table["stages"]["prec3"][k], table["stages"]["prec1"][k]
        print(f"  {k:24s} |ref|max {a['ref_max_abs']:10.3f}   bf16x3 {a['max_abs_err']:.3e}   bf16 {b['max_abs_err']:.3e}")
    return dict(res_o=res_o, out_o=out_o, res_f=runs[3][0], out_f=runs[3][1], res_u=runs[3][2], out_u=runs[3][3], table=table)


def _check_continuous(r, grounding=False):
    t = r["table"]["stages"]["prec3"]
    assert t["pred_masks_maskdino"]["max_abs_err"] < 1e-3, t["pred_masks_maskdino"]          # north-star: 1e-3 ABS
    assert t["pred_logits"]["max_abs_err"] < 2e-3, t["pred_logits"]
    assert t["pred_logits_maskdino"]["max_abs_err"] < 2e-3, t["pred_logits_maskdino"]
    assert t["pred_boxes"]["max_abs_err"] < 1e-4 and t["pred_boxes_maskdino"]["max_abs_err"] < 1e-4
    assert t["pred_masks"]["max_abs_err"] < 3e-4 * t["pred_masks"]["ref_max_abs"], t["pred_masks"]   # CondInst: relative (see header)
    # (the plain-bf16 column of the printed table is the measurement behind the 3-pass parity mode, DESIGN.md §3)


def _match_instances(io, iu, tie=2e-5):
    """Order-insensitive comparison of two instance lists.  The reference emits the flat top-100 over (kept query x class)
    sorted by score (hipie_img.py:640-648); with seeded random weights hundreds of candidates sit within 1e-5 of each other, so
    fp32-level differences permute neighbours and decide membership at the cut-off.  Every instance of one side must have a
    partner on the other with the SAME class, score within 1e-4 and box within 0.05 px; the only instances allowed to stay
    unmatched are cut-off ties (score within `tie` of the 100th score)."""
    so, co, bo = io["scores"], io["pred_classes"], io["pred_boxes"]
    su, cu, bu = iu.scores.cpu(), iu.pred_classes.cpu(), iu.pred_boxes.tensor.cpu()
    used = torch.zeros(len(su), dtype=torch.bool)
    unmatched_o = []
    for i in range(len(so)):
        ok = (cu == co[i]) & ((su - so[i]).abs() < 1e-4) & ((bu - bo[i]).abs().amax(-1) < 0.05) & ~used
        j = torch.nonzero(ok)
        if len(j):
            used[j[0, 0]] = True
        else:
            unmatched_o.append(i)
    cut = min(float(so.min()), float(su.min()))
    bad = [i for i in unmatched_o if float(so[i]) > cut + tie] + [j for j in torch.nonzero(~used).flatten().tolist() if float(su[j]) > cut + tie]
    in_order = int((co[:len(cu)] == cu[:len(co)]).sum()) if len(co) == len(cu) else -1
    return dict(n=len(so), matched=int(used.sum()), unmatched_cutoff_ties=len(unmatched_o) - len([i for i in unmatched_o if float(so[i]) > cut + tie]),
                bad=len(bad), same_position_classes=in_order)


def _check_unforced(r, detection=True):
    """NOTHING pinned: the engine's own proposal top-k / NMS / top-100 selections.

    What can and cannot be identical: the reference pairs the i-th ranked proposal with the i-th learned content query
    (deformable_transformer_dino.py:228-248), so the RANK ORDER inside the top-k matters, and with seeded random weights the
    encoder scores contain (a) hundreds of EXACT ties -- every border position whose proposal is invalid gets the same
    score, utils: (op > 0.01) & (op < 0.99) -- which torch.topk breaks differently on CPU and CUDA (the reference's own CUDA
    top-k is not deterministic there), and (b) neighbours closer than fp32 rounding.  Two scores can change order only when they are
    closer than twice the largest score error eps = max|s_engine - s_oracle| (asserted < 2e-4 on logits of magnitude ~5, i.e. well
    inside the 2e-3 class-logit tolerance), so the tie width is 2 eps (at least 5e-5).  Asserted here: the engine's selection is a
    valid top-k OF THE ORACLE'S SCORES up to such ties, every rank swap is between scores closer than the tie width, and the final
    discrete outputs agree except where such a swap re-paired a query (>= 90 % of the instances one-to-one with identical class,
    score within 1e-4 and box within 0.05 px; semantic argmax >= 99.5 % of the pixels).  The forced variant of the same case
    (proposal ranks pinned, everything downstream unforced) must match completely."""
    out_o, out_u = r["out_o"], r["out_u"]
    tk_o, tk_u = out_o["aux"]["topk"], out_u["aux"]["topk"].cpu()
    s_o, s_u = out_o["aux"]["enc_scores"], out_u["aux"]["enc_scores"].cpu()
    same_sets = [len(set(a.tolist()) & set(b.tolist())) / a.numel() for a, b in zip(tk_o, tk_u)]
    kth = torch.gather(s_o, 1, tk_o).min(1)[0]
    sel = torch.gather(s_o, 1, tk_u)                       # the oracle's scores of the engine's picks
    eps = (s_o - s_u).abs().max().item()
    tie = max(5e-5, 2.0 * eps + 1e-6)
    valid_topk = bool((sel >= kth[:, None] - tie).all())
    rank_gap = (torch.gather(s_o, 1, tk_o) - sel).abs().max().item()      # same rank -> (almost) the same score
    stats = {"enc_scores_max_abs_err": eps, "tie_width": tie, "proposal_topk_overlap": same_sets,
             "proposal_topk_identical_order": bool(torch.equal(tk_o, tk_u)), "engine_topk_valid_for_oracle_scores": valid_topk,
             "max_score_gap_at_equal_rank": rank_gap}
    fails = []
    if eps > 2e-4:
        fails.append(f"proposal scores differ by {eps}")
    if not valid_topk:
        fails.append("engine proposal top-k is not a top-k of the oracle's scores")
    if rank_gap > tie:
        fails.append(f"rank swap between scores {rank_gap} apart (tie width {tie})")
    for n, (ro, ru) in enumerate(zip(r["res_o"], r["res_u"])):
        io, iu = ro["instances_post"], ru["instances"]
        m = _match_instances(io, iu)
        stats[f"img{n}.instances"] = m
        if m["matched"] < 0.9 * m["n"] or len(iu) != m["n"]:
            fails.append(f"img{n}: {m}")
        if not detection:
            # top-1 grounding: the single instance must be the same query (same class id 0, same score / box)
            if not (ru["sem_seg"] is None and ru["panoptic_seg"][0] is None):
                fails.append("grounding must not produce sem/pano outputs")
            if m["n"] == 1 and m["matched"] == 1:
                agree = (io["pred_masks"] == iu.pred_masks.cpu()).float().mean().item()
                stats[f"img{n}.mask_agreement"] = agree
                if agree <= 0.9999:
                    fails.append(f"img{n}: mask agreement {agree}")
            continue
        so, su = ro["sem_seg"], ru["sem_seg"].cpu()
        a = (so.argmax(0) == su.argmax(0)).float().mean().item()
        po, pu = ro["panoptic_seg"], ru["panoptic_seg"]
        cat_o, cat_u = [s["category_id"] for s in po[1]], [s["category_id"] for s in pu[1]]
        pa = (po[0] == pu[0].cpu()).float().mean().item()
        stats[f"img{n}.sem_seg_argmax_agreement"] = a
        stats[f"img{n}.sem_seg_max_abs_err"] = (so - su).abs().max().item()
        stats[f"img{n}.panoptic"] = dict(segments_oracle=len(cat_o), segments_engine=len(cat_u), categories_identical=cat_o == cat_u, id_map_agreement=pa)
        if a <= 0.995:
            fails.append(f"img{n}: sem_seg argmax agreement {a}")
        if cat_o != cat_u:
            fails.append(f"img{n}: panoptic categories differ: {cat_o} vs {cat_u}")
        if pa <= 0.995:
            fails.append(f"img{n}: panoptic id map agreement {pa}")
    r["table"]["unforced"] = stats
    with open(os.path.join(ROOT, "gpurun_out", f"parity_{r['table']['case']}.json"), "w") as f:
        json.dump(r["table"], f, indent=1)
    print("  unforced:", json.dumps(stats))
    assert not fails, fails


def test_c1_vith_1024_coco80_lt512(cuda):
    _budget(200)
    from hipie_oracle import hparams, synth
    hp = hparams.get("vit_h")
    inputs, ids, am = synth.make_batch(1, 1024, 1024, 80, hp["max_query_len"])
    r = _run_case("c1_vith_1024_coco80", hp, inputs, ids, am, seed=0)
    _check_continuous(r)
    _check_unforced(r)
    _check_forced(r)


def _check_forced(r, detection=True):
    """proposal ranks pinned to the oracle's, everything downstream (NMS, flat top-100, argmax maps, panoptic merge) unforced:
    every instance must find its partner, argmax maps must agree"""
    for n, (ro, rf) in enumerate(zip(r["res_o"], r["res_f"])):
        m = _match_instances(ro["instances_post"], rf["instances"])
        assert m["bad"] == 0 and m["matched"] >= m["n"] - 2, m
        if detection:
            so, sf = ro["sem_seg"], rf["sem_seg"].cpu()
            a = (so.argmax(0) == sf.argmax(0)).float().mean().item()
            assert a > 0.9995, a
            assert (so - sf).abs().max() < 1e-3 * max(1.0, so.abs().max().item())
            po, pf = ro["panoptic_seg"], rf["panoptic_seg"]
            assert [s["category_id"] for s in po[1]] == [s["category_id"] for s in pf[1]]
            assert (po[0] == pf[0].cpu()).float().mean().item() > 0.9995


def test_c4_vith_1280_grounding(cuda):
    _budget(220)
    from hipie_oracle import hparams, synth
    hp = hparams.get("vit_h")
    inputs, ids, am = synth.make_batch(1, 1280, 1280, 1, hp["max_query_len"], task="grounding", seed=3)
    r = _run_case("c4_vith_1280_grounding", hp, inputs, ids, am, seed=4)
    _check_continuous(r, grounding=True)
    _check_unforced(r, detection=False)
    _check_forced(r, detection=False)


def test_c5_vith_ade847_lt4096_chunked_bert(cuda):
    _budget(200)
    from hipie_oracle import hparams, synth
    hp = hparams.get("vit_h")
    hp.update(max_query_len=4096, max_pool=True, bg_cls_agnostic=True)
    inputs, ids, am = synth.make_batch(1, 512, 512, 847, 4096, seed=5)
    assert int(am[0].sum()) > 512          # the prompt really takes the chunk path
    r = _run_case("c5_vith_512_ade847_lt4096", hp, inputs, ids, am, seed=6)
    _check_continuous(r)
    _check_unforced(r)
    _check_forced(r)


def test_c0_r50_512_three_queries(cuda):
    """BASELINE configs[0]: ResNet-50 backbone, 1 x 512 x 512, 3 text queries (the reference's CPU-runnable plumbing case) through
    the same public entry point, on the engine's R50 path (convolutions as GEMMs, frozen BN folded, bottleneck ReLU after the residual)."""
    _budget(120)
    from hipie_oracle import hparams, synth
    hp = hparams.get("r50")
    inputs, ids, am = synth.make_batch(1, 512, 512, 3, hp["max_query_len"], seed=8)
    r = _run_case("c0_r50_512_3queries", hp, inputs, ids, am, seed=9, taps=())
    _check_continuous(r)
    _check_unforced(r)
    _check_forced(r)
