"""GPU: MaskCLIP re-scoring (SURVEY a22 / f2) -- the support kernels against torch restatements of the reference lines, the GPU
MaskCLIP engine against the fixture produced by the UNMODIFIED reference classes (tests/golden/ref_maskclip.pt, oracle/
gen_golden_modules.py gen_maskclip) and the whole model with CLIP attached against the CPU oracle."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops(cuda):
    from hipie_b200 import ops as o
    o.set_precision(3)
    return o


def _pack(m):
    from hipie_b200.modeling.maskclip import MaskCLIP
    pad = (-m.shape[1]) % 32
    return MaskCLIP._pack_bits(F.pad(m, (0, pad)).cpu())


def test_attention_boolean_key_mask(ops, cuda):
    """hipie_attention with key_mask == nn.MultiheadAttention's boolean attn_mask (True = masked out), per (batch, query) row"""
    g = torch.Generator(device="cuda").manual_seed(3)
    B, H, hd, Tq, Tk = 2, 3, 64, 100, 77
    qkv = torch.randn(B, Tq, 3, H, hd, device=cuda, generator=g)
    S = ops.split(qkv)
    mask = torch.rand(B, Tq, Tk, device=cuda, generator=g) < 0.6
    mask[:, :, 0] = False                                         # every query keeps one key (MaskCLIP: the CLS token)
    mask[1, 5, :] = True
    mask[1, 5, 40] = False
    bits = torch.stack([_pack(mask[b]) for b in range(B)]).to(cuda)
    ts, bs = 3 * H * hd, Tq * 3 * H * hd
    o, _ = ops.attention(ops.BF2(S.hi[:, :, 0], S.lo[:, :, 0]), ops.BF2(S.hi[:, :Tk, 1], S.lo[:, :Tk, 1]), ops.BF2(S.hi[:, :Tk, 2], S.lo[:, :Tk, 2]),
                         B, H, Tq, Tk, hd, (bs, ts, hd), (bs, ts, hd), (bs, ts, hd), hd ** -0.5, key_mask=bits, want_f32=True, want_split=False)
    q, k, v = (qkv[:, :, 0].permute(0, 2, 1, 3).double(), qkv[:, :Tk, 1].permute(0, 2, 1, 3).double(), qkv[:, :Tk, 2].permute(0, 2, 1, 3).double())
    s = (q * hd ** -0.5) @ k.transpose(-1, -2)
    s = s.masked_fill(mask[:, None], float("-inf"))
    ref = (torch.softmax(s, -1) @ v).permute(0, 2, 1, 3).reshape(B, Tq, H * hd)
    assert (o.double() - ref).abs().max() < 2e-5


def test_gemm_quick_gelu(ops, cuda):
    g = torch.Generator(device="cuda").manual_seed(4)
    a, w, b = torch.randn(300, 128, device=cuda, generator=g), torch.randn(512, 128, device=cuda, generator=g) * 0.2, torch.randn(512, device=cuda, generator=g)
    c, cs, _ = ops.gemm(ops.split(a), ops.split_weight(w), bias=b, act=ops.ACT_QUICK_GELU, want_f32=True, want_split=True)
    y = a.double() @ w.double().t() + b.double()
    ref = y * torch.sigmoid(1.702 * y)
    assert (c.double() - ref).abs().max() < 3e-5 * ref.abs().max()
    assert (cs.float().double() - ref).abs().max() < 3e-5 * ref.abs().max()


@pytest.mark.parametrize("up", [1, 4])
def test_patch_mask_bits_match_reference_ops(ops, cuda, up):
    """clip.py:296-309: interpolate(mask -> S x S) -> sigmoid -> max_pool2d(P) < 0.5; up = 4: the source is the x4 bilinear upsample of
    the stored map, cropped (hipie_img.py:733-741)"""
    g = torch.Generator().manual_seed(5 + up)
    Q, h, w, S, P = 11, 20, 27, 56, 14
    masks = torch.randn(Q, h, w, generator=g) * 3
    masks[3] = -4.0                                               # everything masked out
    masks[4] = 4.0                                                # nothing masked out
    crop = (h, w) if up == 1 else (4 * h - 6, 4 * w - 9)
    src = masks[None]
    if up > 1:
        src = F.interpolate(src, size=(4 * h, 4 * w), mode="bilinear", align_corners=False)[:, :, :crop[0], :crop[1]]
    big = F.interpolate(src, size=(S, S), mode="bilinear", align_corners=False)
    ref = (F.max_pool2d(big.sigmoid(), P, P) < 0.5).reshape(Q, -1)
    G2 = (S // P) ** 2
    words = (1 + G2 + 31) // 32
    bits = torch.full((Q + 2, words), -1, dtype=torch.int32, device=cuda)
    ops.maskclip_patch_mask(masks.to(cuda), S, P, bits, key_offset=1, up=up, crop=crop)
    got = torch.zeros(Q, G2, dtype=torch.bool)
    b = bits.cpu().long() & 0xFFFFFFFF
    for kk in range(G2):
        key = 1 + kk
        got[:, kk] = ((b[:Q, key >> 5] >> (key & 31)) & 1).bool()
    assert (b[:Q, 0] & 1).sum() == 0                              # CLS key never masked
    assert torch.equal(b[Q:], torch.full((2, words), 0xFFFFFFFF))   # rows beyond Q untouched
    # a sample within 1e-6 of zero may round either way; none expected with random data
    assert torch.equal(got, ref), (got != ref).sum()
    assert bool(ref[3].all()) and not bool(ref[4].any())


def test_clip_patches_match_resize_normalize_unfold(ops, cuda):
    from hipie_b200.modeling.maskclip import OPENAI_MEAN, OPENAI_STD
    g = torch.Generator().manual_seed(6)
    img = torch.rand(3, 45, 70, generator=g)
    S, P = 56, 14
    big = F.interpolate(img[None], size=(S, S), mode="bilinear", align_corners=False)
    big = (big - torch.tensor(OPENAI_MEAN).view(1, 3, 1, 1)) / torch.tensor(OPENAI_STD).view(1, 3, 1, 1)
    ref = F.unfold(big, P, stride=P)[0].t()                       # (G*G, 3*P*P) in Conv2d weight order
    out = ops.clip_patches(img.to(cuda), S, P, OPENAI_MEAN, OPENAI_STD)
    got = (out.hi.float() + out.lo.float()).cpu()
    assert got.shape == (16, 592) and bool((got[:, 588:] == 0).all())
    assert (got[:, :588] - ref).abs().max() < 1e-4


@pytest.mark.parametrize("agg", ["MUL", "ADD"])
@pytest.mark.parametrize("C", [1, 5])
def test_clip_fuse_modes(ops, cuda, agg, C):
    from hipie_oracle import clip as oc
    g = torch.Generator().manual_seed(7 + C)
    R, D = 9, 64
    labels = [["a", "b", "c"], ["d"], ["e", "f"], ["g"], ["h", "i"]][:C]
    seg = [0]
    for ls in labels:
        seg.append(seg[-1] + len(ls))
    Np = seg[-1]
    emb, text = torch.randn(R, D, generator=g) * 2, torch.randn(Np, D, generator=g)
    text_n = F.normalize(text, dim=-1)
    scores0 = torch.randn(R, C, generator=g) * 2
    overlap = torch.tensor([1, 0, 0, 1, 1][:C], dtype=torch.long)
    iou = torch.randn(R, generator=g)
    scale = 14.285
    clip_logits = oc.ensemble_logits_with_labels(torch.einsum("qc,nc->qn", F.normalize(emb, dim=-1), text_n) * scale, labels)
    dev = lambda t: t.to(cuda)
    raw = dev(emb @ text_n.t())
    args = (raw, dev(emb), scale, dev(torch.tensor(seg, dtype=torch.int32)))
    ov8 = dev(overlap.to(torch.int8))
    for temp in (0.06, 0.0):
        if C == 1 and temp > 0:
            continue
        scores = scores0.clone()
        if temp > 0:                  # a masked class (-9999): only with the softmax form -- with plain sigmoid the reference's own
            scores[:, 1] = -9999.0    # formula gives log(0) * 0 = NaN, and that combination never occurs (hipie_img.py:595-598, 729-732)
        p_model = F.softmax(scores.sigmoid() / temp, -1) if temp > 0 else scores.sigmoid()
        fused = oc.fuse_clip_probs(p_model, clip_logits, overlap, 0.35, 0.7, agg)
        got0 = ops.clip_fuse(*args, dev(scores), temp, ov8, 0.35, 0.7, agg == "ADD", 0).cpu()
        fin = torch.isfinite(fused)
        assert torch.equal(torch.isfinite(got0), fin) and (got0[fin] - fused[fin]).abs().max() < 1e-4
        got2 = ops.clip_fuse(*args, dev(scores), temp, ov8, 0.35, 0.7, agg == "ADD", 2).cpu()
        assert (got2 - fused.softmax(-1)).abs().max() < 1e-5
        thing = (~(scores[:1] == -9999.0)).float()
        ref1 = torch.sqrt((fused.sigmoid() * thing) ** 0.3 * (iou.sigmoid() ** 1.7).unsqueeze(1))
        got1, rmax, rarg = ops.clip_fuse(*args, dev(scores), temp, ov8, 0.35, 0.7, agg == "ADD", 1, iou=dev(iou), fg_a=0.3, fg_b=1.7)
        assert (got1.cpu() - ref1).abs().max() < 1e-5
        m, a = ref1.max(1)
        assert (rmax.cpu() - m).abs().max() < 1e-5 and torch.equal(rarg.cpu().long(), a)


def test_maskclip_engine_matches_reference_fixture(cuda, golden_dir):
    """The GPU MaskCLIP (tiny CLIP weights recreated by name) against what the reference's own MaskCLIP / get_clip_logits produced"""
    import os
    from hipie_b200 import ops
    from hipie_b200.modeling.maskclip import MaskCLIP, class_tables, config_from_state_dict
    from hipie_oracle import clip as oc
    ops.set_precision(3)
    g = torch.load(os.path.join(golden_dir, "ref_maskclip.pt"), weights_only=False)
    model = oc.init_clip_(oc.CLIP(g["cfg"]), g["seed"])
    sd = model.state_dict()
    assert config_from_state_dict(sd) == g["cfg"]
    mc = MaskCLIP(sd, device=cuda)
    assert abs(mc.logit_scale - g["logit_scale"]) < 1e-4
    text_unit, emb_t = mc.build_text_embed(g["ids"])
    assert (emb_t.cpu() - g["text_embed"]).abs().max() < 1e-4 * g["text_embed"].abs().max()
    emb = mc.get_mask_embed(g["image"][0].to(cuda), g["mask"][0].to(cuda))
    assert (emb.cpu() - g["mask_embed"][0]).abs().max() < 2e-4 * g["mask_embed"].abs().max()
    prompts, seg, overlap = class_tables(g["test_labels"], g["train_labels"], cuda)
    assert prompts == g["labels"] and overlap.tolist() == [1, 0, 0, 1, 1]
    raw = mc.raw_logits(emb, text_unit)
    scores = torch.logit(g["pred_open_prob"].clamp(1e-6, 1 - 1e-6)).to(cuda)          # temp 0: p_model = sigmoid(scores) = pred_open_prob
    for mode, ref in g["fused"].items():
        got = ops.clip_fuse(raw, emb, mc.logit_scale, seg, scores, 0.0, overlap, 0.35, 0.7, mode == "ADD", 0).cpu()
        assert (got - ref).abs().max() < 2e-3, mode


def test_model_with_maskclip_matches_oracle(cuda):
    """tiny HIPIE + tiny CLIP, MODEL.CLIP.ENABLED semantics: both re-scoring sites (foreground NMS scores, panoptic / semantic class
    probabilities) against the CPU oracle with the same selections forced"""
    from hipie_oracle import clip as oc
    from hipie_oracle import hparams, synth
    from hipie_oracle.model import HipieOracle
    from hipie_b200 import ops
    from hipie_b200.modeling.hipie_img import HIPIE_IMG
    torch.manual_seed(5)
    hp = hparams.get("vit_tiny")
    oracle = HipieOracle(hp).eval()
    synth.perturb_(oracle, seed=6)
    clip = oc.init_clip_(oc.CLIP(oc.TINY), 41)
    C = 7
    inputs, ids, am = synth.make_batch(2, 96, 128, C, hp["max_query_len"], seed=8)
    names = ["person,people", "wall", "zebra,okapi", "sky", "traffic light,signal", "tree", "okra,gumbo,lady finger"]
    test_labels = [{"id": i + 1, "name": n} for i, n in enumerate(names)]
    train_labels = [{"id": 1, "name": "person,child"}, {"id": 2, "name": "sky,clouds"}, {"id": 3, "name": "tree"}]
    flat = [t for ls in oc.prompt_labels([n.split(",") for n in names]) for t in ls]
    pids = oc.synth_clip_tokenize(flat, oc.TINY["text_ctx"], oc.TINY["vocab"])
    for x, i, a in zip(inputs, ids, am):
        x.update(input_ids=i, attention_mask=a, open_seg_labels=test_labels, clip_prompt_ids=pids)
    oracle.attach_clip(oc.MaskCLIPOracle(clip), train_labels)
    with torch.no_grad():
        res_o, out_o = oracle(inputs, ids, am)
    ops.set_precision(3)
    hp2 = dict(hp, clip_enabled=True)
    model = HIPIE_IMG(hp=hp2, state_dict=oracle.state_dict(), device="cuda:0")
    with pytest.raises(RuntimeError):
        model(inputs)                                             # enabled but no CLIP weights attached
    model.attach_clip(clip.state_dict(), train_labels)
    forced = {"topk_fg": out_o["aux"]["topk"].to(cuda), "topk_md": out_o["md"]["topk"].to(cuda)}
    res_g = model(inputs, forced=forced)
    for ro, rg in zip(res_o, res_g):
        io, ig = ro["instances_post"], rg["instances"]
        assert torch.equal(io["pred_classes"], ig.pred_classes.cpu())
        assert (io["scores"] - ig.scores.cpu()).abs().max() < 2e-4
        so, sg = ro["sem_seg"], rg["sem_seg"].cpu()
        assert (so - sg).abs().max() < 5e-3 and (so.argmax(0) == sg.argmax(0)).float().mean() > 0.999
        assert [s["category_id"] for s in ro["panoptic_seg"][1]] == [s["category_id"] for s in rg["panoptic_seg"][1]]
