"""Parameter inventory of HIPIE_IMG under the reference's state_dict key names, and a seeded random
initialiser for synthetic runs (no checkpoints are available offline).

Key names follow the attribute names of /root/reference/projects/HIPIE/hipie/hipie_img.py:51-262 and the
modules it builds (SURVEY.md §8b2): `detr.detr.backbone.0.backbone.*`, `detr.detr.transformer.*`,
`detr.detr.{input_proj,class_embed,bbox_embed,iou_head}.*`, `detr.{controller,mask_head,resizer}.*`,
`detr.mask_dino.{pixel_decoder,predictor}.*`, `detr.mask_dino_cls_embed.*`, `text_encoder.body.model.*`.
Aliased modules of the reference (decoder.bbox_embed / decoder.class_embed / predictor.bbox_embed.N) are listed
in ALIASES so a reference checkpoint loads with its duplicates ignored.
"""
import math
from collections import OrderedDict

import torch


class Spec:
    def __init__(self):
        self.shapes = OrderedDict()
        self.kinds = {}

    def add(self, name, shape, kind="w"):
        self.shapes[name] = tuple(shape)
        self.kinds[name] = kind

    def linear(self, p, out_f, in_f, bias=True):
        self.add(p + ".weight", (out_f, in_f))
        if bias:
            self.add(p + ".bias", (out_f,), "b")

    def norm(self, p, c):
        self.add(p + ".weight", (c,), "one")
        self.add(p + ".bias", (c,), "zero")

    def conv(self, p, out_c, in_c, k, bias=True):
        self.add(p + ".weight", (out_c, in_c, k, k))
        if bias:
            self.add(p + ".bias", (out_c,), "b")

    def mlp(self, p, dims):
        for i in range(len(dims) - 1):
            self.linear(f"{p}.layers.{i}", dims[i + 1], dims[i])

    def msda(self, p, d=256):
        self.linear(p + ".sampling_offsets", 256, d)
        self.linear(p + ".attention_weights", 128, d)
        self.linear(p + ".value_proj", d, d)
        self.linear(p + ".output_proj", d, d)

    def vl_align(self, p, lang, d):
        self.linear(p + ".dot_product_projection_text", d, lang)
        self.add(p + ".log_scale", (1,), "zero")
        self.add(p + ".bias_lang", (lang,), "b")
        self.add(p + ".bias0", (1,), "prior")

    def mha(self, p, d):
        self.add(p + ".in_proj_weight", (3 * d, d))
        self.add(p + ".in_proj_bias", (3 * d,), "b")
        self.linear(p + ".out_proj", d, d)

    def input_proj(self, p, d, ch):
        """1x1 conv + GN on each of the three backbone levels, then the 3x3 stride-2 conv + GN on the last."""
        for l in range(3):
            self.conv(f"{p}.input_proj.{l}.0", d, ch[l], 1)
            self.norm(f"{p}.input_proj.{l}.1", d)
        self.conv(f"{p}.input_proj.3.0", d, ch[2], 3)
        self.norm(f"{p}.input_proj.3.1", d)

    def deformable_encoder_layer(self, p, d, ff):
        self.msda(p + ".self_attn", d)
        self.norm(p + ".norm1", d)
        self.linear(p + ".linear1", ff, d)
        self.linear(p + ".linear2", d, ff)
        self.norm(p + ".norm2", d)

    def deformable_decoder_layer(self, p, d, ff):
        self.msda(p + ".cross_attn", d)
        self.norm(p + ".norm1", d)
        self.mha(p + ".self_attn", d)
        self.norm(p + ".norm2", d)
        self.linear(p + ".linear1", ff, d)
        self.linear(p + ".linear2", d, ff)
        self.norm(p + ".norm3", d)


def backbone_channels(hp):
    if hp["backbone"] == "vit":
        e = hp["vit"]["embed_dim"]
        return [e // 2, e, e]
    return [512, 1024, 2048]


def build_spec(hp) -> Spec:
    s = Spec()
    d = hp.get("hidden_dim", 256)
    lang = hp.get("lang_dim", 768)
    ff = hp.get("dim_ff", 2048)
    bb = "detr.detr.backbone.0.backbone"
    if hp["backbone"] == "vit":
        v = hp["vit"]
        e, hd = v["embed_dim"], v["embed_dim"] // v["num_heads"]
        grid = v["img_size"] // v["patch_size"]
        s.conv(bb + ".patch_embed.proj", e, 3, v["patch_size"])
        s.add(bb + ".pos_embed", (1, (v["pretrain_img_size"] // v["patch_size"]) ** 2 + 1, e), "small")
        for i in range(v["depth"]):
            b = f"{bb}.blocks.{i}"
            sz = v["window_size"] if i in v["window_block_indexes"] else grid
            s.norm(b + ".norm1", e)
            s.linear(b + ".attn.qkv", 3 * e, e)
            s.linear(b + ".attn.proj", e, e)
            s.add(b + ".attn.rel_pos_h", (2 * sz - 1, hd), "small")
            s.add(b + ".attn.rel_pos_w", (2 * sz - 1, hd), "small")
            s.norm(b + ".norm2", e)
            s.linear(b + ".mlp.fc1", 4 * e, e)
            s.linear(b + ".mlp.fc2", e, 4 * e)
        s.add(bb + ".fpn1.0.weight", (e, e // 2, 2, 2))
        s.add(bb + ".fpn1.0.bias", (e // 2,), "b")
    else:
        def convnorm(p, cout, cin, k):
            s.add(p + ".weight", (cout, cin, k, k))
            s.add(p + ".norm.weight", (cout,), "one")
            s.add(p + ".norm.bias", (cout,), "b")
            s.add(p + ".norm.running_mean", (cout,), "b")
            s.add(p + ".norm.running_var", (cout,), "var")
        convnorm(bb + ".stem.conv1", 64, 3, 7)
        cin, bott, cout = 64, 64, 256
        for name, n in (("res2", 3), ("res3", 4), ("res4", 6), ("res5", 3)):
            for i in range(n):
                p = f"{bb}.{name}.{i}"
                if cin != cout:
                    convnorm(p + ".shortcut", cout, cin, 1)
                convnorm(p + ".conv1", bott, cin, 1)
                convnorm(p + ".conv2", bott, bott, 3)
                convnorm(p + ".conv3", cout, bott, 1)
                cin = cout
            bott *= 2
            cout *= 2
    ch = backbone_channels(hp)
    dd = "detr.detr"
    s.input_proj(dd, d, ch)
    t = dd + ".transformer"
    s.add(t + ".level_embed", (4, d), "normal1")
    vl = t + ".encoder.vl_layers.0.b_attn"
    s.add(vl + ".gamma_v", (d,), "gamma")
    s.add(vl + ".gamma_l", (lang,), "gamma")
    s.norm(vl + ".layer_norm_v", d)
    s.norm(vl + ".layer_norm_l", lang)
    E = hp.get("vl_hidden", 2048)
    for n, (o, i) in {"v_proj": (E, d), "l_proj": (E, lang), "values_v_proj": (E, d), "values_l_proj": (E, lang),
                      "out_v_proj": (d, E), "out_l_proj": (lang, E)}.items():
        s.linear(f"{vl}.attn.{n}", o, i)
    for i in range(hp.get("enc_layers", 6)):
        s.deformable_encoder_layer(f"{t}.encoder.layers.{i}", d, ff)
    for i in range(hp.get("dec_layers", 6)):
        s.deformable_decoder_layer(f"{t}.decoder.layers.{i}", d, ff)
    s.mlp(t + ".decoder.ref_point_head", [2 * d, d, d])
    s.add(t + ".tgt_embed.weight", (hp.get("num_queries", 900), d), "normal1")
    s.add(t + ".tgt_embed_bg.weight", (hp.get("num_bg", 10), d), "normal1")
    s.add(t + ".bg_query_refs.weight", (hp.get("num_bg", 10), 4), "normal1")
    s.linear(t + ".enc_output", d, d)
    s.norm(t + ".enc_output_norm", d)
    s.linear(t + ".resizer.fc", d, lang)
    s.norm(t + ".resizer.layer_norm", d)
    nd = hp.get("dec_layers", 6)
    for i in range(nd):
        s.vl_align(f"{dd}.class_embed.{i}", lang, d)
    s.linear(f"{dd}.class_embed.{nd}.body", 1, d)
    for i in range(nd + 1):
        s.mlp(f"{dd}.bbox_embed.{i}", [d, d, d, 4])
    for i in range(nd):
        s.linear(f"{dd}.iou_head.{i}", 1, d)
    s.mlp("detr.controller", [d, d, d, 169])
    mh = "detr.mask_head"
    s.conv(mh + ".lay1", d // 4, d, 3)
    s.conv(mh + ".lay2", d // 32, d // 4, 3)
    s.conv(mh + ".lay3", d, d, 3)
    s.conv(mh + ".lay4", d, d, 3)
    s.conv(mh + ".jia_dcn", d, d, 3)
    s.linear("detr.resizer.fc", d, lang)
    s.norm("detr.resizer.layer_norm", d)
    # ---- MaskDINO branch
    pd = "detr.mask_dino.pixel_decoder"
    mff = hp.get("md_dim_ff", 2048)
    s.input_proj(pd, d, ch)
    for i in range(hp.get("md_enc_layers", 6)):
        s.deformable_encoder_layer(f"{pd}.transformer.encoder.layers.{i}", d, mff)
    s.add(pd + ".transformer.level_embed", (4, d), "normal1")       # after the encoder layers, unlike DETR's
    s.add(pd + ".mask_features.0.weight", (d, d, 2, 2))
    s.add(pd + ".mask_features.0.bias", (d,), "b")
    s.norm(pd + ".mask_features.1", d)
    s.conv(pd + ".mask_features.3", d, d, 1)
    s.add(pd + ".adapter_1.weight", (d, ch[0], 1, 1))
    s.norm(pd + ".adapter_1.norm", d)
    s.add(pd + ".layer_1.weight", (d, d, 3, 3))
    s.norm(pd + ".layer_1.norm", d)
    pr = "detr.mask_dino.predictor"
    s.linear(pr + ".enc_output", d, d)
    s.norm(pr + ".enc_output_norm", d)
    s.linear(pr + ".class_embed", d, d)
    s.linear(pr + ".resizer.fc", d, lang)
    s.norm(pr + ".resizer.layer_norm", d)
    s.mlp(pr + ".mask_embed", [d, d, d, d])
    s.norm(pr + ".decoder_norm", d)
    for i in range(hp.get("md_dec_layers", 9)):
        s.deformable_decoder_layer(f"{pr}.decoder.layers.{i}", d, mff)
    s.mlp(pr + ".decoder.ref_point_head", [2 * d, d, d])
    s.mlp(pr + "._bbox_embed", [d, d, d, 4])
    for i in range(hp.get("md_dec_layers", 9) + 2):
        s.vl_align(f"detr.mask_dino_cls_embed.{i}", lang, d)
    # ---- BERT
    b = hp["bert"]
    te = "text_encoder.body.model"
    s.add(te + ".embeddings.word_embeddings.weight", (b["vocab"], b["hidden"]), "small")
    s.add(te + ".embeddings.position_embeddings.weight", (b["max_pos"], b["hidden"]), "small")
    s.add(te + ".embeddings.token_type_embeddings.weight", (2, b["hidden"]), "small")
    s.norm(te + ".embeddings.LayerNorm", b["hidden"])
    for i in range(b["layers"]):
        p = f"{te}.encoder.layer.{i}"
        for n in ("query", "key", "value"):
            s.linear(f"{p}.attention.self.{n}", b["hidden"], b["hidden"])
        s.linear(p + ".attention.output.dense", b["hidden"], b["hidden"])
        s.norm(p + ".attention.output.LayerNorm", b["hidden"])
        s.linear(p + ".intermediate.dense", b["inter"], b["hidden"])
        s.linear(p + ".output.dense", b["hidden"], b["inter"])
        s.norm(p + ".output.LayerNorm", b["hidden"])
    return s


def alias_prefixes(hp):
    """(alias prefix -> canonical prefix) for modules the reference registers more than once."""
    nd = hp.get("dec_layers", 6)
    al = {}
    for i in range(nd + 1):
        al[f"detr.detr.transformer.decoder.bbox_embed.{i}."] = f"detr.detr.bbox_embed.{i}."
        al[f"detr.detr.transformer.decoder.class_embed.{i}."] = f"detr.detr.class_embed.{i}."
    for i in range(hp.get("md_dec_layers", 9)):
        al[f"detr.mask_dino.predictor.bbox_embed.{i}."] = "detr.mask_dino.predictor._bbox_embed."
        al[f"detr.mask_dino.predictor.decoder.bbox_embed.{i}."] = "detr.mask_dino.predictor._bbox_embed."
    al["detr.mask_dino.predictor.decoder.norm."] = "detr.mask_dino.predictor.decoder_norm."
    return al


def canonical_name(name, hp, _cache={}):
    key = (hp.get("dec_layers", 6), hp.get("md_dec_layers", 9))      # everything alias_prefixes depends on (not id(hp): ids are reused)
    if key not in _cache:
        _cache[key] = alias_prefixes(hp)
    for a, c in _cache[key].items():
        if name.startswith(a):
            return c + name[len(a):]
    return name


def random_state_dict(hp, seed=0, device="cpu"):
    """Seeded synthetic weights of the right shapes: N(0, 1/sqrt(fan_in)) matrices, small random biases,
    unit norms — every stage is input dependent (sampling offsets and attention logits included)."""
    spec = build_spec(hp)
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()
    prior = -math.log((1 - 0.01) / 0.01)
    for name, shape in spec.shapes.items():
        kind = spec.kinds[name]
        if kind == "w":
            fan_in = 1
            for v in shape[1:]:
                fan_in *= v
            if name.endswith("fpn1.0.weight") or name.endswith("mask_features.0.weight"):
                fan_in = shape[0]          # ConvTranspose2d: (in, out, k, k)
            std = 1.0 / math.sqrt(max(fan_in, 1))
            if "sampling_offsets.weight" in name:
                std = 0.02
            t = torch.randn(shape, generator=g) * std
        elif kind == "b":
            t = torch.randn(shape, generator=g) * 0.02
            if "sampling_offsets.bias" in name:     # reference grid init (ms_deform_attn.py:62-70)
                thetas = torch.arange(8, dtype=torch.float32) * (2.0 * math.pi / 8)
                grid = torch.stack([thetas.cos(), thetas.sin()], -1)
                grid = (grid / grid.abs().max(-1, keepdim=True)[0]).view(8, 1, 1, 2).repeat(1, 4, 4, 1)
                for i in range(4):
                    grid[:, :, i, :] *= i + 1
                t = grid.view(-1)
        elif kind == "one":
            t = torch.ones(shape) + torch.randn(shape, generator=g) * 0.02
        elif kind == "zero":
            t = torch.randn(shape, generator=g) * 0.02 if len(shape) and shape[0] > 1 else torch.zeros(shape)
        elif kind == "small":
            t = torch.randn(shape, generator=g) * 0.02
        elif kind == "normal1":
            t = torch.randn(shape, generator=g)
            if name.endswith("bg_query_refs.weight"):
                t = t * 0.5
        elif kind == "gamma":
            t = torch.full(shape, 1.0 / hp.get("enc_layers", 6))
        elif kind == "prior":
            t = torch.full(shape, prior)
        elif kind == "var":
            t = 1.0 + torch.rand(shape, generator=g) * 0.2
        else:
            raise ValueError(kind)
        sd[name] = t.to(device)
    return sd
