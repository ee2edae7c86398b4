"""MaskCLIP re-scoring on the GPU (SURVEY.md row a22 / f2).

Reference: projects/HIPIE/hipie/open_vocab/clip.py:243-383 (`MaskCLIP`: mask tokens = copies of the CLS token that attend to CLS and
to the patches their mask touches; nobody attends to them), open_vocab/helper.py:79-130, hipie_img.py:811-868 (`get_clip_logits`)
on top of open_clip's CLIP ViT (ViT-L/14-336 by default, MODEL.CLIP.NAME; third-party `open_clip_torch==2.0.2`).

Weights arrive under open_clip's state_dict names (`visual.conv1.weight`, `visual.transformer.resblocks.N.attn.in_proj_weight`, ...,
`text_projection`, `logit_scale`), e.g. `open_clip.create_model(name, pretrained="openai").state_dict()` saved with torch.save.
The forward is this repo's kernels only: hipie_clip_patches -> hipie_gemm (patch embedding) -> per layer hipie_layernorm, hipie_gemm
(qkv), hipie_attention with the per-query key bit mask (keys = the image tokens only: K / V of the mask tokens are never needed),
hipie_gemm (out_proj + residual), hipie_layernorm, hipie_gemm (c_fc + QuickGELU), hipie_gemm (c_proj + residual) -> ln_post +
projection of the mask tokens -> hipie_clip_fuse.  No CPU path.
"""
import math

import torch

from .. import ops

OPENAI_MEAN = (0.48145466, 0.4578275, 0.40821073)
OPENAI_STD = (0.26862954, 0.26130258, 0.27577711)


def config_from_state_dict(sd):
    """Model geometry from the tensor shapes (what open_clip's load_openai_model does for OpenAI checkpoints)."""
    width = sd["visual.conv1.weight"].shape[0]
    patch = sd["visual.conv1.weight"].shape[-1]
    grid = int(round((sd["visual.positional_embedding"].shape[0] - 1) ** 0.5))
    layers = len({k.split(".")[3] for k in sd if k.startswith("visual.transformer.resblocks.")})
    tlayers = len({k.split(".")[2] for k in sd if k.startswith("transformer.resblocks.")})
    twidth = sd["ln_final.weight"].shape[0]
    return dict(embed_dim=sd["text_projection"].shape[1], image_size=grid * patch, patch=patch, width=width, layers=layers, heads=width // 64,
                text_ctx=sd["positional_embedding"].shape[0], vocab=sd["token_embedding.weight"].shape[0], text_width=twidth,
                text_heads=twidth // 64, text_layers=tlayers)


class MaskCLIP:
    def __init__(self, state_dict, device="cuda:0", cfg=None):
        if not torch.cuda.is_available():
            raise RuntimeError("hipie_b200 MaskCLIP: CUDA (sm_90a) only")
        self.device = torch.device(device)
        sd = {k: v.detach().to(self.device, torch.float32) for k, v in state_dict.items() if v.dtype.is_floating_point}
        self.cfg = dict(cfg) if cfg is not None else config_from_state_dict(sd)
        c = self.cfg
        if c["width"] % 64 or c["text_width"] % 64:
            raise ValueError("CLIP widths must be multiples of the head width 64 (clip.py:320)")
        self.sd = sd
        self.S, self.P, self.G = c["image_size"], c["patch"], c["image_size"] // c["patch"]
        self.n_img = self.G * self.G + 1
        k = 3 * self.P * self.P
        kp = (k + 7) // 8 * 8                                    # GEMM rows are 16-byte aligned: pad K with zero columns
        w = torch.zeros(c["width"], kp, device=self.device)
        w[:, :k] = sd["visual.conv1.weight"].reshape(c["width"], k)
        self.w_patch = ops.split_weight(w)
        self.vis = [self._block("visual.transformer.resblocks.%d" % i) for i in range(c["layers"])]
        self.txt = [self._block("transformer.resblocks.%d" % i) for i in range(c["text_layers"])]
        self.w_proj = ops.split_weight(sd["visual.proj"].t().contiguous())                 # x @ proj
        self.w_tproj = ops.split_weight(sd["text_projection"].t().contiguous())
        self.logit_scale = min(math.exp(float(sd["logit_scale"])), 100.0)                  # clip.py:252-255
        self.cache_text = {}
        # causal mask of the text tower as key-mask bits: query t may not see keys > t
        ctx = c["text_ctx"]
        words = (ctx + 31) // 32
        cm = torch.zeros(ctx, words * 32, dtype=torch.bool)
        cm[:, :ctx] = torch.ones(ctx, ctx, dtype=torch.bool).triu(1)
        self.causal_bits = self._pack_bits(cm).to(self.device)

    @staticmethod
    def _pack_bits(m):
        """(R, 32 * words) bool -> (R, words) int32, bit k of word j = column 32 j + k"""
        R, n = m.shape
        sh = torch.arange(32, dtype=torch.int64)
        v = (m.view(R, n // 32, 32).to(torch.int64) << sh).sum(-1)
        return torch.where(v >= 2 ** 31, v - 2 ** 32, v).to(torch.int32)

    def _block(self, p):
        sd = self.sd
        return dict(ln1=(sd[p + ".ln_1.weight"], sd[p + ".ln_1.bias"]), ln2=(sd[p + ".ln_2.weight"], sd[p + ".ln_2.bias"]),
                    qkv=(ops.split_weight(sd[p + ".attn.in_proj_weight"]), sd[p + ".attn.in_proj_bias"].contiguous()),
                    out=(ops.split_weight(sd[p + ".attn.out_proj.weight"]), sd[p + ".attn.out_proj.bias"].contiguous()),
                    fc=(ops.split_weight(sd[p + ".mlp.c_fc.weight"]), sd[p + ".mlp.c_fc.bias"].contiguous()),
                    proj=(ops.split_weight(sd[p + ".mlp.c_proj.weight"]), sd[p + ".mlp.c_proj.bias"].contiguous()))

    # ------------------------------------------------------------ transformer (open_clip ResidualAttentionBlock, pre-LN, QuickGELU)
    def _layers(self, x, blocks, B, T, width, kv_row0, Tk, key_mask):
        """x (B*T, width) f32 residual stream.  Keys / values are rows [kv_row0, kv_row0 + Tk) of every sequence."""
        heads, hd = width // 64, 64
        for blk in blocks:
            _, xn, _ = ops.layernorm(x, blk["ln1"][0], blk["ln1"][1], 1e-5)
            _, qkv, _ = ops.gemm(xn, blk["qkv"][0], bias=blk["qkv"][1], want_f32=False, want_split=True)             # (B*T, 3 width)
            sl = lambda c, r0: qkv[r0:, c * width:(c + 1) * width]
            st = (T * 3 * width, 3 * width, hd)
            _, ao = ops.attention(sl(0, 0), sl(1, kv_row0), sl(2, kv_row0), B, heads, T, Tk, hd, st, st, st, hd ** -0.5, key_mask=key_mask)
            ops.gemm(ao.view(B * T, width), blk["out"][0], bias=blk["out"][1], residual=x, out_f32=x)
            _, xn2, _ = ops.layernorm(x, blk["ln2"][0], blk["ln2"][1], 1e-5)
            _, hmid, _ = ops.gemm(xn2, blk["fc"][0], bias=blk["fc"][1], act=ops.ACT_QUICK_GELU, want_f32=False, want_split=True)
            ops.gemm(hmid, blk["proj"][0], bias=blk["proj"][1], residual=x, out_f32=x)
        return x

    # ------------------------------------------------------------ text tower (CLIP.encode_text; clip.py:29-73 after the tokenizer)
    @torch.no_grad()
    def build_text_embed(self, token_ids, cache_key=None):
        """token_ids (N, context_length) int64 (open_clip.tokenize output: SOT ... EOT, zero padded; EOT is the highest id).
        Returns the UNIT-norm prompt embeddings (N, D) as a BF2 GEMM operand + the f32 tensor; cached by `cache_key`
        (clip.py:363-373 caches by the label list)."""
        if cache_key is not None and cache_key in self.cache_text:
            return self.cache_text[cache_key]
        c = self.cfg
        ids = token_ids.to(self.device)
        N, ctx = ids.shape
        assert ctx == c["text_ctx"]
        x = (self.sd["token_embedding.weight"][ids] + self.sd["positional_embedding"]).reshape(N * ctx, c["text_width"]).contiguous()
        km = self.causal_bits.unsqueeze(0).expand(N, -1, -1).contiguous()
        x = self._layers(x, self.txt, N, ctx, c["text_width"], 0, ctx, km)
        eot = ids.argmax(dim=-1) + torch.arange(N, device=self.device) * ctx
        _, xs, _ = ops.layernorm(x[eot].contiguous(), self.sd["ln_final.weight"], self.sd["ln_final.bias"], 1e-5)
        emb, _, _ = ops.gemm(xs, self.w_tproj)
        unit = emb / emb.norm(dim=-1, keepdim=True).clamp_min(1e-12)          # F.normalize of clip.py:354 (once per vocabulary)
        out = (ops.split_weight(unit), emb)
        if cache_key is not None:
            self.cache_text[cache_key] = out
        return out

    # ------------------------------------------------------------ image + mask tokens (clip.py:257-349)
    @torch.no_grad()
    def get_mask_embed(self, image01, masks, up=1, crop=None):
        """image01 (3, H, W) f32 in 0..1 on the device; masks (Q, h, w) f32 logits.  up / crop: see ops.maskclip_patch_mask.
        Returns mask_embed (Q, D) f32."""
        c = self.cfg
        width, Q = c["width"], masks.shape[0]
        T = Q + self.n_img
        patches = ops.clip_patches(image01, self.S, self.P, OPENAI_MEAN, OPENAI_STD)
        tok, _, _ = ops.gemm(patches, self.w_patch)                                                        # (G*G, width)
        seq = torch.cat([self.sd["visual.class_embedding"].view(1, width), tok], 0) + self.sd["visual.positional_embedding"]
        img, _, _ = ops.layernorm(seq, self.sd["visual.ln_pre.weight"], self.sd["visual.ln_pre.bias"], 1e-5, want_f32=True, want_split=False)
        x = torch.cat([img[0:1].expand(Q, -1), img], 0).contiguous()                                       # mask tokens first (:277-279)
        words = (self.n_img + 31) // 32
        bits = torch.zeros((T, words), dtype=torch.int32, device=self.device)      # image-token rows: nothing masked (keys = image tokens)
        ops.maskclip_patch_mask(masks, self.S, self.P, bits, key_offset=1, up=up, crop=crop)
        x = self._layers(x, self.vis, 1, T, width, Q, self.n_img, bits.view(1, T, words))
        _, xs, _ = ops.layernorm(x[:Q].contiguous(), self.sd["visual.ln_post.weight"], self.sd["visual.ln_post.bias"], 1e-5)
        emb, _, _ = ops.gemm(xs, self.w_proj)
        return emb

    @torch.no_grad()
    def raw_logits(self, mask_embed, text_unit):
        """mask_embed . unit(text)^T; hipie_clip_fuse applies 1 / |mask_embed| and the logit scale."""
        raw, _, _ = ops.gemm(ops.split(mask_embed), text_unit)
        return raw


def class_tables(test_labels, train_labels, device):
    """hipie_img.py:818-830 + helper.py:112-130: prompt list ("a photo of a {synonym}."), prompt offsets per class and the seen-class
    flags (a test class is 'seen' when it shares a synonym with a training class)."""
    names = [x["name"].split(",") for x in test_labels]
    prompts = [["a photo of a %s." % l for l in ls] for ls in names]
    train = {l for x in train_labels for l in x["name"].split(",")}
    seg = [0]
    for ls in prompts:
        seg.append(seg[-1] + len(ls))
    overlap = [int(not train.isdisjoint(set(ls))) for ls in names]
    return (prompts, torch.tensor(seg, dtype=torch.int32, device=device), torch.tensor(overlap, dtype=torch.int8, device=device))
