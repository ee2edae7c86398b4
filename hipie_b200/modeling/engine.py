"""CUDA engine: HIPIE's eval forward expressed over the C-ABI operators (hipie_b200.ops).

Functional, driven by a flat weight dictionary under the reference's state_dict names.  Layout choices are
GPU-first rather than a translation of the reference modules:
  * activations are token-major / NHWC fp32 "residual streams"; everything that feeds a tensor-core GEMM is
    produced directly as bf16 hi/lo planes by the preceding kernel's epilogue (LayerNorm, GELU, attention …),
  * convolutions are GEMMs over NHWC rows (1x1: plain; kxk: im2col; ConvTranspose 2x2: GEMM + pixel shuffle),
  * windowed ViT blocks use a row map in the LayerNorm / proj-GEMM epilogues instead of partition copies,
  * sampling-offset and attention-weight linears of MSDeformAttn are one fused GEMM (N = 384) feeding the fused
    softmax+location+gather kernel; the value map is projected once per layer,
  * the mask-embed contraction runs transposed (M = H*W pixels, N = queries) so the NHWC pixel features are the
    K-major A operand and the (Q, H, W) output is written coalesced straight from the accumulator.
torch is used for allocation, views and a few tiny input-independent / index ops (top-k, gather, sine tables).

Reference call sites are cited next to each stage (H = /root/reference/projects/HIPIE/hipie).
"""
import math

import types

import torch
import torch.nn.functional as F

from .. import ops
from ..ops import BF2
from . import params as P


# ================================================================ weights
class WeightStore:
    def __init__(self, state_dict, hp, device):
        self.hp = hp
        self.device = device
        self.f = {}
        for k, v in state_dict.items():
            c = P.canonical_name(k, hp) if hp is not None else k       # hp None: names are used as given (the SAM weights)
            if c not in self.f:
                self.f[c] = v.detach().to(device=device, dtype=torch.float32).contiguous()
        self._c = {}

    def __getitem__(self, name):
        return self.f[name]

    def cached(self, key, fn):
        if key not in self._c:
            self._c[key] = fn()
        return self._c[key]

    def lin(self, prefix):
        """(BF2 weight (out, in), bias or None)"""
        return self.cached(("lin", prefix), lambda: (ops.split_weight(self.f[prefix + ".weight"].reshape(self.f[prefix + ".weight"].shape[0], -1)),
                                                      self.f.get(prefix + ".bias")))

    def lin_cat(self, key, prefixes):
        def mk():
            w = torch.cat([self.f[p + ".weight"] for p in prefixes], 0)
            b = torch.cat([self.f[p + ".bias"] for p in prefixes], 0)
            return ops.split_weight(w), b.contiguous()
        return self.cached(("lincat", key), mk)

    def mat(self, key, fn):
        """BF2 of an arbitrary derived matrix."""
        return self.cached(("mat", key), lambda: ops.split_weight(fn()))

    def conv_kxk(self, prefix):
        def mk():
            w = self.f[prefix + ".weight"]
            return ops.split_weight(w.permute(0, 2, 3, 1).reshape(w.shape[0], -1)), self.f.get(prefix + ".bias")
        return self.cached(("convk", prefix), mk)

    def convT2(self, prefix):
        def mk():
            w = self.f[prefix + ".weight"]                     # (in, out, 2, 2)
            wk = w.permute(2, 3, 1, 0).reshape(4 * w.shape[1], w.shape[0])   # rows (dy, dx, co)
            return ops.split_weight(wk), self.f[prefix + ".bias"].repeat(4).contiguous()
        return self.cached(("convT", prefix), mk)


def _get_rel_pos_table(q_size, k_size, rel_pos):
    """get_rel_pos (H/backbone/utils.py:63-93) -> (q, k, C); input independent, evaluated once per grid size."""
    max_rel_dist = int(2 * max(q_size, k_size) - 1)
    if rel_pos.shape[0] != max_rel_dist:
        r = F.interpolate(rel_pos.reshape(1, rel_pos.shape[0], -1).permute(0, 2, 1), size=max_rel_dist, mode="linear")
        r = r.reshape(-1, max_rel_dist).permute(1, 0)
    else:
        r = rel_pos
    q_coords = torch.arange(q_size, device=rel_pos.device)[:, None] * max(k_size / q_size, 1.0)
    k_coords = torch.arange(k_size, device=rel_pos.device)[None, :] * max(q_size / k_size, 1.0)
    rel = (q_coords - k_coords) + (k_size - 1) * max(q_size / k_size, 1.0)
    return r[rel.long()]


def _abs_pos(abs_pos, hw):
    """get_abs_pos (utils.py:128-157), cls token dropped, bicubic resize; input independent."""
    h, w = hw
    abs_pos = abs_pos[:, 1:]
    size = int(math.sqrt(abs_pos.shape[1]))
    if size != h or size != w:
        a = F.interpolate(abs_pos.reshape(1, size, size, -1).permute(0, 3, 1, 2), size=(h, w), mode="bicubic", align_corners=False)
        return a.permute(0, 2, 3, 1).reshape(h * w, -1).contiguous()
    return abs_pos.reshape(h * w, -1).contiguous()


def _sine_pos(mask, num_pos_feats, offset):
    """PositionEmbeddingSine (H/models/deformable_detr/position_encoding.py:20-56 with offset -0.5;
    H/models/maskdino/pixel_decoder/position_encoding.py:15-55 with offset 0) -> (B, h*w, 2*num_pos_feats)."""
    not_mask = ~mask
    y_embed = not_mask.cumsum(1, dtype=torch.float32)
    x_embed = not_mask.cumsum(2, dtype=torch.float32)
    eps, scale = 1e-6, 2 * math.pi
    y_embed = (y_embed + offset) / (y_embed[:, -1:, :] + eps) * scale
    x_embed = (x_embed + offset) / (x_embed[:, :, -1:] + eps) * scale
    dim_t = torch.arange(num_pos_feats, dtype=torch.float32, device=mask.device)
    dim_t = 10000 ** (2 * torch.div(dim_t, 2, rounding_mode="floor") / num_pos_feats)
    pos_x = x_embed[:, :, :, None] / dim_t
    pos_y = y_embed[:, :, :, None] / dim_t
    pos_x = torch.stack((pos_x[..., 0::2].sin(), pos_x[..., 1::2].cos()), dim=4).flatten(3)
    pos_y = torch.stack((pos_y[..., 0::2].sin(), pos_y[..., 1::2].cos()), dim=4).flatten(3)
    return torch.cat((pos_y, pos_x), dim=3).flatten(1, 2)


def _sine_embed_points(pos, num_pos_feats=128):
    """get_sine_pos_embed / gen_sineembed_for_position ([y, x, w, h] order; deformable_transformer_dino.py:636-670,
    maskdino/utils/utils.py:74-100).  pos (..., 4) -> (..., 512)."""
    scale = 2 * math.pi
    dim_t = torch.arange(num_pos_feats, dtype=torch.float32, device=pos.device)
    dim_t = 10000 ** (2 * torch.div(dim_t, 2, rounding_mode="floor") / num_pos_feats)

    def emb(v):
        p = (v * scale)[..., None] / dim_t
        return torch.stack((p[..., 0::2].sin(), p[..., 1::2].cos()), dim=-1).flatten(-2)

    return torch.cat([emb(pos[..., 1]), emb(pos[..., 0]), emb(pos[..., 2]), emb(pos[..., 3])], dim=-1)


def inverse_sigmoid(x, eps=1e-5):
    x = x.clamp(min=0, max=1)
    return torch.log(x.clamp(min=eps) / (1 - x).clamp(min=eps))


# ================================================================ engine
class Engine:
    def __init__(self, state_dict, hp, device="cuda:0"):
        self.hp = hp
        self.device = torch.device(device)
        self.W = WeightStore(state_dict, hp, self.device)
        self._maps = {}
        self._bufs = {}
        self.bf16_value_map = False     # fast mode: MSDeformAttn value map stored as bf16
        self.use_tc_attention = True    # wgmma flash attention for the global ViT blocks
        self.attn_fp16 = True           # precision map (DESIGN.md 3): QK^T / PV / rel-pos of the ViT attention run as ONE fp16 MMA pass
        self.qkv_f16x2 = True           # ... and the qkv linears feeding it as TWO fp16 passes (LN output one fp16 plane, W fp16 hi + lo)
        self.fp16_value_map = False     # value maps of the deformable ENCODERS (Lq == S) as one fp16 plane (msda_layer): measured and REJECTED
                                        # (DESIGN.md 3: the proposal scores move by 1.9e-4 and re-rank the two-stage top-k; 78 % instance matches)
        self.mlp_f16e4m3 = True         # fc1 / fc2 of the ViT blocks: fp16 hi x hi pass + ONE e4m3 pass for both cross terms (gemm prec 6)
        self.taps = None                # parity harness: {"blocks": (7, 15, 31)} -> residual stream copies "vit.block<i>"

    # ------------------------------------------------------------ helpers
    def _window_maps(self, B, gh, gw, ws):
        key = (B, gh, gw, ws)
        if key not in self._maps:
            Hp, Wp = (gh + ws - 1) // ws * ws, (gw + ws - 1) // ws * ws
            nwx = Wp // ws
            nW = (Hp // ws) * nwx
            dev = self.device
            b = torch.arange(B, device=dev)[:, None, None]
            y = torch.arange(gh, device=dev)[None, :, None]
            x = torch.arange(gw, device=dev)[None, None, :]
            row = (b * nW + (y // ws) * nwx + x // ws) * (ws * ws) + (y % ws) * ws + (x % ws)
            tok2win = row.reshape(-1).int().contiguous()
            win2tok = torch.full((B * nW * ws * ws,), -1, dtype=torch.int32, device=dev)
            win2tok[tok2win.long()] = torch.arange(B * gh * gw, device=dev, dtype=torch.int32)
            self._maps[key] = (tok2win, win2tok, nW)
        return self._maps[key]

    def _dev_const(self, values, dtype):
        """Small host lists as cached device tensors (no H2D copy inside a CUDA-graph capture)."""
        key = ("const", dtype, repr(values))
        if key not in self._maps:
            self._maps[key] = torch.tensor(values, dtype=dtype, device=self.device)
        return self._maps[key]

    def _zero_planes(self, key, shape, fmt="bf16x2"):
        """Zero-initialised planes cached per key (the bf16 default carries both planes whatever the precision mode)."""
        if key not in self._bufs:
            self._bufs[key] = BF2.zeros(shape, self.device, fmt)
        return self._bufs[key]

    # ------------------------------------------------------------ ViT backbone (H/backbone/vit.py:233-374)
    def vit(self, img, normalized=False):
        """img: (B, 3, H, W) raw 0..255 fp32 (already padded; `normalized=True`: already (x - mean) / std, the D2ViT registry
        contract) -> {res3,res4,res5: (fp32 NHWC, BF2)}"""
        W, v = self.W, self.hp["vit"]
        bb = "detr.detr.backbone.0.backbone"
        B, _, H, Wd = img.shape
        P_ = v["patch_size"]
        gh, gw = H // P_, Wd // P_
        E = v["embed_dim"]
        pos = W.cached(("abs_pos", gh, gw), lambda: _abs_pos(W[bb + ".pos_embed"], (gh, gw)))
        x = self.vit_patch_embed(W, bb, img, pos, P_, normalized=normalized)
        self.vit_blocks(W, bb, x, B, gh, gw, v["depth"], v["num_heads"], v["window_block_indexes"], v["window_size"], ("fc1", "fc2"),
                        tap="vit")
        # simple FPN (vit.py:340-344,366-374): ConvT(k2,s2) / identity / maxpool
        _, xs = ops.add_split(x)
        x4 = x.view(B, gh, gw, E)
        wt, bt = W.convT2(bb + ".fpn1.0")
        g, _, _ = ops.gemm(xs, wt, bias=bt)
        r3, r3s = ops.pixel_shuffle2(g, B, gh, gw, E // 2, want_f32=True, want_split=True)
        r5, r5s = ops.maxpool2_nhwc(x4, want_f32=True, want_split=True)
        return {"res3": (r3, r3s), "res4": (x4, xs.view(B, gh, gw, E)), "res5": (r5, r5s)}

    def vit_patch_embed(self, W, prefix, img, pos, P_, normalized=False):
        """PatchEmbed + abs-pos: the (x - mean) / std normalisation is fused into the patch rows; `pos` (T, E) enters as the residual
        of the patch GEMM.  Returns the (B*T, E) fp32 residual stream."""
        B, _, H, Wd = img.shape
        T = (H // P_) * (Wd // P_)
        rows = ops.patchify(img, (0.0, 0.0, 0.0), (1.0, 1.0, 1.0), P_) if normalized else \
            ops.patchify(img, (123.675, 116.280, 103.530), (58.395, 57.120, 57.375), P_)
        wp, bp = W.lin(prefix + ".patch_embed.proj")
        E = wp.hi.shape[0]
        x, _, _ = ops.gemm(rows, wp, bias=bp, residual=pos, M=T, N=E, K=3 * P_ * P_, batch=B, lda=3 * P_ * P_, ldw=3 * P_ * P_,
                           a_bstride=T * 3 * P_ * P_, w_bstride=0, ldr=E, r_bstride=0)
        return x.view(B * T, E)

    def vit_blocks(self, W, prefix, x, B, gh, gw, depth, nh, window_blocks, ws, mlp_names, tap=None):
        """The ViTDet block loop (H/backbone/vit.py:147-230; segment_anything image_encoder.py Block is the same computation), in place
        on the (B*gh*gw, E) fp32 residual stream x.  W: weight store, prefix: `<prefix>.blocks.<i>` weight names, window_blocks: the
        windowed block indices (window ws, zero padding after norm1), mlp_names: the two MLP linears ("fc1", "fc2") / ("lin1", "lin2").
        Used by HIPIE's backbone and by the SAM image encoder."""
        fc1, fc2 = mlp_names
        T, E = gh * gw, x.shape[-1]
        hd = E // nh
        for i in range(depth):
            blk = f"{prefix}.blocks.{i}"
            windowed = i in window_blocks
            wqkv, bqkv = W.lin(blk + ".attn.qkv")
            wproj, bproj = W.lin(blk + ".attn.proj")
            if windowed:
                tok2win, win2tok, nW = self._window_maps(B, gh, gw, ws)
                Bq, Tq, qh, qw = B * nW, ws * ws, ws, ws
            else:
                Bq, Tq, qh, qw = B, T, gh, gw
            # wgmma kernel: 64-wide grids (1024-pixel inputs), 80-wide grids (1280-pixel inputs; T a multiple of lcm(256, 320)) and 14x14 windows
            tc_grid = Tq % 256 == 0 and (qw == 64 or (qw == 80 and Tq % 320 == 0))
            use_tc = self.use_tc_attention and hd == 80 and ((not windowed and tc_grid) or (windowed and ws == 14))
            f16 = use_tc and self.attn_fp16 and ops.PREC == 3
            # q, k, v are rounded to fp16 by the attention: the linears that produce them take the LayerNorm output as ONE fp16 plane
            # against fp16 hi + lo weights (two MMA passes; tools/prec_map_emulate.py: +3e-5 on the mask logits, 1-pass would cost 7e-4)
            qkv2 = f16 and self.qkv_f16x2
            if windowed:
                rows_w = B * nW * ws * ws
                if qkv2:
                    xn = self._zero_planes(("winln16", rows_w, E), (rows_w, E), "f16")       # pad rows stay exactly zero
                else:
                    xn = self._zero_planes(("winln", rows_w, E), (rows_w, E))
                ops.layernorm(x, W[blk + ".norm1.weight"], W[blk + ".norm1.bias"], 1e-6, row_map=tok2win, out_split=xn, out_fp16=qkv2)
            else:
                _, xn, _ = ops.layernorm(x, W[blk + ".norm1.weight"], W[blk + ".norm1.bias"], 1e-6, out_fp16=qkv2)
            st = (Tq * 3 * E, 3 * E, hd)
            if use_tc:
                # q,k as one GEMM (N = 2E); V emitted transposed (E, B*T) so it is the K-major B operand of P.V.  With the fp16
                # attention mode both epilogues write ONE fp16 plane instead of bf16 hi/lo (half the bytes of the qkv output).
                wsplit = ops.split_weight_f16 if qkv2 else ops.split_weight
                qprec = 4 if qkv2 else None
                wqk, bqk, wv, bv = W.cached(("qk_v", blk, qkv2), lambda: (wsplit(W[blk + ".attn.qkv.weight"][:2 * E]),
                                                                           W[blk + ".attn.qkv.bias"][:2 * E].contiguous(),
                                                                           wsplit(W[blk + ".attn.qkv.weight"][2 * E:]),
                                                                           W[blk + ".attn.qkv.bias"][2 * E:].contiguous()))
                _, qk, _ = ops.gemm(xn, wqk, bias=bqk, want_f32=False, want_split=True, out_fp16=f16, prec=qprec)   # (B*T, 2E)
                if windowed:
                    # V^T per window at a 200-column pitch (TMA box starts must be 16-byte aligned; 196 is not a multiple of 8);
                    # the 4 pad columns of every window stay zero in this cached buffer
                    if f16:
                        vt = self._zero_planes(("vtwin16", E, Bq), (E, Bq * 200), "f16")
                    else:
                        vt = self._zero_planes(("vtwin", E, Bq), (E, Bq * 200))
                    ops.gemm(xn, wv, bias=bv, want_f32=False, transposed=True, ldc=Bq * 200, out_split=vt, t_row_group=Tq, t_row_pad=200 - Tq,
                             out_fp16=f16, prec=qprec)
                else:
                    _, vt, _ = ops.gemm(xn, wv, bias=bv, want_f32=False, want_split=True, transposed=True, out_fp16=f16, prec=qprec)  # (E, B*T)
                q, k = qk[:, 0:E], qk[:, E:]
                st = (Tq * 2 * E, 2 * E, hd)
            else:
                _, qkv, _ = ops.gemm(xn, wqkv, bias=bqkv, want_f32=False, want_split=True)
                q, k, vv = qkv[:, 0:E], qkv[:, E:2 * E], qkv[:, 2 * E:]
            if f16:
                Rh = W.cached(("relh16", blk, qh), lambda: ops.split_weight_f16(_get_rel_pos_table(qh, qh, W[blk + ".attn.rel_pos_h"])))
                Rw = W.cached(("relw16", blk, qw), lambda: ops.split_weight_f16(_get_rel_pos_table(qw, qw, W[blk + ".attn.rel_pos_w"])))
                rel_h = ops.relpos_bias_tc_f16(q.hi, st, Rh, 0, qh, qw, Bq, nh, hd)
                rel_w = ops.relpos_bias_tc_f16(q.hi, st, Rw, 1, qh, qw, Bq, nh, hd)
            else:
                Rh = W.cached(("relh", blk, qh), lambda: ops.split_weight(_get_rel_pos_table(qh, qh, W[blk + ".attn.rel_pos_h"])))
                Rw = W.cached(("relw", blk, qw), lambda: ops.split_weight(_get_rel_pos_table(qw, qw, W[blk + ".attn.rel_pos_w"])))
                rel_h = ops.relpos_bias_tc(q, st, Rh, 0, qh, qw, Bq, nh, hd)
                rel_w = ops.relpos_bias_tc(q, st, Rw, 1, qh, qw, Bq, nh, hd)
            proj6 = use_tc and f16 and self.mlp_f16e4m3      # attention output as fp16 + e4m3 planes, proj on gemm prec 6
            if use_tc:
                _, ao = ops.attention_tc(q, k, vt, Bq, nh, Tq, hd, st[0], st[1], st[0], st[1], hd ** -0.5, rel_h=rel_h, rel_w=rel_w,
                                         kh=qh, kw=qw, f16=f16, out_e4m3=proj6)
            else:
                _, ao = ops.attention(q, k, vv, Bq, nh, Tq, Tq, hd, st, st, st, hd ** -0.5, rel_h=rel_h, rel_w=rel_w, kh=qh, kw=qw)
            ao = ao.view(Bq * Tq, E)
            if proj6:
                wproj = W.cached(("proj68", blk), lambda: ops.split_f16_e4m3(W[blk + ".attn.proj.weight"], weight=True))
            pprec = 6 if proj6 else None
            if windowed:
                ops.gemm(ao, wproj, bias=bproj, residual=x, out_f32=x, row_map=win2tok, out_rows=B * T, prec=pprec)
            else:
                ops.gemm(ao, wproj, bias=bproj, residual=x, out_f32=x, prec=pprec)
            if self.mlp_f16e4m3 and ops.PREC == 3 and E % 32 == 0:
                # fc1 / fc2 in the fp16 + e4m3 split (gemm prec 6): the hi x hi product in ONE fp16 pass, both cross terms in ONE fp8
                # pass -- two pass-equivalents instead of three for the same ~2^-15.5 operand accuracy.  norm2 and the GELU epilogue
                # emit the planes directly (fp16 + e4m3 pair: the same 4 bytes per element as bf16 hi / lo)
                _, xn2, _ = ops.layernorm(x, W[blk + ".norm2.weight"], W[blk + ".norm2.bias"], 1e-6, out_e4m3=True)
                w1, b1, w2, b2 = W.cached(("mlp68", blk), lambda: (ops.split_f16_e4m3(W[f"{blk}.mlp.{fc1}.weight"], weight=True), W[f"{blk}.mlp.{fc1}.bias"],
                                                                    ops.split_f16_e4m3(W[f"{blk}.mlp.{fc2}.weight"], weight=True), W[f"{blk}.mlp.{fc2}.bias"]))
                _, hmid, _ = ops.gemm(xn2, w1, bias=b1, act=ops.ACT_GELU, want_f32=False, out_e4m3=True, prec=6)
                ops.gemm(hmid, w2, bias=b2, residual=x, out_f32=x, prec=6)
            else:
                _, xn2, _ = ops.layernorm(x, W[blk + ".norm2.weight"], W[blk + ".norm2.bias"], 1e-6)
                w1, b1 = W.lin(f"{blk}.mlp.{fc1}")
                w2, b2 = W.lin(f"{blk}.mlp.{fc2}")
                _, hmid, _ = ops.gemm(xn2, w1, bias=b1, act=ops.ACT_GELU, want_f32=False, want_split=True)
                ops.gemm(hmid, w2, bias=b2, residual=x, out_f32=x)
            if tap is not None and self.taps is not None and i in self.taps.get("blocks", ()):
                self.taps[f"{tap}.block{i}"] = x.view(B, gh, gw, E).clone()
        return x

    # ------------------------------------------------------------ ResNet-50 backbone (config #1; detectron2 resnet.py:105-205,329-366,614-694)
    def _conv_bn(self, prefix, ksz):
        """(BF2 weight (cout, ksz*ksz*cin) in (ky, kx, c) column order, bias) with FrozenBatchNorm2d folded in
        (batch_norm.py:13-118: y = x * (w * rsqrt(var + eps)) + (b - mean * w * rsqrt(var + eps)), eps 1e-5)."""
        W = self.W

        def mk():
            w = W[prefix + ".weight"]
            scale = W[prefix + ".norm.weight"] * (W[prefix + ".norm.running_var"] + 1e-5).rsqrt()
            bias = W[prefix + ".norm.bias"] - W[prefix + ".norm.running_mean"] * scale
            w = w * scale.view(-1, 1, 1, 1)
            if w.shape[1] % 8:                                   # stem: 3 input channels padded to 8 (GEMM rows need 16-byte strides)
                w = F.pad(w, (0, 0, 0, 0, 0, 8 - w.shape[1] % 8))
            return ops.split_weight(w.permute(0, 2, 3, 1).reshape(w.shape[0], -1)), bias.contiguous()
        return W.cached(("convbn", prefix, ksz), mk)

    def resnet50(self, img):
        """img: (B, 3, H, W) raw 0..255 fp32 -> {res3, res4, res5: (fp32 NHWC, BF2)}.  Every convolution is a GEMM over NHWC rows
        (1x1: plain / strided row subsampling through im2col with k = 1; 3x3 and the 7x7 stem: im2col) with the frozen BN folded into
        weights and bias, ReLU in the epilogue, and the bottleneck's relu(conv3 + shortcut) as residual + post-ReLU in the epilogue."""
        bb = "detr.detr.backbone.0.backbone"
        B, _, H, Wd = img.shape
        mean = self._dev_const([123.675, 116.280, 103.530], torch.float32).view(1, 3, 1, 1)
        std = self._dev_const([58.395, 57.120, 57.375], torch.float32).view(1, 3, 1, 1)
        x = ((img - mean) / std).permute(0, 2, 3, 1)
        x = F.pad(x, (0, 5)).contiguous()                        # NHWC, channels 3 -> 8 (zeros)
        cols, Ho, Wo = ops.im2col_nhwc(x, 7, 2, 3)
        w, b = self._conv_bn(bb + ".stem.conv1", 7)
        y, _, _ = ops.gemm(cols, w, bias=b, act=ops.ACT_RELU)
        x, x_s = ops.maxpool3x3s2_nhwc(y.view(B, Ho, Wo, 64), want_f32=True, want_split=True)
        outs = {}
        for name, n, first_stride in (("res2", 3, 1), ("res3", 4, 2), ("res4", 6, 2), ("res5", 3, 2)):
            for i in range(n):
                p_ = f"{bb}.{name}.{i}"
                stride = first_stride if i == 0 else 1
                Bc, Hc, Wc, Cin = x.shape
                w1, b1 = self._conv_bn(p_ + ".conv1", 1)
                y1, _, _ = ops.gemm(x_s.view(-1, Cin), w1, bias=b1, act=ops.ACT_RELU)                    # f32 for the 3x3 im2col
                bott = w1.hi.shape[0]
                cols, Ho, Wo = ops.im2col_nhwc(y1.view(Bc, Hc, Wc, bott), 3, stride, 1)
                w2, b2 = self._conv_bn(p_ + ".conv2", 3)
                _, y2, _ = ops.gemm(cols, w2, bias=b2, act=ops.ACT_RELU, want_f32=False, want_split=True)
                if (p_ + ".shortcut.weight") in self.W.f:
                    ws, bs = self._conv_bn(p_ + ".shortcut", 1)
                    if stride == 1:
                        sc, _, _ = ops.gemm(x_s.view(-1, Cin), ws, bias=bs)
                    else:
                        sub, _, _ = ops.im2col_nhwc(x, 1, stride, 0)                                     # strided 1x1 = row subsampling
                        sc, _, _ = ops.gemm(sub, ws, bias=bs)
                else:
                    sc = x.view(-1, Cin)
                w3, b3 = self._conv_bn(p_ + ".conv3", 1)
                y3, y3_s, _ = ops.gemm(y2, w3, bias=b3, residual=sc, relu_after_residual=True, want_split=True)
                x, x_s = y3.view(Bc, Ho, Wo, -1), y3_s.view(Bc, Ho, Wo, -1)
            if name != "res2":
                outs[name] = (x, x_s)
        return outs

    # ------------------------------------------------------------ generic pieces
    def conv1x1_gn(self, feat_s, prefix_conv, prefix_gn, out_view=None, y_bstride=None, relu=False, bias=True):
        """1x1 conv (GEMM over NHWC rows) + GroupNorm(32).  feat_s: BF2 (B, h, w, Cin)."""
        W = self.W
        B, h, w, Cin = feat_s.hi.shape
        wc, bc = W.lin(prefix_conv)
        y, _, _ = ops.gemm(feat_s.view(B * h * w, Cin), wc, bias=bc if bias else None)
        y = y.view(B, h * w, -1)
        return ops.groupnorm_nhwc(y, W[prefix_gn + ".weight"], W[prefix_gn + ".bias"], relu=relu, out_f32=out_view,
                                  y_bstride=y_bstride)[0]

    def conv_kxk(self, x_nhwc, prefix, ksz=3, stride=1, pad=1, act=ops.ACT_NONE, want_f32=True, want_split=False, bias=True):
        W = self.W
        B = x_nhwc.shape[0]
        cols, Ho, Wo = ops.im2col_nhwc(x_nhwc, ksz, stride, pad)
        wk, bk = W.conv_kxk(prefix)
        f, s, _ = ops.gemm(cols, wk, bias=bk if bias else None, act=act, want_f32=want_f32, want_split=want_split)
        C = wk.hi.shape[0]
        return (f.view(B, Ho, Wo, C) if f is not None else None), (s.view(B, Ho, Wo, C) if s is not None else None)

    def msda_layer(self, prefix, query_s, ref, value_src_s, value_mask, shapes_t, lsi_t, B, Lq, S, want_split=True, shapes_host=None):
        """MSDeformAttn.forward (H/models/deformable_detr/ops/modules/ms_deform_attn.py:79-116) minus output_proj.
        query_s: BF2 (B*Lq, 256); value_src_s: BF2 (B*S, 256); ref (B, Lq, 4, 2|4) fp32."""
        W = self.W
        wv, bv = W.lin(prefix + ".value_proj")
        if self.fp16_value_map and Lq == S and ops.PREC == 3:
            # encoder self-attention: the value map as ONE fp16 plane -- every output is a convex combination of 64 taps, so the 2^-12
            # rounding averages down (tools/prec_map_emulate.py enc_value_out16: +1.4e-4 on the mask logits), and the gather kernel, bound
            # by its L2 -> L1 fill traffic, moves half the bytes
            _, vs, _ = ops.gemm(value_src_s, wv, bias=bv, want_f32=False, want_split=True, out_fp16=True)
            value = vs.hi.view(B, S, 256)
            if value_mask is not None:
                value = value.masked_fill(value_mask[..., None], 0.0)
        elif self.bf16_value_map and value_mask is None:
            _, vs, _ = ops.gemm(value_src_s, wv, bias=bv, want_f32=False, want_split=True)
            value = vs.hi.view(B, S, 256)
        else:
            value, _, _ = ops.gemm(value_src_s, wv, bias=bv)
            value = value.view(B, S, 256)
            if value_mask is not None:
                value = value.masked_fill(value_mask[..., None], 0.0)
                if self.bf16_value_map:
                    value = value.bfloat16()
        wol, bol = W.lin_cat(prefix + ".offs_logits", [prefix + ".sampling_offsets", prefix + ".attention_weights"])
        ol, _, _ = ops.gemm(query_s, wol, bias=bol)
        return ops.msda_fused(value, shapes_t, lsi_t, ol.view(B, Lq, 384), ref, want_split=want_split, shapes_host=shapes_host)

    def mlp(self, x_s, prefix, n, last_f32=True):
        """MLP with ReLU between layers (deformable_transformer_dino.py:599-633).  x_s BF2 (rows, in)."""
        W = self.W
        cur = x_s
        for i in range(n):
            w, b = W.lin(f"{prefix}.layers.{i}")
            last = i == n - 1
            f, s, _ = ops.gemm(cur, w, bias=b, act=ops.ACT_NONE if last else ops.ACT_RELU, want_f32=last and last_f32,
                               want_split=not (last and last_f32))
            cur = s
        return f if last_f32 else cur

    def ffn_postnorm(self, x, x_s, prefix, n1, n2, l1="linear1", l2="linear2"):
        """x = LN(x + linear2(relu(linear1(x))))"""
        W = self.W
        if x_s.fmt == "f16+e4m3":      # fp16 + e4m3 planes (encoder layers): both linears on gemm prec 6
            w1, b1, w2, b2 = W.cached(("ffn68", prefix), lambda: (ops.split_f16_e4m3(W[f"{prefix}.{l1}.weight"], weight=True), W[f"{prefix}.{l1}.bias"],
                                                                   ops.split_f16_e4m3(W[f"{prefix}.{l2}.weight"], weight=True), W[f"{prefix}.{l2}.bias"]))
            prec, hidden = 6, dict(out_e4m3=True)
        else:
            (w1, b1), (w2, b2) = W.lin(f"{prefix}.{l1}"), W.lin(f"{prefix}.{l2}")
            prec, hidden = None, dict(want_split=True)
        _, h, _ = ops.gemm(x_s, w1, bias=b1, act=ops.ACT_RELU, want_f32=False, prec=prec, **hidden)
        y, _, _ = ops.gemm(h, w2, bias=b2, residual=x, prec=prec)
        return ops.layernorm(y, W[f"{prefix}.{n2}.weight"], W[f"{prefix}.{n2}.bias"], 1e-5, want_f32=True, want_split=True)[:2]

    def encoder_layer(self, prefix, src, src_s, pos, ref, mask_flat, shapes_t, lsi_t, B, S, shapes_host=None):
        """DeformableTransformerEncoderLayer (deformable_transformer_dino.py:354-394) == MaskDINO's (:117-157)."""
        W = self.W
        _, q_s = ops.add_split(src, pos)
        a_s = self.msda_layer(prefix + ".self_attn", q_s.view(B * S, 256), ref, src_s.view(B * S, 256), mask_flat, shapes_t, lsi_t, B, S, S,
                              shapes_host=shapes_host)
        wo, bo = W.lin(prefix + ".self_attn.output_proj")
        y, _, _ = ops.gemm(a_s.view(B * S, 256), wo, bias=bo, residual=src.view(B * S, 256))
        x, x_s, _ = ops.layernorm(y, W[prefix + ".norm1.weight"], W[prefix + ".norm1.bias"], 1e-5, want_f32=True, want_split=True,
                                  out_e4m3=self.mlp_f16e4m3 and ops.PREC == 3)       # norm1 feeds linear1 only
        x, x_s = self.ffn_postnorm(x, x_s, prefix, "norm1", "norm2")
        return x.view(B, S, 256), x_s.view(B, S, 256)

    def decoder_layer(self, prefix, tgt, tgt_s, query_pos, ref_in, memory_s, mask_flat, shapes_t, lsi_t, B, Q, S):
        """DeformableTransformerDecoderLayer (deformable_transformer_dino.py:397-450; maskdino dino_decoder.py:171-270):
        MHA self-attn -> norm2 -> MSDeformAttn cross -> norm1 -> FFN -> norm3."""
        W = self.W
        d = 256
        _, qk_s = ops.add_split(tgt, query_pos)
        win = W.cached(("mha_in", prefix), lambda: (ops.split_weight(W[prefix + ".self_attn.in_proj_weight"][:2 * d]),
                                                     W[prefix + ".self_attn.in_proj_bias"][:2 * d].contiguous(),
                                                     ops.split_weight(W[prefix + ".self_attn.in_proj_weight"][2 * d:]),
                                                     W[prefix + ".self_attn.in_proj_bias"][2 * d:].contiguous()))
        _, qk, _ = ops.gemm(qk_s.view(B * Q, d), win[0], bias=win[1], want_f32=False, want_split=True)     # (B*Q, 512)
        _, v, _ = ops.gemm(tgt_s.view(B * Q, d), win[2], bias=win[3], want_f32=False, want_split=True)
        _, ao = ops.attention(qk[:, :d], qk[:, d:], v, B, 8, Q, Q, 32, (Q * 2 * d, 2 * d, 32), (Q * 2 * d, 2 * d, 32), (Q * d, d, 32), 32 ** -0.5)
        wo, bo = W.lin(prefix + ".self_attn.out_proj")
        y, _, _ = ops.gemm(ao.view(B * Q, d), wo, bias=bo, residual=tgt.view(B * Q, d))
        t, t_s, _ = ops.layernorm(y, W[prefix + ".norm2.weight"], W[prefix + ".norm2.bias"], 1e-5, want_f32=True, want_split=False)
        _, q_s = ops.add_split(t, query_pos.view(B * Q, d))
        a_s = self.msda_layer(prefix + ".cross_attn", q_s, ref_in, memory_s.view(B * S, d), mask_flat, shapes_t, lsi_t, B, Q, S)
        wo2, bo2 = W.lin(prefix + ".cross_attn.output_proj")
        y, _, _ = ops.gemm(a_s.view(B * Q, d), wo2, bias=bo2, residual=t)
        t, t_s, _ = ops.layernorm(y, W[prefix + ".norm1.weight"], W[prefix + ".norm1.bias"], 1e-5, want_f32=True, want_split=True)
        t, t_s = self.ffn_postnorm(t, t_s, prefix, "norm1", "norm3")
        return t.view(B, Q, d), t_s.view(B, Q, d)

    @staticmethod
    def encoder_reference_points(shapes, valid_ratios, device):
        """get_reference_points (deformable_transformer_dino.py:313-325) -> (B, S, L, 2)"""
        refs = []
        for lvl, (H_, W_) in enumerate(shapes):
            ry, rx = torch.meshgrid(torch.linspace(0.5, H_ - 0.5, H_, dtype=torch.float32, device=device),
                                    torch.linspace(0.5, W_ - 0.5, W_, dtype=torch.float32, device=device), indexing="ij")
            ry = ry.reshape(-1)[None] / (valid_ratios[:, None, lvl, 1] * H_)
            rx = rx.reshape(-1)[None] / (valid_ratios[:, None, lvl, 0] * W_)
            refs.append(torch.stack((rx, ry), -1))
        ref = torch.cat(refs, 1)
        return (ref[:, :, None] * valid_ratios[:, None]).contiguous()

    @staticmethod
    def proposals(shapes, mask_flat, B, device):
        """gen_encoder_output_proposals geometry (deformable_transformer_dino.py:138-162; maskdino/utils/utils.py:33-66)
        -> (unsigmoided proposals (B,S,4) with +inf on invalid, valid (B,S,1) bool)"""
        props, cur = [], 0
        for lvl, (H_, W_) in enumerate(shapes):
            m = mask_flat[:, cur:cur + H_ * W_].view(B, H_, W_, 1)
            valid_H = torch.sum(~m[:, :, 0, 0], 1)
            valid_W = torch.sum(~m[:, 0, :, 0], 1)
            gy, gx = torch.meshgrid(torch.linspace(0, H_ - 1, H_, dtype=torch.float32, device=device),
                                    torch.linspace(0, W_ - 1, W_, dtype=torch.float32, device=device), indexing="ij")
            grid = torch.cat([gx.unsqueeze(-1), gy.unsqueeze(-1)], -1)
            scale = torch.cat([valid_W.unsqueeze(-1), valid_H.unsqueeze(-1)], 1).view(B, 1, 1, 2)
            grid = (grid.unsqueeze(0).expand(B, -1, -1, -1) + 0.5) / scale
            wh = torch.ones_like(grid) * 0.05 * (2.0 ** lvl)
            props.append(torch.cat((grid, wh), -1).view(B, -1, 4))
            cur += H_ * W_
        op = torch.cat(props, 1)
        valid = ((op > 0.01) & (op < 0.99)).all(-1, keepdim=True)
        op = torch.log(op / (1 - op))
        op = op.masked_fill(mask_flat.unsqueeze(-1), float("inf")).masked_fill(~valid, float("inf"))
        return op, valid

    # ------------------------------------------------------------ BERT (HF BertModel; H/models/deformable_detr/bert_model.py)
    def bert(self, input_ids, attention_mask):
        """-> last hidden state (R, L, 768) fp32 for R rows of <= 512 tokens."""
        W, b = self.W, self.hp["bert"]
        te = "text_encoder.body.model"
        R, L = input_ids.shape
        Hd, nh = b["hidden"], b["heads"]
        hd = Hd // nh
        emb = (W[te + ".embeddings.word_embeddings.weight"][input_ids]
               + W[te + ".embeddings.position_embeddings.weight"][:L][None]
               + W[te + ".embeddings.token_type_embeddings.weight"][0][None, None])
        x, x_s, _ = ops.layernorm(emb.view(R * L, Hd), W[te + ".embeddings.LayerNorm.weight"], W[te + ".embeddings.LayerNorm.bias"],
                                  1e-12, want_f32=True, want_split=True)
        key_bias = ((1.0 - attention_mask.float()) * torch.finfo(torch.float32).min).contiguous()
        for i in range(b["layers"]):
            p = f"{te}.encoder.layer.{i}"
            wqkv, bqkv = W.lin_cat(p + ".qkv", [p + ".attention.self.query", p + ".attention.self.key", p + ".attention.self.value"])
            _, qkv, _ = ops.gemm(x_s, wqkv, bias=bqkv, want_f32=False, want_split=True)
            st = (L * 3 * Hd, 3 * Hd, hd)
            _, ao = ops.attention(qkv[:, :Hd], qkv[:, Hd:2 * Hd], qkv[:, 2 * Hd:], R, nh, L, L, hd, st, st, st, hd ** -0.5, key_bias=key_bias)
            wo, bo = W.lin(p + ".attention.output.dense")
            y, _, _ = ops.gemm(ao.view(R * L, Hd), wo, bias=bo, residual=x)
            x, x_s, _ = ops.layernorm(y, W[p + ".attention.output.LayerNorm.weight"], W[p + ".attention.output.LayerNorm.bias"], 1e-12,
                                      want_f32=True, want_split=True)
            wi, bi = W.lin(p + ".intermediate.dense")
            w2, b2 = W.lin(p + ".output.dense")
            _, hmid, _ = ops.gemm(x_s, wi, bias=bi, act=ops.ACT_GELU, want_f32=False, want_split=True)
            y, _, _ = ops.gemm(hmid, w2, bias=b2, residual=x)
            x, x_s, _ = ops.layernorm(y, W[p + ".output.LayerNorm.weight"], W[p + ".output.LayerNorm.bias"], 1e-12, want_f32=True, want_split=True)
        return x.view(R, L, Hd)

    def forward_text(self, input_ids, attention_mask, same_rows=None, chunk_plan=None):
        """BertEncoder.forward (bert_model.py:32-154): rows > 512 tokens are chunked at '.'/EOS boundaries.
        `same_rows` says whether every row of the batch holds the same prompt (the detection case, hipie_img.py:330-332):
        then row 0 is encoded once and broadcast.  The caller decides it from the host-side token ids (no device sync, safe
        inside a CUDA-graph capture); None = decide here from the tensors, which reads one flag back from the device.
        `chunk_plan` (rows > 512 tokens): the host-side cut plan from `text_chunk_plan`; None = computed here (device -> host copy)."""
        L = input_ids.shape[1]
        if same_rows is None:
            same_rows = self.rows_equal(input_ids, attention_mask)
        same = bool(same_rows) and input_ids.shape[0] > 1
        if same:
            ids_u, am_u = input_ids[:1].contiguous(), attention_mask[:1].contiguous()
        else:
            ids_u, am_u = input_ids, attention_mask
        hid = self.bert(ids_u, am_u) if L <= 512 else self._bert_chunked(ids_u, am_u, chunk_plan)
        if same:
            hid = hid.expand(input_ids.shape[0], -1, -1).contiguous()
        return {"hidden": hid, "masks": attention_mask}

    def text_chunk_plan(self, input_ids, attention_mask, same_rows):
        """The chunk plan forward_text will need for these (host or device) ids, or None for rows of <= 512 tokens."""
        if input_ids.shape[1] <= 512:
            return None
        if bool(same_rows) and input_ids.shape[0] > 1:
            input_ids, attention_mask = input_ids[:1], attention_mask[:1]
        return self.plan_text_chunks(input_ids, attention_mask)

    @staticmethod
    def rows_equal(input_ids, attention_mask):
        """True when every row equals row 0 (value comparison every call: no pointer-keyed cache, the caching allocator
        reuses addresses).  Host tensors are compared on the host; device tensors cost one sync and are refused while a
        CUDA graph is being captured."""
        if input_ids.shape[0] <= 1:
            return True
        if input_ids.is_cuda and torch.cuda.is_current_stream_capturing():
            raise RuntimeError("forward_text: pass same_rows explicitly inside a CUDA-graph capture")
        return bool(((input_ids == input_ids[:1]).all() & (attention_mask == attention_mask[:1]).all()).item())

    def plan_text_chunks(self, input_ids, mask, sep=1012):
        """Host half of the > 512-token path (bert_model.py:48-120): cut every row at its last '.' / EOS before position 510, re-wrap
        each piece as a 512-token BERT input ([CLS] + piece for all but the first) and remember where its hidden states go.
        Pure host work on the token ids -- done BEFORE a CUDA-graph capture; the plan's `signature` (the cut positions) is part
        of the captured launch sequence, its `rows` / `masks` are refilled in place between replays."""
        CLS, EOS = 101, 102
        ids_c, mask_c = input_ids.cpu(), mask.cpu()
        bs = mask_c.shape[0]
        chunks = []
        for bi in range(bs):
            inp, begin, start_src = ids_c[bi].clone(), 0, 0
            while True:
                seps = torch.where((inp == sep) | (inp == EOS))[0]
                seps = seps[seps < 510]
                if len(seps) == 0:
                    break
                last = int(seps[-1])
                first_input = inp[:last + 1].clone()
                first_input[-1] = EOS
                first_mask_on = torch.where(mask_c[bi][:last + 1] == 1)[0]
                l_valid = len(first_input)
                m = torch.zeros(512, dtype=torch.long)
                if start_src == 0:
                    row = torch.cat([first_input, torch.zeros(512 - l_valid, dtype=torch.long)])
                    m[first_mask_on] = 1
                else:
                    pad = torch.zeros(512 - l_valid - 1, dtype=torch.long)
                    pad[0] = sep
                    row = torch.cat([torch.tensor([CLS]), first_input, pad])
                    m[first_mask_on + 1] = 1
                    m[0] = 1
                chunks.append((bi, row, m, (start_src, start_src + l_valid, begin, begin + l_valid)))
                start_src = 1
                inp = inp[l_valid:]
                begin += l_valid
        plan = types.SimpleNamespace()
        plan.spans = [(c[0],) + c[3] for c in chunks]
        plan.signature = (bs, int(mask_c.shape[1])) + tuple(plan.spans)
        plan.rows = torch.stack([c[1] for c in chunks]) if chunks else torch.zeros(0, 512, dtype=torch.long)
        plan.masks = torch.stack([c[2] for c in chunks]) if chunks else torch.zeros(0, 512, dtype=torch.long)
        plan.rows_d, plan.masks_d = plan.rows.to(self.device), plan.masks.to(self.device)
        return plan

    def _bert_chunked(self, input_ids, mask, plan=None):
        bs, seq_len = mask.shape
        if plan is None:
            if input_ids.is_cuda and torch.cuda.is_current_stream_capturing():
                raise RuntimeError("forward_text: > 512 tokens inside a CUDA-graph capture needs chunk_plan= (plan_text_chunks on the host ids)")
            plan = self.plan_text_chunks(input_ids, mask)
        out = torch.zeros(bs, seq_len, self.hp.get("lang_dim", 768), device=self.device)
        if len(plan.spans) == 0:
            return out
        last_hidden = self.bert(plan.rows_d, plan.masks_d)
        for idx, (bi, s0, s1, t0, t1) in enumerate(plan.spans):
            out[bi, t0:t1] = last_hidden[idx, s0:s1]
        return out

    # ------------------------------------------------------------ VL early fusion (fuse_helper.py:54-179)
    def vl_fuse(self, src, lang_hidden, lang_mask, B, S):
        W = self.W
        p = "detr.detr.transformer.encoder.vl_layers.0.b_attn"
        Lt, Ld = lang_hidden.shape[1], lang_hidden.shape[2]
        E = W[p + ".attn.v_proj.weight"].shape[0]
        nh = 8
        hd = E // nh
        v, v_s, _ = ops.layernorm(src.view(B * S, 256), W[p + ".layer_norm_v.weight"], W[p + ".layer_norm_v.bias"], 1e-5, want_f32=True, want_split=True)
        l, l_s, _ = ops.layernorm(lang_hidden.reshape(B * Lt, Ld), W[p + ".layer_norm_l.weight"], W[p + ".layer_norm_l.bias"], 1e-5, want_f32=True, want_split=True)
        scale = hd ** -0.5
        # Precision map (DESIGN.md 3): the S x Lt score and P.V contractions of the bi-attention run as ONE fp16 MMA pass (operands
        # rounded at 2^-12: measured 2e-5 on the encoder memory, 7e-6 on the class logits, tools/prec_emulate.py); the six projections
        # around them stay 3-pass.  q / k / value maps leave their projection GEMMs as single fp16 planes, the softmaxes write fp16.
        f16 = self.attn_fp16 and ops.PREC == 3
        aprec = 2 if f16 else ops.PREC
        # (v_proj(v) * scale): scale = 256^-0.5 = 2^-4 for the shipped embed 2048 / 8 heads -> exact to fold into W and b
        wq, bq = W.cached(("vlq", p), lambda: (ops.split_weight(W[p + ".attn.v_proj.weight"] * scale),
                                               (W[p + ".attn.v_proj.bias"] * scale).contiguous()))
        _, q_s, _ = ops.gemm(v_s, wq, bias=bq, want_f32=False, want_split=True, out_fp16=f16)                      # (B*S, E)
        wk, bk = W.lin(p + ".attn.l_proj")
        _, k_s, _ = ops.gemm(l_s, wk, bias=bk, want_f32=False, want_split=True, out_fp16=f16)                      # (B*Lt, E)
        wvv, bvv = W.lin(p + ".attn.values_v_proj")
        wvl, bvl = W.lin(p + ".attn.values_l_proj")
        # value maps are needed K-major for the P.V GEMMs -> emit them transposed: (E, B*S) and (E, B*Lt)
        _, vvT, _ = ops.gemm(v_s, wvv, bias=bvv, want_f32=False, want_split=True, transposed=True, out_fp16=f16)   # (E, B*S)
        _, vlT, _ = ops.gemm(l_s, wvl, bias=bvl, want_f32=False, want_split=True, transposed=True, out_fp16=f16)   # (E, B*Lt)
        # additive text mask: valid tokens +1, invalid -9e15 (fuse_helper.py:96-107)
        am = lang_mask.float()
        colbias = torch.where(am == 0, torch.full_like(am, -9e15), am).contiguous()
        out_v, out_l = BF2.empty((B * S, E), self.device), BF2.empty((B * Lt, E), self.device)
        # the text->image P.V contraction runs over K = S pixels; TMA rows need 16-byte strides, i.e. a pixel count that is a multiple
        # of 8.  Image sizes whose level sum is not (e.g. 192 x 256 -> S = 1020) get zero-padded operand pitches (zeros add nothing).
        Sp = (S + 7) // 8 * 8
        padS = lambda a, rows: a.map(lambda t: F.pad(t.reshape(rows, -1, S), (0, Sp - S)).reshape(rows, -1))
        if Sp != S:
            vvT = padS(vvT, E)                                   # (E, B*Sp): every image at an Sp pitch
        for h in range(nh):
            c0, c1 = h * hd, (h + 1) * hd
            qh, kh = q_s[:, c0:c1], k_s[:, c0:c1]
            # scores (B, S, Lt) and its transpose (B, Lt, S): two GEMMs instead of a transpose pass
            sc, _, _ = ops.gemm(qh, kh, M=S, N=Lt, K=hd, batch=B, lda=E, ldw=E, a_bstride=S * E, w_bstride=Lt * E, prec=aprec)
            scT, _, _ = ops.gemm(kh, qh, M=Lt, N=S, K=hd, batch=B, lda=E, ldw=E, a_bstride=Lt * E, w_bstride=S * E, prec=aprec)
            _, pv = ops.row_softmax(sc.view(B * S, Lt), colbias=colbias, rows_per_batch=S, out_fp16=f16)          # softmax over text
            _, pl = ops.row_softmax(scT.view(B * Lt, S), sub_rowmax=True, out_fp16=f16)                            # softmax over pixels
            if Sp != S:
                pl = padS(pl, B * Lt)                            # (B*Lt, Sp)
            # out_v[b, s, c0:c1] = P_v[b] (S x Lt) . value_l[b]^T ; value_l^T rows c0:c1 of vlT, cols b*Lt..
            ops.gemm(pv, vlT[c0:c1], want_f32=False, out_split=out_v[:, c0:c1], M=S, N=hd, K=Lt, batch=B, lda=Lt, ldw=B * Lt,
                     a_bstride=S * Lt, w_bstride=Lt, ldc=E, c_bstride=S * E, prec=aprec)
            ops.gemm(pl, vvT[c0:c1], want_f32=False, out_split=out_l[:, c0:c1], M=Lt, N=hd, K=Sp, batch=B, lda=Sp, ldw=B * Sp,
                     a_bstride=Lt * Sp, w_bstride=Sp, ldc=E, c_bstride=Lt * E, prec=aprec)
        wov, bov = W.lin(p + ".attn.out_v_proj")
        wol, bol = W.lin(p + ".attn.out_l_proj")
        new_v, new_v_s, _ = ops.gemm(out_v, wov, bias=bov, colscale=W[p + ".gamma_v"], residual=v, want_split=True)
        new_l, _, _ = ops.gemm(out_l, wol, bias=bol, colscale=W[p + ".gamma_l"], residual=l)
        return new_v.view(B, S, 256), new_v_s.view(B, S, 256), new_l.view(B, Lt, Ld)

    # ------------------------------------------------------------ deformable-DINO stages of the DETR and MaskDINO branches
    def _levels(self, feats):
        """The four encoder levels (res3..res5 and the 3x3 stride-2 level on res5) -> (lv, shapes, starts, S, shapes_t, lsi_t)"""
        lv = [feats["res3"], feats["res4"], feats["res5"]]
        shapes = [tuple(f[0].shape[1:3]) for f in lv]
        h5, w5 = shapes[2]
        shapes.append(((h5 + 2 - 3) // 2 + 1, (w5 + 2 - 3) // 2 + 1))
        return (lv, shapes) + self._level_index(shapes)

    def _level_index(self, shapes):
        """Levels flattened in the order of `shapes` -> (starts, S, shapes_t, lsi_t), the last two as device constants."""
        starts = [0]
        for h, w in shapes[:-1]:
            starts.append(starts[-1] + h * w)
        S = starts[-1] + shapes[-1][0] * shapes[-1][1]
        return starts, S, self._dev_const([list(x) for x in shapes], torch.long), self._dev_const(list(starts), torch.long)

    def _input_proj(self, prefix, lv, starts, S, B):
        """input_proj.{0,1,2} (1x1 conv + GN on res3..res5) and input_proj.3 (3x3/2 conv + GN on res5), written level-flattened into
        one (B, S, 256) buffer (H/models/ddetrs_dn.py:821-847; maskdino_encoder.py:380-396)."""
        W = self.W
        src = torch.empty(B, S, 256, device=self.device)
        for l in range(3):
            self.conv1x1_gn(lv[l][1], f"{prefix}.input_proj.{l}.0", f"{prefix}.input_proj.{l}.1", out_view=src[:, starts[l]:], y_bstride=S * 256)
        cols, Ho, Wo = ops.im2col_nhwc(lv[2][0], 3, 2, 1)
        wk, bk = W.conv_kxk(f"{prefix}.input_proj.3.0")
        y, _, _ = ops.gemm(cols, wk, bias=bk)
        ops.groupnorm_nhwc(y.view(B, Ho * Wo, 256), W[f"{prefix}.input_proj.3.1.weight"], W[f"{prefix}.input_proj.3.1.bias"],
                           out_f32=src[:, starts[3]:], y_bstride=S * 256)
        return src

    @staticmethod
    def _level_pos(masks, offset, level_embed):
        """Per-level sine position + level_embed, level-flattened -> (B, S, 256) (deformable_transformer_dino.py:187-207;
        maskdino_encoder.py:94-101)."""
        return torch.cat([_sine_pos(m, 128, offset) + level_embed[l].view(1, 1, -1) for l, m in enumerate(masks)], 1).contiguous()

    def _enc_proposals(self, prefix, memory, shapes, mask_flat, B, S, pad_fill):
        """Two-stage encoder output (deformable_transformer_dino.py:222-224; maskdino_decoder.py:413-415): enc_output + LN on the memory,
        invalid proposals (and with `pad_fill` padded pixels) zeroed -> (unsigmoided proposals (B, S, 4), om_n (B*S, 256), om_ns)"""
        W = self.W
        props, valid = self.proposals(shapes, mask_flat, B, self.device)
        om = memory.masked_fill(mask_flat.unsqueeze(-1), 0.0) if pad_fill else memory
        om = om.masked_fill(~valid, 0.0)
        _, om_s = ops.add_split(om.view(B * S, 256))
        we, be = W.lin(prefix + ".enc_output")
        y, _, _ = ops.gemm(om_s, we, bias=be)
        om_n, om_ns, _ = ops.layernorm(y, W[prefix + ".enc_output_norm.weight"], W[prefix + ".enc_output_norm.bias"], 1e-5,
                                       want_f32=True, want_split=True)
        return props, om_n, om_ns

    def _select_queries(self, om_n, props, scores, nq, bbox_prefix, B, forced_topk):
        """Two-stage selection (deformable_transformer_dino.py:225-230; maskdino_decoder.py:416-426): top-k of `scores` (B, S), the
        selected encoder outputs and their boxes sigmoid(bbox MLP + proposal).  -> (topk, sel (B, nq, 256), sel_s, ref (B, nq, 4))"""
        # on the device (ops.topk: values descending, lowest index first among exact ties -> deterministic)
        topk = ops.topk(scores.contiguous(), nq)[1].long() if forced_topk is None else forced_topk
        # the bbox MLP only on the selected rows (same values as computing all and gathering)
        sel = torch.gather(om_n.view(B, -1, 256), 1, topk.unsqueeze(-1).expand(-1, -1, 256)).contiguous()
        _, sel_s = ops.add_split(sel)
        delta = self.mlp(sel_s.view(B * nq, 256), bbox_prefix, 3).view(B, nq, 4)
        ref = (delta + torch.gather(props, 1, topk.unsqueeze(-1).expand(-1, -1, 4))).sigmoid()
        return topk, sel, sel_s, ref

    def _dino_decoder(self, prefix, bbox_prefixes, tgt, tgt_s, ref, vr2, memory_s, mask_flat, shapes_t, lsi_t, B, Q, S):
        """Decoder loop (deformable_transformer_dino.py:467-525; dino_decoder.py:94-168), one layer per box MLP in `bbox_prefixes`;
        vr2 (B, L, 4) valid ratios.  -> (hs: [(tgt, tgt_s)] per layer, refs: the box refined by each layer)"""
        hs, refs = [], []
        for lid, bbox_prefix in enumerate(bbox_prefixes):
            ref_in = (ref[:, :, None] * vr2[:, None]).contiguous()              # (B, Q, L, 4)
            _, sine_s = ops.sine_embed(ref_in[:, :, 0, :])                      # (B*Q, 512) planes, one kernel
            qpos = self.mlp(sine_s, prefix + ".ref_point_head", 2).view(B, Q, 256)
            tgt, tgt_s = self.decoder_layer(f"{prefix}.layers.{lid}", tgt, tgt_s, qpos, ref_in, memory_s, mask_flat, shapes_t, lsi_t, B, Q, S)
            tmp = self.mlp(tgt_s.view(B * Q, 256), bbox_prefix, 3).view(B, Q, 4)
            ref = (tmp + inverse_sigmoid(ref)).sigmoid()
            hs.append((tgt, tgt_s))
            refs.append(ref)
        return hs, refs

    # ------------------------------------------------------------ DETR: input projections + transformer + heads
    def detr_inputs(self, feats, pad_mask, B, any_pad=True):
        """input_proj + sine positions + flatten (H/models/ddetrs_dn.py:821-847, deformable_transformer_dino.py:187-207).
        feats: {res3,res4,res5: (fp32 NHWC, BF2)}; pad_mask (B, H, W) bool.  -> dict"""
        dd = "detr.detr"
        lv, shapes, starts, S, shapes_t, lsi_t = self._levels(feats)
        src = self._input_proj(dd, lv, starts, S, B)
        masks = [F.interpolate(pad_mask[None].float(), size=shapes[l]).to(torch.bool)[0] for l in range(3)]
        masks.append(F.interpolate(masks[0][None].float(), size=shapes[3]).to(torch.bool)[0])
        make_pos = lambda: self._level_pos(masks, -0.5, self.W[f"{dd}.transformer.level_embed"])
        # without padding the masks are all-False and the encoding depends on the shapes only: computed once per resolution
        pos = make_pos() if any_pad else self.W.cached(("sine_pos_detr", B, tuple(shapes)), make_pos)
        mask_flat = torch.cat([m.flatten(1) for m in masks], 1)
        vr = []
        for m in masks:
            _, Hh, Ww = m.shape
            vr.append(torch.stack([torch.sum(~m[:, 0, :], 1).float() / Ww, torch.sum(~m[:, :, 0], 1).float() / Hh], -1))
        valid_ratios = torch.stack(vr, 1)
        return dict(src=src, pos=pos, mask_flat=mask_flat, any_pad=any_pad, valid_ratios=valid_ratios,
                    shapes=shapes, shapes_t=shapes_t, lsi_t=lsi_t, S=S, starts=starts)

    def detr_transformer(self, di, lang, B, forced_topk=None):
        """DeformableTransformerVLDINO.forward (deformable_transformer_dino.py:180-299), eval flags of every shipped yaml."""
        W, hp = self.W, self.hp
        t = "detr.detr.transformer"
        S, shapes, shapes_t, lsi_t = di["S"], di["shapes"], di["shapes_t"], di["lsi_t"]
        mask_flat = di["mask_flat"] if di["any_pad"] else None
        src, pos = di["src"], di["pos"]
        ref_enc = self.encoder_reference_points(shapes, di["valid_ratios"], self.device)
        # layer 0: VL fusion, then the deformable encoder layers
        src, src_s, lang_hidden = self.vl_fuse(src, lang["hidden"], lang["masks"], B, S)
        for i in range(hp.get("enc_layers", 6)):
            src, src_s = self.encoder_layer(f"{t}.encoder.layers.{i}", src, src_s, pos, ref_enc, mask_flat, shapes_t, lsi_t, B, S, shapes_host=shapes)
        memory, memory_s = src, src_s
        # two-stage proposals: enc_output + LN on the masked memory, Still_Classifier score, top-k, bbox_embed[nd]
        props, om_n, om_ns = self._enc_proposals(t, memory, shapes, di["mask_flat"], B, S, pad_fill=True)
        nd = hp.get("dec_layers", 6)
        wc, bc = W.lin(f"detr.detr.class_embed.{nd}.body")
        scores, _, _ = ops.gemm(om_ns, wc, bias=bc)
        scores = scores.view(B, S)
        nq = hp.get("num_queries", 900)
        topk, _, _, ref = self._select_queries(om_n, props, scores, nq, f"detr.detr.bbox_embed.{nd}", B, forced_topk)
        nbg = hp.get("num_bg", 10)
        tgt = torch.cat([W[t + ".tgt_embed_bg.weight"], W[t + ".tgt_embed.weight"]], 0)[None].repeat(B, 1, 1).contiguous()
        ref = torch.cat([W[t + ".bg_query_refs.weight"][None].repeat(B, 1, 1), ref], 1).contiguous()
        _, tgt_s = ops.add_split(tgt)
        vr2 = torch.cat([di["valid_ratios"], di["valid_ratios"]], -1)           # (B, L, 4)
        hs, refs = self._dino_decoder(t + ".decoder", [f"detr.detr.bbox_embed.{lid}" for lid in range(nd)], tgt, tgt_s, ref, vr2,
                                      memory_s, mask_flat, shapes_t, lsi_t, B, nbg + nq, S)
        return dict(hs=hs, refs=refs, memory=memory, memory_s=memory_s, lang_hidden=lang_hidden, enc_scores=scores, topk=topk)

    def vl_align(self, prefix, q_s, lang_hidden, B, Q):
        """VL_Align.forward (H/models/deformable_detr/deformable_detr.py:55-73). q_s: BF2 (B*Q, 256); lang (B, Lt, 768) -> (B, Q, Lt)"""
        W = self.W
        Lt = lang_hidden.shape[1]
        e = F.normalize(lang_hidden, p=2, dim=-1)
        _, e_s = ops.add_split((e / 2.0).reshape(B * Lt, -1).contiguous())
        wt, bt = W.lin(prefix + ".dot_product_projection_text")
        _, tok_s, _ = ops.gemm(e_s, wt, bias=bt, want_f32=False, want_split=True)                    # (B*Lt, 256)
        bias = (torch.matmul(e, W[prefix + ".bias_lang"]) + W[prefix + ".bias0"]).contiguous()        # (B, Lt)
        alpha = W.cached(("vl_alpha", prefix), lambda: float(1.0 / W[prefix + ".log_scale"].exp()))
        outs = []
        for b in range(B):       # per-image column bias; B tiny GEMMs (Q x Lt x 256)
            lg, _, _ = ops.gemm(q_s[b * Q:(b + 1) * Q], tok_s[b * Lt:(b + 1) * Lt], bias=bias[b].contiguous(), alpha=alpha)
            outs.append(lg)
        return torch.stack(outs, 0).clamp(min=-50000, max=50000)

    def condinst(self, memory, tr, di, image_sizes, B):
        """controller + MaskHeadSmallConv + fused dynamic mask head (ddetrs_dn.py:952-973,1006-1069,1411-1502,1581-1689)."""
        W, hp = self.W, self.hp
        shapes, starts = di["shapes"], di["starts"]
        lvl = len(tr["hs"]) - 1
        hs_s = tr["hs"][lvl][1]
        Q = hs_s.hi.shape[1]
        params = self.mlp(hs_s.view(B * Q, 256), "detr.controller", 3).view(B, Q, 169)
        ref_points = tr["refs"][-2][:, :, :2]
        scale = self._dev_const([[float(s[1]), float(s[0])] for s in image_sizes], torch.float32).view(B, 1, 2)
        ref_px = (ref_points * scale).contiguous()
        lv = [memory[:, starts[l]:starts[l] + shapes[l][0] * shapes[l][1]].reshape(B, shapes[l][0], shapes[l][1], 256) for l in range(3)]
        mh = "detr.mask_head"
        f, _ = self.conv_kxk(lv[2].contiguous(), mh + ".lay3", act=ops.ACT_RELU)
        f = lv[1] + self._nearest_up(f, shapes[1])
        f, _ = self.conv_kxk(f.contiguous(), mh + ".lay4", act=ops.ACT_RELU)
        f = lv[0] + self._nearest_up(f, shapes[0])
        f, _ = self.conv_kxk(f.contiguous(), mh + ".jia_dcn", act=ops.ACT_RELU)
        f, _ = self.conv_kxk(f, mh + ".lay1", act=ops.ACT_RELU)
        f, _ = self.conv_kxk(f, mh + ".lay2", act=ops.ACT_RELU)                                 # (B, H/8, W/8, 8)
        Hf, Wf = shapes[0]
        masks = ops.condinst_masks(f.view(B, Hf * Wf, 8), params, ref_px, Hf, Wf, 8)
        return masks, f, params, ref_px

    @staticmethod
    def _nearest_up(x_nhwc, size):
        """F.interpolate(mode='nearest') on NHWC (index glue; ddetrs_dn.py:1661,1673)."""
        B, h, w, C = x_nhwc.shape
        H, Wd = size
        yi = (torch.arange(H, device=x_nhwc.device) * h // H)
        xi = (torch.arange(Wd, device=x_nhwc.device) * w // Wd)
        return x_nhwc[:, yi][:, :, xi]

    # ------------------------------------------------------------ MaskDINO branch
    def maskdino(self, feats, B, forced_topk=None, pixel_decoder_only=False):
        """MaskDINOEncoder.forward_features + MaskDINODecoder.forward (H/models/maskdino/pixel_decoder/maskdino_encoder.py:368-434,
        transformer_decoder/maskdino_decoder.py:377-529, dino_decoder.py:94-168)."""
        W, hp = self.W, self.hp
        pd, pr = "detr.mask_dino.pixel_decoder", "detr.mask_dino.predictor"
        lv, shapes, starts, S, shapes_t, lsi_t = self._levels(feats)
        src = self._input_proj(pd, lv, starts, S, B)
        # MaskDINO always passes mask=None (maskdino_encoder.py:82-88): shape-only, cached per resolution
        pos = W.cached(("sine_pos_md", B, tuple(shapes)), lambda: self._level_pos(
            [torch.zeros(B, h, w, dtype=torch.bool, device=self.device) for h, w in shapes], 0.0, W[pd + ".transformer.level_embed"]))
        ref_enc = self.encoder_reference_points(shapes, torch.ones(B, 4, 2, device=self.device), self.device)
        _, src_s = ops.add_split(src)
        for i in range(hp.get("md_enc_layers", 6)):
            src, src_s = self.encoder_layer(f"{pd}.transformer.encoder.layers.{i}", src, src_s, pos, ref_enc, None, shapes_t, lsi_t, B, S,
                                            shapes_host=shapes)
        # FPN level on res3 (:418-427): lateral 1x1+GN, + out[0] (same size -> bilinear resize is the identity), 3x3+GN+ReLU
        h3, w3 = shapes[0]
        lat = self.conv1x1_gn(lv[0][1], pd + ".adapter_1", pd + ".adapter_1.norm", bias=False)              # (B, hw, 256)
        yv = (lat + src[:, :h3 * w3]).view(B, h3, w3, 256).contiguous()
        cols, _, _ = ops.im2col_nhwc(yv, 3, 1, 1)
        wl, _ = W.conv_kxk(pd + ".layer_1")
        o, _, _ = ops.gemm(cols, wl)
        _, o_s = ops.groupnorm_nhwc(o.view(B, h3 * w3, 256), W[pd + ".layer_1.norm.weight"], W[pd + ".layer_1.norm.bias"], relu=True,
                                    want_f32=False, want_split=True)
        # mask_features: ConvT(2x2,s2) -> GN -> ReLU -> 1x1 conv, kept NHWC (B, 4*h3*w3, 256) as bf16 planes
        wt, bt = W.convT2(pd + ".mask_features.0")
        g, _, _ = ops.gemm(o_s.view(B * h3 * w3, 256), wt, bias=bt)
        up, _ = ops.pixel_shuffle2(g, B, h3, w3, 256)
        HWm = 4 * h3 * w3
        _, up_s = ops.groupnorm_nhwc(up.view(B, HWm, 256), W[pd + ".mask_features.1.weight"], W[pd + ".mask_features.1.bias"], relu=True,
                                     want_f32=False, want_split=True)
        w1, b1 = W.lin(pd + ".mask_features.3")
        _, mf_s, _ = ops.gemm(up_s.view(B * HWm, 256), w1, bias=b1, want_f32=False, want_split=True)       # (B*HWm, 256)
        if pixel_decoder_only:       # MaskDINOEncoder.forward_features contract: NCHW mask features + the 4 encoder levels
            ms = [src[:, starts[i]:starts[i] + shapes[i][0] * shapes[i][1]].reshape(B, shapes[i][0], shapes[i][1], 256).permute(0, 3, 1, 2)
                  for i in range(4)]
            return dict(mask_features=mf_s.float().view(B, 2 * h3, 2 * w3, 256).permute(0, 3, 1, 2), multi_scale=ms)
        # ---- decoder: levels re-flattened coarse -> fine (maskdino_decoder.py:398-404)
        order = [3, 2, 1, 0]
        dshapes = [shapes[i] for i in order]
        mem = torch.cat([src[:, starts[i]:starts[i] + shapes[i][0] * shapes[i][1]] for i in order], 1).contiguous()
        _, mem_s = ops.add_split(mem)
        _, _, dshapes_t, dlsi_t = self._level_index(dshapes)
        zmask = torch.zeros(B, S, dtype=torch.bool, device=self.device)
        props, om_n, om_ns = self._enc_proposals(pr, mem, dshapes, zmask, B, S, pad_fill=False)
        wc, bc = W.lin(pr + ".class_embed")
        cls_all, _, _ = ops.gemm(om_ns, wc, bias=bc)
        enc_scores = cls_all.view(B, S, -1).max(-1)[0]
        nq = hp.get("md_queries", 300)
        topk, tgt, tgt_s, ref = self._select_queries(om_n, props, enc_scores, nq, pr + "._bbox_embed", B, forced_topk)
        dec_hs, refs = self._dino_decoder(pr + ".decoder", [pr + "._bbox_embed"] * hp.get("md_dec_layers", 9), tgt, tgt_s, ref,
                                          torch.ones(B, 4, 4, device=self.device), mem_s, None, dshapes_t, dlsi_t, B, nq, S)
        refs = [ref] + refs
        # intermediate = decoder_norm(output); prediction heads apply decoder_norm again (double LN, dino_decoder.py:163 + :521)
        gn, bn = W[pr + ".decoder_norm.weight"], W[pr + ".decoder_norm.bias"]
        hs, hs_s, _ = ops.layernorm(dec_hs[-1][0].view(B * nq, 256), gn, bn, 1e-5, want_f32=True, want_split=True)
        dec, dec_s, _ = ops.layernorm(hs, gn, bn, 1e-5, want_f32=True, want_split=True)
        cls_emb, cls_emb_s, _ = ops.gemm(dec_s, wc, bias=bc, want_split=True)                              # (B*nq, 256) "pred_logits" embedding
        me_s = self.mlp(dec_s, pr + ".mask_embed", 3, last_f32=False)                                      # BF2 (B*nq, 256)
        # mask-embed contraction out[b, q, hw] = sum_c mask_embed[b, q, c] * mask_features[b, hw, c]: the queries are the (3) M tiles,
        # the pixel map is the streamed W operand -- read from HBM once (the M tiles of one pixel tile run back to back and
        # share it through L2), rows written with coalesced stores, sigmoid > 0.5 fused as a bit-packed second output
        pm, _, bits = ops.gemm(me_s, mf_s, M=nq, N=HWm, K=256, batch=B, lda=256, ldw=256, a_bstride=nq * 256, w_bstride=HWm * 256,
                               bits_threshold=0.0)
        pred_masks = pm.view(B, nq, 2 * h3, 2 * w3)
        box = (self.mlp(hs_s, pr + "._bbox_embed", 3).view(B, nq, 4) + inverse_sigmoid(refs[-2])).sigmoid()
        return dict(pred_logits_emb=cls_emb.view(B, nq, 256), pred_logits_emb_s=cls_emb_s, pred_masks=pred_masks, mask_bits=bits,
                    pred_boxes=box, enc_scores=enc_scores, topk=topk, mask_features_s=mf_s)
