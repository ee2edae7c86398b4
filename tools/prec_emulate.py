"""CPU emulation of tensor-core operand formats on the oracle (experiment driver, test infrastructure).

Rounds the operands of every nn.Linear / conv / ViT attention matmul to a 16-bit format before the fp32 product, which is
what a one-pass fp16 tensor-core contraction (wgmma) computes (exact products, fp32 accumulation), and reports how far the
final outputs move from the plain fp32 oracle.  Used to choose the per-contraction precision map (DESIGN.md §3).
"""
import argparse, os, sys, time
import torch
import torch.nn as nn
import torch.nn.functional as F
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from hipie_oracle import hparams, synth, vit as ovit
from hipie_oracle.model import HipieOracle

MODE = {"vit_lin": None, "vit_attn": None, "other": None}


def q(x, fmt):
    if fmt is None:
        return x
    if fmt == "f16":
        return x.half().float()
    if fmt == "bf16":
        return x.bfloat16().float()
    if fmt == "f16x2":       # hi + lo: ~22 bits
        h = x.half().float()
        return h + (x - h).half().float()
    raise ValueError(fmt)


_orig_linear = F.linear
_scope = ["other"]


def linear_q(x, w, b=None):
    fmt = MODE[_scope[0]] if _scope[0] != "vit_attn" else MODE["vit_lin"]
    return _orig_linear(q(x, fmt), q(w, fmt), b)


def attn_forward(self, x):
    B, H, W, _ = x.shape
    qkv = self.qkv(x).reshape(B, H * W, 3, self.num_heads, -1).permute(2, 0, 3, 1, 4)
    qq, k, v = qkv.reshape(3, B * self.num_heads, H * W, -1).unbind(0)
    f = MODE["vit_attn"]
    attn = q(qq * self.scale, f) @ q(k, f).transpose(-2, -1)
    attn = ovit.add_decomposed_rel_pos(attn, qq, self.rel_pos_h, self.rel_pos_w, (H, W), (H, W))
    attn = attn.softmax(dim=-1)
    x = (q(attn, f) @ q(v, f)).view(B, self.num_heads, H, W, -1).permute(0, 2, 3, 1, 4).reshape(B, H, W, -1)
    return self.proj(x)


def run(model, inputs, ids, am, modes, forced=None):
    MODE.update(modes)
    vit = model.detr.detr.backbone[0].backbone
    orig_fwd = vit.forward

    def vit_fwd(x):
        _scope[0] = "vit_lin"
        try:
            return orig_fwd(x)
        finally:
            _scope[0] = "other"
    vit.forward = vit_fwd
    F.linear = linear_q
    ovit.Attention.forward_orig = getattr(ovit.Attention, "forward_orig", ovit.Attention.forward)
    ovit.Attention.forward = attn_forward
    try:
        with torch.no_grad():
            return model(inputs, ids, am, forced=forced)
    finally:
        F.linear = _orig_linear
        vit.forward = orig_fwd
        ovit.Attention.forward = ovit.Attention.forward_orig


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hp", default="vit_tiny")
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--classes", type=int, default=5)
    ap.add_argument("--depth", type=int, default=0)
    ap.add_argument("--combos", default="")
    args = ap.parse_args()
    torch.manual_seed(0)
    hp = hparams.get(args.hp)
    if args.depth:
        hp["vit"] = dict(hp["vit"], depth=args.depth)
    model = HipieOracle(hp).eval()
    synth.perturb_(model)
    inputs, ids, am = synth.make_batch(1, args.size, args.size, args.classes, hp["max_query_len"])
    t0 = time.time()
    res0, out0 = run(model, inputs, ids, am, dict(vit_lin=None, vit_attn=None, other=None))
    print(f"baseline {time.time()-t0:.1f}s", flush=True)
    forced = {'topk_fg': out0['aux']['topk'], 'topk_md': out0['md']['topk']}
    combos = [("vit_lin f16", dict(vit_lin="f16", vit_attn=None, other=None)),
              ("vit_attn f16 only", dict(vit_lin=None, vit_attn="f16", other=None)),
              ("vit_attn bf16 only", dict(vit_lin=None, vit_attn="bf16", other=None)),
              ("other f16 only", dict(vit_lin=None, vit_attn=None, other="f16")),
              ("all bf16", dict(vit_lin="bf16", vit_attn="bf16", other="bf16")),
              ("all f16x2", dict(vit_lin="f16x2", vit_attn="f16x2", other="f16x2"))]
    if args.combos:
        combos = [c for c in combos if c[0] in args.combos.split(",")]
    keys = ["pred_masks_maskdino", "pred_masks", "pred_logits", "pred_boxes", "pred_logits_maskdino"]
    for name, m in combos:
        res, out = run(model, inputs, ids, am, m, forced=forced)
        errs = {k: (out[k] - out0[k]).abs().max().item() for k in keys}
        f0 = out0["features"]["res4"]
        ef = (out["features"]["res4"] - f0).abs().max().item()
        tk = len(set(out["aux"]["topk"][0].tolist()) & set(out0["aux"]["topk"][0].tolist())) / out0["aux"]["topk"].shape[1]
        print(f"{name:22s} res4 {ef:.2e} (max {f0.abs().max():.1f}) | " + " ".join(f"{k}={v:.2e}" for k, v in errs.items()) + f" | topk overlap {tk:.3f}"
              f" | max|md mask| {out0['pred_masks_maskdino'].abs().max():.1f} max|fg mask| {out0['pred_masks'].abs().max():.1f}", flush=True)


if __name__ == "__main__":
    main()
