"""CPU emulation of a PER-MODULE operand-format map on the oracle (experiment driver, test infrastructure).

tools/prec_emulate.py rounds whole classes of contractions; this one takes rules `regex=A_FMT/W_FMT` over the oracle's module
names (optional third field: format the OUTPUT is rounded to) (nn.Linear only) and rounds the activation / weight operand of the matching linears before the exact fp32 product:
`f16/f16` is what ONE fp16 wgmma pass computes, `f16/-` a two-pass scheme (A in one fp16 plane, W in hi + lo planes),
`-/f16` the other two-pass scheme.  The ViT attention itself (QK^T, P.V) always runs in the adopted fp16 mode here, so the
numbers are increments on top of the shipped precision map (DESIGN.md 3).

    python tools/prec_map_emulate.py --hp vit_h --size 512 --classes 20 --rules 'qkv1:blocks\.\d+\.attn\.qkv=f16/f16' ...
"""
import argparse, os, re, sys, time
import torch
import torch.nn as nn
import torch.nn.functional as F
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from hipie_oracle import hparams, synth, vit as ovit
from hipie_oracle.model import HipieOracle
import prec_emulate as pe


def q(x, fmt):
    return x if fmt in (None, "-", "") else pe.q(x, fmt)


def install(model, rules):
    n = 0
    for name, m in model.named_modules():
        m._emu = None
        if isinstance(m, nn.Linear):
            for rx, a, w, o in rules:
                if rx.search(name):
                    m._emu = (a, w, o)
                    n += 1
                    break
    return n


_orig_forward = nn.Linear.forward


def linear_forward(self, x):
    e = getattr(self, "_emu", None)
    if e is None:
        return _orig_forward(self, x)
    if e[0] == "f16+e4m3":      # fp16 hi x hi pass + ONE fp8 pass for the two cross terms: Ah.Wh + 2^-14 [e4m3(Ah) | e4m3(2^10 Al)] . [e4m3(2^14 Wl) | e4m3(2^4 Wh)]
        f8 = lambda t: t.clamp(-448.0, 448.0).to(torch.float8_e4m3fn).float()
        w = self.weight
        xh, wh = x.half().float(), w.half().float()
        xl, wl = x - xh, w - wh
        y = F.linear(xh, wh) + (F.linear(f8(xh), f8(wl * 2.0 ** 14)) + F.linear(f8(xl * 2.0 ** 10), f8(wh * 2.0 ** 4))) * 2.0 ** -14
        return y if self.bias is None else y + self.bias
    return q(F.linear(q(x, e[0]), q(self.weight, e[1]), self.bias), e[2])


def run(model, inputs, ids, am, forced=None, attn_fmt="f16"):
    pe.MODE.update(dict(vit_lin=None, vit_attn=attn_fmt, other=None))
    nn.Linear.forward = linear_forward
    orig = ovit.Attention.forward
    ovit.Attention.forward = pe.attn_forward
    try:
        with torch.no_grad():
            return model(inputs, ids, am, forced=forced)
    finally:
        nn.Linear.forward = _orig_forward
        ovit.Attention.forward = orig


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hp", default="vit_tiny")
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--classes", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--rules", nargs="*", default=[], help="name:regex=A/W[,regex=A/W...]")
    args = ap.parse_args()
    torch.manual_seed(args.seed)
    hp = hparams.get(args.hp)
    model = HipieOracle(hp).eval()
    synth.perturb_(model)
    inputs, ids, am = synth.make_batch(1, args.size, args.size, args.classes, hp["max_query_len"])
    install(model, [])
    t0 = time.time()
    res0, out0 = run(model, inputs, ids, am, attn_fmt=None)
    print(f"fp32 oracle {time.time()-t0:.1f}s", flush=True)
    forced = {'topk_fg': out0['aux']['topk'], 'topk_md': out0['md']['topk']}
    keys = ["pred_masks_maskdino", "pred_masks", "pred_logits", "pred_boxes", "pred_logits_maskdino"]
    combos = [("shipped (attention fp16 only)", [])]
    for r in args.rules:
        name, spec = r.split(":", 1)
        rules = []
        for part in spec.split(","):
            rx, fm = part.rsplit("=", 1)
            a, w, o = (fm.split("/") + ["-"])[:3]
            rules.append((re.compile(rx), a, w, o))
        combos.append((name, rules))
    for name, rules in combos:
        n = install(model, rules)
        res, out = run(model, inputs, ids, am, forced=forced)
        errs = {k: (out[k] - out0[k]).abs().max().item() for k in keys}
        f0 = out0["features"]["res4"]
        ef = (out["features"]["res4"] - f0).abs().max().item()
        print(f"{name:34s} [{n:3d} linears] res4 {ef:.2e} | " + " ".join(f"{k}={v:.2e}" for k, v in errs.items()), flush=True)


if __name__ == "__main__":
    main()
