"""Micro-benchmark of the instance-overlap kernels against the reference's per-image host hand-off.

  pack      hipie_mask_pack on N (H, W) uint8 masks: bytes read / time
  expand    hipie_rle_expand of M GT run lists (random blobs, a few hundred runs each)
  overlaps  hipie_mask_overlaps, the N x M intersection table (b1 MMA)
  d2h       the reference's COCOEvaluator.process starts with instances.to(cpu): the N masks copied to pageable host memory.  That copy
            is a lower bound on its per-image cost; the pycocotools RLE encoding that follows is absent here and not timed.

N = 100 at M in {20, 300}, 512 x 683 and 1024 x 1365.  Kernel times are CUDA events over many launches after a warm-up; the copy is
a wall clock over repetitions.  The card's name and power limit are read in the same run.

    python tools/instance_eval_micro.py [--iters 50] [--out profiles/instance_eval_micro.txt]
"""
import argparse
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.eval_micro import gpu_info, time_kernel  # noqa: E402

SHAPES = [(512, 683), (1024, 1365)]


def blobs(rng, n, H, W):
    """n masks of random ellipses (the shape of real instance masks: a few runs per column)."""
    yy, xx = np.mgrid[:H, :W]
    out = np.zeros((n, H, W), bool)
    for i in range(n):
        cy, cx = rng.rand() * H, rng.rand() * W
        ry, rx = (0.05 + rng.rand() * 0.3) * H, (0.05 + rng.rand() * 0.3) * W
        out[i] = ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 < 1
    return out


def runs_of(mask):
    flat = mask.T.reshape(-1).astype(np.int8)
    bounds = np.concatenate([[0], np.flatnonzero(np.diff(flat)) + 1, [flat.size]])
    counts = np.diff(bounds).tolist()
    return [0] + counts if flat[0] else counts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from hipie_b200 import ops
    rng = np.random.RandomState(0)
    lines = [f"# {gpu_info()}", "# N = 100 predicted masks; times in ms (CUDA events, mean of --iters launches); d2h = pageable copy of the "
             "masks (wall clock)"]
    for H, W in SHAPES:
        N = 100
        pm = torch.from_numpy(blobs(rng, N, H, W).astype(np.uint8)).cuda()
        t_pack = time_kernel(lambda: ops.mask_pack(pm), args.iters)
        pbits, _ = ops.mask_pack(pm)
        gbs = pm.numel() / (t_pack * 1e-3) / 1e9
        torch.cuda.synchronize()
        pm.cpu()
        t0 = time.perf_counter()
        for _ in range(5):
            pm.cpu()
        t_d2h = (time.perf_counter() - t0) * 1e3 / 5
        for M in (20, 300):
            gm = blobs(rng, M, H, W)
            ends, off = ops.rle_ends([runs_of(g) for g in gm], H, W)
            ends_d, off_d = torch.from_numpy(ends).cuda(), torch.from_numpy(off).cuda()
            err = torch.zeros(1, dtype=torch.int64, device="cuda")
            t_exp = time_kernel(lambda: ops.rle_expand(ends_d, off_d, H, W, err=err), args.iters)
            gbits = ops.rle_expand(ends_d, off_d, H, W)
            t_ov = time_kernel(lambda: ops.mask_overlaps(pbits, gbits, H, W), args.iters)
            inter = ops.mask_overlaps(pbits, gbits, H, W).cpu().numpy()
            want = pm.cpu().numpy().reshape(N, -1).astype(np.int64) @ gm.reshape(M, -1).astype(np.int64).T
            assert np.array_equal(inter, want), "overlap table differs from numpy"
            lines.append(f"{H}x{W} N={N} M={M} runs/GT={len(ends) / M:.0f}: pack {t_pack:.3f} ms ({gbs:.0f} GB/s read) | expand "
                         f"{t_exp:.3f} ms | overlaps {t_ov:.3f} ms | device total {t_pack + t_exp + t_ov:.3f} ms | masks d2h "
                         f"{t_d2h:.2f} ms ({pm.numel() / 1e6:.1f} MB)")
    text = "\n".join(lines)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
