"""GPU: d3_koleo_topk_rows (distributed top-k KoLeo, forward and backward) at the shapes the training step runs.

(B, N, D, k) = (64, 64, 1024, 1)    one ViT-L rank, its own 64 rows (the plain KoLeo through the new kernel);
               (8, 16, 4096, 1)     dinov3_vit7b16_high_res_adapt: 8 images per GPU, loss groups of 16, D = 4096;
               (64, 4096, 1024, 4)  64 ranks of 64 ViT-L rows in one group, top-4.
Each is one call per crop of the step: the local rows [0, B) against every row of the group.  Timed with CUDA events
over many calls after a warm-up; the call includes its workspace allocation from the stream-ordered pool.

Prints the card, its power limit and maximum SM clock with the numbers.   python tools/bench_koleo.py [--iters N]
"""
import argparse
import json
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path[:0] = [os.path.join(ROOT, "dinov3-jax_b200"), ROOT]
import torch

from dinov3_jax import _native, ops
from gpu_timing import card, cuda_ms

SHAPES = [(64, 64, 1024, 1), (8, 16, 4096, 1), (64, 4096, 1024, 4)]


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--iters", type=int, default=200)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU: nothing here runs on the CPU")
    _native.init(0)
    out = {"card": card(), "kernel": "d3_koleo_topk_rows (norm, scan, select + loss, backward gather, metric)",
           "shapes": []}
    for B, N, D, k in SHAPES:
        torch.manual_seed(0)
        x = torch.randn(N, D, device="cuda")
        dx, met = torch.zeros_like(x), torch.zeros(1, device="cuda")
        scratch = ops.koleo_topk_scratch(N, D, B, k, "cuda")
        fn = lambda: ops.koleo_topk(x, (0, N), 0, B, k, scratch, met, dx, 1.0, 1.0)
        ms = cuda_ms(fn, a.iters, warmup=20)
        out["shapes"].append({"B": B, "N": N, "D": D, "k": k, "us_per_call": round(ms * 1e3, 2),
                              "dot_flops": 2 * B * N * D})
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
