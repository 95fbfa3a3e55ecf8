"""GPU: the linear depth probe (dinov3_jax/eval/depth.py) at the NYU Depth v2 train shape: ViT-L/16, crop 416 x 544
(26 x 34 patches), B = 16, 256 depth bins, the last block's patch and class tokens (n = 1, 2 048 channels).

Timed apart, with CUDA events after a warm-up:
  1. d3_depth_head_fwd_bwd: 16 x 26 x 34 bin logits -> 16 x 416 x 544 pixels, the scale-invariant log loss and the
     bf16 dZ; against the torch path on the same GPU (bin normalisation + F.interpolate(bilinear,
     align_corners=False) + the loss + autograd, fp32).  The bytes it needs: the fp32 logits and ground truth read,
     dZ (bf16) written.
  2. the head step of DepthLinearHead.step: BatchNorm statistics and x_hat, the logit GEMM, the loss, the weight and
     bias gradients and the AdamW update;
  3. d3_depth_predict_metrics for one NYU val frame: 30 x 40 cells -> 480 x 640 pixels with the Eigen crop.

Prints the card and its power limit with the numbers.   python tools/bench_depth.py [--iters N]
"""
import argparse
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path[:0] = [os.path.join(ROOT, "dinov3-jax_b200"), ROOT]
import torch
import torch.nn.functional as Fn

from dinov3_jax import ops
from dinov3_jax.eval.depth import EIGEN_CROP, DepthLinearHead
from gpu_timing import card, cuda_ms

bf16, f32 = torch.bfloat16, torch.float32
B, NB, D, HC, WC, P = 16, 256, 1024, 416, 544, 16
h, w = HC // P, WC // P
LO, HI = 0.001, 10.0


def _gt(Bn, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    gt = torch.rand(Bn, H, W, generator=g) * 9.0 + 0.5
    gt[torch.rand(Bn, H, W, generator=g) < 0.1] = 0.0          # missing depth
    return gt.cuda()


def bench_loss(iters):
    g = torch.Generator().manual_seed(0)
    L = (torch.randn(B * h * w, NB, generator=g) * 2).cuda()
    gt = _gt(B, HC, WC, 1)
    loss, count = torch.empty(1, device="cuda"), torch.empty(1, dtype=torch.int32, device="cuda")
    dz = torch.empty(B * h * w, NB, dtype=bf16, device="cuda")
    ms = cuda_ms(lambda: ops.depth_head_fwd_bwd(L, gt, (h, w), NB, LO, HI, loss, count, dz_bf16=dz, Cp=NB), iters, 3)
    nbytes = L.numel() * 4 + gt.numel() * 4 + dz.numel() * 2
    Lt = L.clone().requires_grad_(True)
    c = torch.linspace(LO, HI, NB, device="cuda")
    valid = (gt > LO) & (gt <= HI)

    def torch_path():
        q = torch.relu(Lt) + 0.1
        d = ((q * c).sum(-1) / q.sum(-1)).view(B, 1, h, w)
        dh = Fn.interpolate(d, size=(HC, WC), mode="bilinear", align_corners=False)[:, 0]
        gl = torch.log(dh[valid] + 1e-3) - torch.log(gt[valid] + 1e-3)
        Lt.grad = None
        torch.sqrt(torch.var(gl) + 0.15 * gl.mean() ** 2).backward()

    ms_t = cuda_ms(torch_path, max(iters // 4, 3), 2)
    torch_path()
    err = ((dz.float() - Lt.grad).norm() / Lt.grad.norm()).item()
    print(f"d3_depth_head_fwd_bwd B={B} {h}x{w} -> {HC}x{WC} bins={NB}: {ms:.3f} ms, {nbytes / ms / 1e6:.1f} GB/s of "
          f"the {nbytes / 1e6:.1f} MB it must move; torch bins + interpolate + loss + autograd: {ms_t:.3f} ms "
          f"({ms_t / ms:.1f}x); dZ vs torch fp32 rel L2 {err:.1e}; loss {loss.item():.5f}")


def bench_head(iters):
    g = torch.Generator().manual_seed(1)
    K = 2 * D
    head = DepthLinearHead(K, B * h * w, 38400, n_bins=NB, min_depth=LO, max_depth=HI, device="cuda")
    x = (torch.randn(B * h * w, K, generator=g) * 2 + 1).to(bf16).cuda()
    gt = _gt(B, HC, WC, 2)
    it = [0]

    def step():
        head.step(x, gt, (h, w), it[0])
        it[0] += 1

    ms = cuda_ms(step, iters, 3)
    gemm_flop = 2 * 2.0 * B * h * w * K * head.Cp
    print(f"head step (BN stats + x_hat, logit GEMM, loss, dW GEMM, db, AdamW) B={B} rows={B * h * w} K={K} "
          f"bins={NB}: {ms:.3f} ms ({gemm_flop / 1e9:.1f} GFLOP of GEMM)")


def bench_metrics(iters):
    g = torch.Generator().manual_seed(3)
    hv, wv = 30, 40
    L = (torch.randn(hv * wv, NB, generator=g) * 2).cuda()
    gt = _gt(1, 480, 640, 4)
    sums = torch.empty(1, 9, dtype=torch.float64, device="cuda")
    ms = cuda_ms(lambda: ops.depth_predict_metrics(L, gt, (hv, wv), NB, LO, HI, sums, crop=EIGEN_CROP), iters, 3)
    print(f"d3_depth_predict_metrics {hv}x{wv} -> 480x640 bins={NB}, Eigen crop: {ms * 1e3:.1f} us per image")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    from dinov3_jax import _native
    _native.init(0)
    print(card())
    bench_loss(args.iters)
    bench_head(args.iters)
    bench_metrics(args.iters)
    print(card())


if __name__ == "__main__":
    main()
