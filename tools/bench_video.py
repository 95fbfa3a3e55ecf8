"""GPU: video object segmentation by label propagation (dinov3_jax/eval/video.py) at the DAVIS 2017 480p shape: ViT-L/16
(random weights), 854 x 480 frames resized to 832 x 480 (52 x 30 = 1 560 patches), n_ctx = 8 context frames (frame 0
and the 7 last), size_mask_neighborhood 12, topk 5, C = 4 channels.

Timed apart, with CUDA events after a warm-up:
  1. feature extraction per frame, in batches of 16: d3_video_resize, get_intermediate_layers(n=1), d3_knn_normalize;
  2. propagation per frame: the two similarity GEMMs (1 560 x 12 480 x 1 024 in all), d3_video_propagate and
     d3_video_label_map to 854 x 480, together and each alone;
  3. d3_video_jf_counts for one 854 x 480 frame and 3 objects (disk radius 8).

Prints the card and its power limit with the numbers.   python tools/bench_video.py [--iters N]
"""
import argparse
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path[:0] = [os.path.join(ROOT, "dinov3-jax_b200"), ROOT]
import numpy as np
import torch

from bench_features import CONFIGS, PATCH, R, random_tree
from dinov3_jax import ops
from dinov3_jax.eval.video import boundary_radius, sequence_features
from dinov3_jax.models import DinoVisionTransformer
from gpu_timing import card, cuda_ms

bf16, f32 = torch.bfloat16, torch.float32
H, W, RH, RW, B, N_CTX, C = 480, 854, 480, 832, 16, 8, 4
h, w = RH // PATCH, RW // PATCH
P = h * w
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def vit_l():
    _, D, L, Hh, ffn, ratio, mkb, norm_layer = CONFIGS["vitl"]
    g = torch.Generator(device="cuda").manual_seed(0)
    return DinoVisionTransformer(random_tree(D, L, ffn, ratio, g), patch_size=PATCH, embed_dim=D, n_blocks=L,
                                 num_heads=Hh, ffn_ratio=ratio, ffn_layer=ffn, mask_k_bias=mkb, n_storage_tokens=R,
                                 norm_layer=norm_layer)


def bench_features(model, iters):
    rng = np.random.default_rng(0)
    frames = torch.from_numpy(rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)).cuda()
    with torch.no_grad():
        ms = cuda_ms(lambda: sequence_features(model, frames, (RH, RW), B, MEAN, STD), iters, 2)
    print(f"features (resize {W}x{H} -> {RW}x{RH}, ViT-L/16 get_intermediate_layers n=1, L2 normalise) batch {B}: "
          f"{ms:.2f} ms, {ms / B:.2f} ms per frame")


def bench_propagation(iters):
    g = torch.Generator().manual_seed(1)
    D = CONFIGS["vitl"][1]
    feats = torch.nn.functional.normalize(torch.randn(N_CTX * P + P, D, generator=g), dim=1).to(bf16).cuda()
    labels = torch.rand(N_CTX * P, C, generator=g).cuda()
    tgt = feats[N_CTX * P:]
    ld = -(-P // 8) * 8
    sim0 = torch.empty(P, ld, device="cuda")[:, :P]
    simr = torch.empty(P, -(-(N_CTX - 1) * P // 8) * 8, device="cuda")[:, :(N_CTX - 1) * P]
    soft = torch.empty(P, C, device="cuda")
    pred = torch.empty(H, W, dtype=torch.uint8, device="cuda")

    def gemms():
        ops.gemm(tgt, feats[:P], sim0)
        ops.gemm(tgt, feats[P:N_CTX * P], simr)

    prop = lambda: ops.video_propagate(sim0, simr, labels[:P], labels[P:], (h, w), 12, 5, 0.1, soft)
    label = lambda: ops.video_label_map(soft, (h, w), PATCH, pred)

    def frame():
        gemms(); prop(); label()

    t = {name: cuda_ms(fn, iters, 3) for name, fn in (("frame", frame), ("gemms", gemms), ("propagate", prop),
                                                       ("label map", label))}
    flop = 2.0 * P * N_CTX * P * D
    print(f"propagation per frame ({h}x{w} patches, n_ctx {N_CTX}, r 12, k 5, C {C}, label map to {W}x{H}): "
          f"{t['frame']:.3f} ms; similarity GEMMs {t['gemms']:.3f} ms ({flop / t['gemms'] / 1e9:.0f} TFLOP/s of "
          f"{flop / 1e9:.1f} GFLOP), d3_video_propagate {t['propagate']:.3f} ms, d3_video_label_map "
          f"{t['label map']:.3f} ms")


def bench_jf(iters):
    rng = np.random.default_rng(2)
    cells = rng.integers(0, 4, (12, 20))
    gt = np.ascontiguousarray(cells[np.arange(H) * 12 // H][:, np.arange(W) * 20 // W], dtype=np.uint8)
    pred = np.roll(gt, 3, axis=1)
    gt[rng.random((H, W)) < 0.01] = 255
    g, p = torch.from_numpy(gt[None]).cuda(), torch.from_numpy(pred[None]).cuda()
    counts = torch.empty(1, 3, 6, dtype=torch.int64, device="cuda")
    r = boundary_radius(H, W)
    ms = cuda_ms(lambda: ops.video_jf_counts(p, g, 3, r, counts), iters, 3)
    print(f"d3_video_jf_counts {W}x{H}, 3 objects, radius {r}: {ms * 1e3:.1f} us per frame")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    from dinov3_jax import _native
    _native.init(0)
    print(card())
    bench_features(vit_l(), max(args.iters // 4, 3))
    bench_propagation(args.iters)
    bench_jf(args.iters)
    print(card())


if __name__ == "__main__":
    main()
