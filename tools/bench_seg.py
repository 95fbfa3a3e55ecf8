"""GPU: the linear segmentation probe (dinov3_jax/eval/segmentation.py) at the ADE20K shape: ViT-L/16, crop 512^2
(32 x 32 patches), B = 16, 150 classes, the last block's patch tokens (n = 1, 1 024 channels).

Timed apart, with CUDA events after a warm-up:
  1. d3_seg_xent_fwd_bwd: 16 x 32 x 32 logits -> 16 x 512^2 pixels, 150 classes, the loss and the bf16 dZ; against the
     torch path on the same GPU (F.interpolate(bilinear, align_corners=False) + F.cross_entropy(ignore_index=255) +
     autograd, fp32).  The bytes it needs: the fp32 logits and the uint8 labels read, dZ (bf16) written.
  2. the head step of SegLinearHead.step: BatchNorm statistics and x_hat, the logit GEMM, the loss, the weight and
     bias gradients and the AdamW update;
  3. the ViT-L/16 feature forward at 512^2 (1 024 patch tokens per image, random weights) and the feature rows;
  4. whole-image evaluation: 512 x 683 val images resized to 512 x 688, the forward, the head's logits and the
     confusion matrix, images per second (decoding not included).

Prints the card and its power limit with the numbers.   python tools/bench_seg.py [--iters N]
"""
import argparse
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path[:0] = [os.path.join(ROOT, "dinov3-jax_b200"), ROOT]
import torch
import torch.nn.functional as Fn

from dinov3_jax import ops
from dinov3_jax.eval.segmentation import SegLinearHead, eval_size, write_seg_features
from gpu_timing import card, cuda_ms

bf16, f32 = torch.bfloat16, torch.float32
B, C, D, S, P = 16, 150, 1024, 512, 16
h = w = S // P


def bench_xent(iters):
    g = torch.Generator().manual_seed(0)
    Cp = -(-C // 8) * 8
    logits = torch.zeros(B * h * w, Cp)
    logits[:, :C] = torch.randn(B * h * w, C, generator=g) * 4
    labels = torch.randint(0, C, (B, S, S), generator=g).to(torch.uint8)
    labels[torch.rand(B, S, S, generator=g) < 0.1] = 255
    L, lab = logits.cuda(), labels.cuda()
    loss, count = torch.empty(1, device="cuda"), torch.empty(1, dtype=torch.int32, device="cuda")
    dz = torch.empty(B * h * w, Cp, dtype=bf16, device="cuda")
    ms = cuda_ms(lambda: ops.seg_xent_fwd_bwd(L, lab, (h, w), C, loss, count, dz_bf16=dz, Cp=Cp), iters, 3)
    nbytes = L.numel() * 4 + lab.numel() + dz.numel() * 2
    Lt = L[:, :C].reshape(B, h, w, C).permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    yl = lab.long()

    def torch_path():
        up = Fn.interpolate(Lt, size=(S, S), mode="bilinear", align_corners=False)
        Lt.grad = None
        Fn.cross_entropy(up, yl, ignore_index=255).backward()

    ms_t = cuda_ms(torch_path, max(iters // 4, 3), 2)
    torch_path()
    ref = Lt.grad.permute(0, 2, 3, 1).reshape(-1, C)
    err = ((dz[:, :C].float() - ref).norm() / ref.norm()).item()
    print(f"d3_seg_xent_fwd_bwd B={B} {h}x{w} -> {S}^2 C={C}: {ms:.3f} ms, {nbytes / ms / 1e6:.1f} GB/s of the "
          f"{nbytes / 1e6:.1f} MB it must move; torch interpolate + cross_entropy + autograd: {ms_t:.3f} ms "
          f"({ms_t / ms:.1f}x); dZ vs torch fp32 rel L2 {err:.1e}; loss {loss.item():.5f}")


def bench_head(iters):
    g = torch.Generator().manual_seed(1)
    head = SegLinearHead(D, C, B * h * w, 40000, device="cuda")
    x = (torch.randn(B * h * w, D, generator=g) * 2 + 1).to(bf16).cuda()
    labels = torch.randint(0, C, (B, S, S), generator=g).to(torch.uint8).cuda()
    it = [0]

    def step():
        head.step(x, labels, (h, w), it[0])
        it[0] += 1

    ms = cuda_ms(step, iters, 3)
    gemm_flop = 2 * 2.0 * B * h * w * D * head.Cp
    print(f"head step (BN stats + x_hat, logit GEMM, loss, dW GEMM, db, AdamW) B={B} rows={B * h * w} K={D} C={C}: "
          f"{ms:.3f} ms ({gemm_flop / 1e9:.1f} GFLOP of GEMM)")


def vit_l():
    from dinov3_jax.checkpointer import tree_from_flat
    from dinov3_jax.models import DinoVisionTransformer
    from oracle.arch import ModelCfg
    from oracle.model import init_backbone
    cfg = ModelCfg(embed_dim=D, depth=24, heads=16)
    return DinoVisionTransformer(tree_from_flat(init_backbone(cfg, torch.Generator().manual_seed(0))), embed_dim=D,
                                 n_blocks=24, num_heads=16)


def bench_features(model, iters):
    images = torch.randn(B, S, S, 3, generator=torch.Generator().manual_seed(2)).to(bf16).cuda()
    out = torch.empty(B * h * w, D, dtype=bf16, device="cuda")
    ms = cuda_ms(lambda: write_seg_features(model, images, 1, out), iters, 2)
    print(f"ViT-L/16 features at {S}^2 ({h * w} patch tokens, last block): {ms:.1f} ms per batch of {B}, "
          f"{B / ms * 1e3:,.1f} images/s")


def bench_eval(model, iters):
    from dinov3_jax.eval.segmentation import _pack_seg
    import numpy as np
    rng = np.random.default_rng(3)
    H, W = 512, 683
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    lab = rng.integers(0, C, (H, W), dtype=np.uint8)
    flat, lab_flat, desc = _pack_seg([(img, lab)])
    flat, lab_flat, desc = flat.cuda(), lab_flat.cuda(), desc.cuda()
    head = SegLinearHead(D, C, 64, 10, device="cuda")
    rh, rw = eval_size(H, W, S, P)
    box = torch.tensor([[rh, rw, 0, 0, 0, 0]], dtype=torch.int32, device="cuda")
    conf = torch.zeros(C, C, dtype=torch.int64, device="cuda")
    taps = ops.seg_max_taps([(H, W)], [(rh, rw)])

    def one():
        x = torch.empty(1, rh, rw, 3, dtype=bf16, device="cuda")
        ops.seg_crop(flat, desc, box, x, max_taps=taps, mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225))
        feats = torch.empty((rh // P) * (rw // P), D, dtype=bf16, device="cuda")
        write_seg_features(model, x, 1, feats)
        ops.seg_predict_confusion(head.logits(feats), lab_flat.view(1, H, W), (rh // P, rw // P), C, conf)

    ms = cuda_ms(one, iters, 2)
    print(f"whole-image evaluation {H}x{W} -> {rh}x{rw} (ViT-L/16, C={C}): {ms:.1f} ms per image, "
          f"{1e3 / ms:.1f} images/s")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    from dinov3_jax import _native
    _native.init(0)
    print(card())
    bench_xent(args.iters)
    bench_head(args.iters)
    model = vit_l()
    bench_features(model, max(args.iters // 4, 3))
    bench_eval(model, args.iters)
    print(card())


if __name__ == "__main__":
    main()
